"""Cost of the per-token entropy and the high-entropy token selection (top_entropy_quantile) at config (c) (Qwen3-4B, 36 layers, random
init, LoRA r = 32 with B ~ N(0, 0.01), 1 prompt x G = 8, P = 1852, C = 512, EOS suppressed).  Settings alternate in one process after
a warm-up; GPU times are CUDA events.  Measures:
  - the fused lm-head pass (br_lmhead_logprob_fwd) with and without the entropy output at M in {2048, 4096}, V = 151 936, K = 2560;
  - the entropy threshold at n = 4096 and n = 2^20;
  - training_step with top_entropy_quantile = 1 (off), log_entropy, and top_entropy_quantile = 0.2, dense with micro_rows = 4 (two row
    chunks: the no-grad entropy pre-pass runs) and with share_prompt_prefix (one chunk: the loss pass's entropies decide), plus the
    pre-pass's own GPU time from the trainer's phase events.
Prints one JSON object with the card name and power limit it was measured on.

    python scripts/entropy_bench.py [--reps 2] [--out FILE]
"""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:                                                  # the numbers stay usable without it
        return f"unknown ({e})"


def events_ms(fn, n=1):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def median(v):
    return sorted(v)[len(v) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--text", default="qwen3-4b")
    ap.add_argument("--completion", type=int, default=512)
    ap.add_argument("--no-train", action="store_true", help="skip the training_step timings")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    from bioreason_b200.build import ensure_built
    ensure_built()
    from bioreason_b200 import ops
    from bioreason_b200.configs import dna_config, text_config
    from bioreason_b200.models import DNALLMModel
    from bioreason_b200.synth import synth_batch
    from bioreason_b200.trainer import DNALLMGRPOConfig
    from bioreason_b200.trainer.grpo_trainer import DNALLMGRPOTrainer
    tc, dc = text_config(args.text), dna_config("nt-v2-500m")
    G, C, V, K = 8, args.completion, tc.vocab_size, tc.hidden_size
    res = {"card": card(), "model": args.text, "layers": tc.num_hidden_layers, "rows": G, "C": C}

    # ---- the lm-head pass alone
    g = torch.Generator(device="cuda").manual_seed(0)
    w = (torch.randn(V, K, generator=g, device="cuda") * K ** -0.5).to(torch.bfloat16)
    lm = {}
    for M in (2048, 4096):
        h = torch.randn(M, K, generator=g, device="cuda").to(torch.bfloat16)
        tgt = torch.randint(0, V, (M,), generator=g, device="cuda")
        fns = {"plain": lambda: ops.lmhead_logprob(h, w, tgt), "entropy": lambda: ops.lmhead_logprob(h, w, tgt, want_entropy=True)}
        for f in fns.values():
            events_ms(f, 3)
        t = {k: [] for k in fns}
        for _ in range(5):
            for k, f in fns.items():
                t[k].append(events_ms(f, 20))
        flops = 2.0 * M * V * K
        lm[str(M)] = {k: {"ms": round(median(v), 4), "tflops": round(flops / median(v) / 1e9, 1)} for k, v in t.items()}
        lm[str(M)]["extra_pct"] = round(100 * (median(t["entropy"]) / median(t["plain"]) - 1), 2)
    res["lmhead_V151936_K2560"] = lm
    del w

    # ---- the threshold kernel
    thr = {}
    for n in (4096, 1 << 20):
        x = torch.rand(n, device="cuda") * 8
        m_ = (torch.rand(n, device="cuda") < 0.8).to(torch.int32)
        f = lambda: ops.entropy_threshold(x, m_, 0.8)
        events_ms(f, 5)
        thr[str(n)] = round(median([events_ms(f, 50) for _ in range(3)]) * 1e3, 1)
    res["threshold_us"] = thr

    if not args.no_train:
        m = DNALLMModel(tc, dc, seed=1234)
        m.enable_lora(r=32, alpha=64.0, seed=3)
        with torch.no_grad():
            for p in m._lora.params[1::2]:
                p.normal_(0, 0.01)
        m.sync_adapters(rollout=False)
        b = synth_batch(tc, dc, batch=G, n_seq=2, dna_len=668, text_len=512, seed=8, same_prompt=True)
        batch = dict(input_ids=b["input_ids"], attention_mask=b["attention_mask"], dna_tokenized=b["dna_tokenized"], batch_idx_map=b["batch_idx_map"])
        res["P"] = b["input_ids"].shape[1]

        def reward(completion_ids, **kw_):
            return (completion_ids % 7 == 0).float().sum(1)
        settings = {}
        for layout, lkw in (("dense_2chunks", dict(micro_rows=4)), ("shared_1chunk", dict(share_prompt_prefix=True))):
            for name, ekw in (("off", {}), ("log_entropy", dict(log_entropy=True)), ("rho0.2", dict(top_entropy_quantile=0.2))):
                settings[f"{layout}/{name}"] = DNALLMGRPOConfig(
                    num_generations=G, max_completion_length=C, per_device_train_batch_size=G, suppress_eos=True, beta=0.04,
                    learning_rate=1e-6, lora_r=32, lora_alpha=64.0, **lkw, **ekw)
        trainers = {k: DNALLMGRPOTrainer(m, [reward], cfg) for k, cfg in settings.items()}
        steps = {k: [] for k in settings}
        prepass = {k: [] for k in settings}
        metrics = {}
        for rep in range(args.reps + 1):                                    # round 0: warm-up (weights, decode graph)
            for k, tr in trainers.items():
                tr.gpu_phase_ms()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                tr.training_step(batch)
                torch.cuda.synchronize()
                ph = tr.gpu_phase_ms()
                if rep:
                    steps[k].append(time.perf_counter() - t0)
                    prepass[k].append(ph.get("entropy_prepass", 0.0))
                metrics[k] = {n: round(v, 5) for n, v in tr.log_metrics().items() if n.startswith("entropy")}
        res["training_step_s"] = {k: [round(t, 3) for t in v] for k, v in steps.items()}
        res["grpo_tokens_per_s_median"] = {k: round(G * C / median(v), 1) for k, v in steps.items()}
        res["entropy_prepass_ms_median"] = {k: round(median(v), 1) for k, v in prepass.items() if median(v) > 0}
        res["entropy_metrics"] = metrics
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
