"""Cost and size of the rollout log-probs and the truncated importance-sampling (TIS) correction at config (c) (Qwen3-4B, 36 layers,
random init, LoRA r = 32 with B ~ N(0, 0.01), 1 prompt x G = 8, P = 1852, C = 512, EOS suppressed, the trainer's sampling settings
T = 0.6 / top_k = 20 / top_p = 0.95).  Settings with and without the log-prob output alternate in one process after a warm-up; GPU
times are CUDA events.  Measures:
  - the two-stage sampler at R = 8, V = 151 936, with and without the log-prob output;
  - the rollout with and without the output, bf16 and FP8 decode;
  - the four TIS statistics at cap 2 (br_grpo_loss_is_fwd_bwd) of the bf16 rollout (decode kernels versus the training kernels) and
    of the FP8 rollout, against the bf16 policy's log-probs from the training forward;
  - training_step tokens/s with the correction off and on, FP8 rollout off and on.
Prints one JSON object with the card name and power limit it was measured on.

    python scripts/rollout_is_bench.py [--reps 3] [--out FILE]
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
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1) / n


def median(v):
    return sorted(v)[len(v) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--text", default="qwen3-4b")
    ap.add_argument("--completion", type=int, default=512)
    ap.add_argument("--no-train", action="store_true", help="skip the training_step timings")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    from bioreason_b200.build import ensure_built
    ensure_built()
    from bioreason_b200 import ops, training
    from bioreason_b200.configs import dna_config, text_config
    from bioreason_b200.models import DNALLMModel
    from bioreason_b200.synth import synth_batch
    from bioreason_b200.trainer import DNALLMGRPOConfig
    from bioreason_b200.trainer.grpo_trainer import DNALLMGRPOTrainer
    tc, dc = text_config(args.text), dna_config("nt-v2-500m")
    G, C, V = 8, args.completion, tc.vocab_size
    res = {"card": card(), "model": args.text, "layers": tc.num_hidden_layers, "rows": G, "C": C}

    # ---- the two-stage sampler alone, R = 8
    logits = torch.randn(G, V, device="cuda") * 3
    ws = ops.sample_workspace(G, V, "cuda", logp=True)
    tok = torch.zeros(G, 1, device="cuda", dtype=torch.int64)
    lpb = torch.zeros(G, 1, device="cuda")
    uu = torch.rand(1, G, device="cuda")
    samp = lambda lp: (lambda: ops.sample_next(logits, workspace=ws, temperature=0.6, top_k=20, top_p=0.95, do_sample=True, uniforms=uu,
                                               max_steps=1, tokens=tok, logp=lp))
    for lp in (None, lpb):
        events_ms(samp(lp), 50)
    st = {"off": [], "on": []}
    for _ in range(args.reps):
        for name, lp in (("off", None), ("on", lpb)):
            st[name].append(events_ms(samp(lp), 500)[1] * 1e3)
    res["sampler_R8_us"] = {k: round(median(v), 2) for k, v in st.items()}
    res["sampler_R8_extra_us"] = round(median(st["on"]) - median(st["off"]), 2)

    # ---- model
    m = DNALLMModel(tc, dc, seed=1234)
    m.enable_lora(r=32, alpha=64.0, seed=3)
    with torch.no_grad():
        for p in m._lora.params[1::2]:
            p.normal_(0, 0.01)
    m.sync_adapters(rollout=False)
    b = synth_batch(tc, dc, batch=G, n_seq=2, dna_len=668, text_len=512, seed=8, same_prompt=True)
    batch = dict(input_ids=b["input_ids"], attention_mask=b["attention_mask"], dna_tokenized=b["dna_tokenized"], batch_idx_map=b["batch_idx_map"])
    res["P"] = b["input_ids"].shape[1]
    u = torch.rand(C, G, generator=torch.Generator().manual_seed(5))
    kw = dict(max_new_tokens=C, do_sample=True, temperature=0.6, top_k=20, top_p=0.95, uniforms=u, eos_token_id=-1, pad_token_id=0)

    # ---- rollout: output off / on alternating, per decode format
    roll, samples = {}, {}
    for fp8 in (False, True):
        fmt = "fp8" if fp8 else "bf16"
        m.set_fp8_rollout(fp8)
        for logp in (False, True):                                          # warm-up: weights + one captured graph per setting
            m.generate(**batch, return_logprobs=logp, **kw)
        t = {"off": [], "on": []}
        for _ in range(args.reps):
            for name, logp in (("off", False), ("on", True)):
                out, ms = events_ms(lambda: m.generate(**batch, return_logprobs=logp, **kw))
                t[name].append(ms)
                if logp:
                    samples[fmt] = out
        roll[fmt] = {"ms_off": [round(x, 1) for x in t["off"]], "ms_on": [round(x, 1) for x in t["on"]],
                     "median_ms_off": round(median(t["off"]), 1), "median_ms_on": round(median(t["on"]), 1),
                     "overhead_pct": round(100 * (median(t["on"]) / median(t["off"]) - 1), 3)}
        ids_off = m.generate(**batch, **kw).cpu()
        roll[fmt]["ids_equal_with_output"] = bool(torch.equal(ids_off, samples[fmt][0].cpu()))
    res["rollout"] = roll

    # ---- TIS statistics at cap 2: rollout log-probs b against the bf16 policy's training-forward log-probs o
    m.set_fp8_rollout(False)
    dna = {k: v.cuda() for k, v in b["dna_tokenized"].items()}
    stats = {}
    for fmt, (ids_c, b_lp) in samples.items():
        ids = torch.cat([b["input_ids"].cuda(), ids_c], 1)
        with torch.no_grad():
            o = training.policy_forward(m, ids, torch.ones_like(ids), dna, b["batch_idx_map"], C, save=False)[0]
        ones = torch.ones(G, C, device="cuda", dtype=torch.int32)
        _, s, _ = ops.grpo_loss_is_raw(o, None, None, b_lp, torch.zeros(G, device="cuda"), ones, 0.0, 0.2, 0.2, 2.0, want_grad=False)
        s = s.tolist()
        stats[fmt] = {"ratio_mean": round(s[0], 6), "capped_frac": round(s[1], 6), "logp_diff": round(s[2], 6), "kl": round(s[3], 7),
                      "max_abs_logp_diff": round((o - b_lp).abs().max().item(), 5), "mean_rollout_logp": round(b_lp.mean().item(), 4)}
    res["is_stats_cap2"] = stats

    # ---- training_step tokens/s: correction off / on x FP8 rollout off / on
    if not args.no_train:
        def reward(completion_ids, **kw_):
            return (completion_ids % 7 == 0).float().sum(1)
        cfgs = {}
        for fp8 in (False, True):
            for tis in (False, True):
                cfgs[("fp8" if fp8 else "bf16") + ("_is" if tis else "")] = DNALLMGRPOConfig(
                    num_generations=G, max_completion_length=C, per_device_train_batch_size=G, suppress_eos=True, beta=0.04,
                    learning_rate=1e-6, lora_r=32, lora_alpha=64.0, fp8_rollout=fp8, rollout_is_correction=tis, rollout_is_cap=2.0)
        steps = {k: [] for k in cfgs}
        for name, cfg in cfgs.items():
            tr = DNALLMGRPOTrainer(m, [reward], cfg)
            for rep in range(args.reps + 1):                                # first step: warm-up (weights, decode graph)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                tr.training_step(batch)
                torch.cuda.synchronize()
                if rep:
                    steps[name].append(time.perf_counter() - t0)
            if cfg.rollout_is_correction:
                res.setdefault("trainer_is_metrics", {})[name] = {k: round(v, 6) for k, v in tr.log_metrics().items() if k.startswith("rollout_is/")}
            del tr
        res["training_step_s"] = {k: [round(t, 3) for t in v] for k, v in steps.items()}
        res["grpo_tokens_per_s_median"] = {k: round(G * C / median(v), 1) for k, v in steps.items()}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
