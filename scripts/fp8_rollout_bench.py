"""bf16 versus weight-only FP8 (e4m3) rollout decode at config (c) (Qwen3-4B, 36 layers, random init, LoRA r = 32, 1 prompt x G = 8,
P = 1852, C = 512, EOS suppressed).  The two formats alternate in one process after a warm-up; GPU times are CUDA events.  Measures the
four layer linears (time and GB/s; bytes = weight codes + scales + activations), the rollout, the peak allocation of each rollout,
the first step where the FP8 and bf16 rollouts diverge under the same uniforms, the mean per-token log-prob the bf16 policy assigns to
FP8- and bf16-sampled completions, and training_step tokens/s with share_prompt_prefix off and on.  Prints one JSON object with the
card name and power limit it was measured on.

    python scripts/fp8_rollout_bench.py [--reps 2] [--out FILE]
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
    from bioreason_b200 import ops, training
    from bioreason_b200.configs import dna_config, text_config
    from bioreason_b200.lora import build_rollout_weights, build_rollout_weights_fp8
    from bioreason_b200.models import DNALLMModel
    from bioreason_b200.synth import synth_batch
    from bioreason_b200.trainer import DNALLMGRPOConfig
    from bioreason_b200.trainer.grpo_trainer import DNALLMGRPOTrainer
    tc, dc = text_config(args.text), dna_config("nt-v2-500m")
    G, C = 8, args.completion
    m = DNALLMModel(tc, dc, seed=1234)
    m.enable_lora(r=32, alpha=64.0, seed=3)
    with torch.no_grad():
        for p in m._lora.params[1::2]:
            p.normal_(0, 0.01)
    m.sync_adapters(rollout=False)
    b = synth_batch(tc, dc, batch=G, n_seq=2, dna_len=668, text_len=512, seed=8, same_prompt=True)
    res = {"card": card(), "model": args.text, "layers": tc.num_hidden_layers, "rows": G, "C": C, "P": b["input_ids"].shape[1]}

    # ---- the four layer linears, R = 8, layer 0 of the merged + folded weights
    wb = build_rollout_weights(m._dec, m._lora)
    wf = build_rollout_weights_fp8(m._dec, m._lora)
    scratch = ops.skinny_scratch(max(tc.vocab_size, 2 * tc.intermediate_size), "cuda")
    R, d, F = G, tc.hidden_size, tc.intermediate_size
    HqD = tc.num_attention_heads * tc.head_dim
    x = {n: torch.randn(R, k, device="cuda").bfloat16() for n, k in (("w_qkv", d), ("w_o", HqD), ("w_gu", d), ("w_down", F))}
    mode = {"w_qkv": 0, "w_o": 1, "w_gu": 2, "w_down": 1}
    resid = torch.randn(R, d, device="cuda").bfloat16()
    gemm = {}
    for name in ("w_qkv", "w_o", "w_gu", "w_down"):
        row = {}
        for fmt, W in (("bf16", wb), ("fp8", wf)):
            w = getattr(W.layers[0], name)
            N, K = w.shape
            fn = lambda: ops.skinny_gemm(x[name], w, scratch, mode=mode[name], residual=resid if mode[name] == 1 else None)
            events_ms(fn, 20)
            t = min(events_ms(fn, 200)[1] for _ in range(args.reps))
            wbytes = N * K * (1 if fmt == "fp8" else 2) + (4 * N if fmt == "fp8" else 0)
            abytes = 2 * R * K + 2 * R * (N // 2 if mode[name] == 2 else N) + (2 * R * N if mode[name] == 1 else 0)
            row[fmt] = {"us": round(t * 1e3, 2), "GB_per_s": round((wbytes + abytes) / (t * 1e-3) / 1e9, 1), "MB": round((wbytes + abytes) / 1e6, 2)}
        row["speedup"] = round(row["bf16"]["us"] / row["fp8"]["us"], 3)
        gemm[name] = row
    res["layer_gemm_R8"] = gemm
    res["rollout_weight_bytes_GB"] = {
        "bf16": round(sum(getattr(L, n).numel() * 2 for L in wb.layers for n in mode) / 1e9, 3),
        "fp8": round(sum(getattr(L, n).q.numel() + getattr(L, n).scale.numel() * 4 for L in wf.layers for n in mode) / 1e9, 3)}
    del wb, wf
    torch.cuda.empty_cache()

    # ---- rollout, alternating formats
    batch = dict(input_ids=b["input_ids"], attention_mask=b["attention_mask"], dna_tokenized=b["dna_tokenized"], batch_idx_map=b["batch_idx_map"])
    u = torch.rand(C, G, generator=torch.Generator().manual_seed(5))
    kw = dict(max_new_tokens=C, do_sample=True, temperature=1.0, top_k=50, top_p=1.0, uniforms=u, eos_token_id=-1, pad_token_id=0)

    def rollout(fp8):
        m.set_fp8_rollout(fp8)
        m._rollout_dec = None
        m._rollout._cached.clear() if getattr(m, "_rollout", None) is not None else None
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        m.generate(**batch, **kw)                                           # builds the weights and captures the decode graph
        torch.cuda.synchronize()
        build_peak = torch.cuda.max_memory_allocated() - base
        times = []
        for _ in range(args.reps):
            out, t = events_ms(lambda: m.generate(**batch, **kw))
            times.append(t)
        return out.cpu(), times, build_peak
    roll = {}
    for fp8 in (False, True, False, True):
        out, times, peak = rollout(fp8)
        r = roll.setdefault("fp8" if fp8 else "bf16", {"ms": [], "peak_over_base_GB": 0.0})
        r["ms"] += [round(t, 1) for t in times]
        r["peak_over_base_GB"] = round(peak / 1e9, 3)
        r["tokens"] = out
    for r in roll.values():
        r["median_ms"] = sorted(r["ms"])[len(r["ms"]) // 2]
        r["decode_step_ms"] = round(r["median_ms"] / C, 3)
    res["rollout_speedup"] = round(roll["bf16"]["median_ms"] / roll["fp8"]["median_ms"], 3)

    # ---- accuracy on the random-init model: divergence and the bf16 policy's log-probs of both samples
    tb, tf = roll["bf16"].pop("tokens"), roll["fp8"].pop("tokens")
    diff = (tb != tf)
    first = [int(r.nonzero()[0]) if r.any() else C for r in diff]
    m.set_fp8_rollout(False)
    mm = dict(dna_tokenized={k: v.cuda() for k, v in b["dna_tokenized"].items()}, batch_idx_map=b["batch_idx_map"])
    lp = {}
    for name, comp in (("bf16_sampled", tb), ("fp8_sampled", tf)):
        ids = torch.cat([b["input_ids"], comp], 1).cuda()
        with torch.no_grad():
            l = training.policy_forward(m, ids, torch.ones_like(ids), mm["dna_tokenized"], mm["batch_idx_map"], C, save=False)[0]
        lp[name] = round(l.float().mean().item(), 4)
    res["rollout"] = roll
    res["first_divergence_step"] = first
    res["mean_logp_under_bf16_policy"] = lp

    # ---- training_step tokens/s: bf16 / fp8 rollout x share_prompt_prefix off / on
    if not args.no_train:
        def reward(completion_ids, **kw_):
            return (completion_ids % 7 == 0).float().sum(1)
        trainers = {}
        for fp8 in (False, True):
            for share in (False, True):
                cfg = DNALLMGRPOConfig(num_generations=G, max_completion_length=C, per_device_train_batch_size=G, suppress_eos=True, beta=0.04,
                                       learning_rate=1e-6, lora_r=32, lora_alpha=64.0, share_prompt_prefix=share, fp8_rollout=fp8)
                trainers[("fp8" if fp8 else "bf16") + ("_shared" if share else "_dense")] = cfg
        steps = {k: [] for k in trainers}
        for name, cfg in trainers.items():
            tr = DNALLMGRPOTrainer(m, [reward], cfg)                        # sets the rollout format on the model
            for rep in range(args.reps + 1):                                # first step: warm-up (weights, decode graph)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                tr.training_step(batch)
                torch.cuda.synchronize()
                if rep:
                    steps[name].append(time.perf_counter() - t0)
            del tr
        res["training_step_s"] = {k: [round(t, 3) for t in v] for k, v in steps.items()}
        res["grpo_tokens_per_s_median"] = {k: round(G * C / sorted(v)[len(v) // 2], 1) for k, v in steps.items()}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
