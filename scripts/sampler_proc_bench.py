"""Cost of the logits processors of the fused sampler (repetition penalty, min-p, min_new_tokens).  Settings alternate in one process after
a warm-up; GPU times are CUDA events.  Measures:
  - the sampler alone, V = 151 936, R in {8, 32}, two-stage (top_k = 20) and single-stage (top_k = 64), without and with the log-prob
    output: processors off (the plain entry points), theta = 1.1 only, theta = 1.1 + min_p = 0.05 + min_new_tokens = 4;
  - the config (c) rollout (Qwen3-4B, 36 layers, random init, 1 prompt x G = 8, C = 512, EOS suppressed, T = 0.6 / top_k = 20 /
    top_p = 0.95) with theta = 1 against theta = 1.1, medians of --reps.
Prints one JSON object with the card name and power limit it was measured on.

    python scripts/sampler_proc_bench.py [--reps 3] [--out FILE]
"""
import argparse, json, os, subprocess, sys
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
    ap.add_argument("--no-rollout", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    from bioreason_b200.build import ensure_built
    ensure_built()
    from bioreason_b200 import ops
    from bioreason_b200.configs import dna_config, text_config
    tc, dc = text_config(args.text), dna_config("nt-v2-500m")
    V = tc.vocab_size
    res = {"card": card(), "model": args.text, "V": V}

    # ---- the sampler alone
    settings = {"off": dict(), "theta": dict(repetition_penalty=1.1),
                "theta_minp_minnew": dict(repetition_penalty=1.1, min_p=0.05, min_new_tokens=4)}
    samp = {}
    for R in (8, 32):
        logits = torch.randn(R, V, device="cuda") * 3
        ws = ops.sample_workspace(R, V, "cuda", logp=True)
        tok = torch.zeros(R, 1, device="cuda", dtype=torch.int64)
        lpb = torch.zeros(R, 1, device="cuda")
        uu = torch.rand(1, R, device="cuda")
        step = torch.zeros(1, device="cuda", dtype=torch.int32)
        pres = ops.presence_bitmap(R, V, "cuda")
        pres.view(torch.uint8)[:, ::7] = 0x11                              # some emitted tokens in every row
        for path, k in (("two_stage", 20), ("single_stage", 64)):
            for lp_name, lp in (("no_logp", None), ("logp", lpb)):
                fns = {}
                for name, kw in settings.items():
                    extra = dict(kw, presence=pres) if kw else {}
                    fns[name] = (lambda extra=extra, lp=lp, k=k: ops.sample_next(
                        logits, workspace=ws, temperature=0.6, top_k=k, top_p=0.95, do_sample=True, uniforms=uu, step=step, max_steps=1,
                        tokens=tok, logp=lp, **extra))
                for f in fns.values():
                    events_ms(f, 50)
                t = {n: [] for n in fns}
                for _ in range(args.reps):
                    for n, f in fns.items():
                        t[n].append(events_ms(f, 500)[1] * 1e3)
                samp[f"R{R}_{path}_{lp_name}"] = {n: round(median(v), 2) for n, v in t.items()}
    res["sampler_us"] = samp

    # ---- config (c) rollout, theta = 1 against theta = 1.1
    if not args.no_rollout:
        from bioreason_b200.models import DNALLMModel
        from bioreason_b200.synth import synth_batch
        G, C = 8, args.completion
        m = DNALLMModel(tc, dc, seed=1234)
        b = synth_batch(tc, dc, batch=G, n_seq=2, dna_len=668, text_len=512, seed=8, same_prompt=True)
        batch = dict(input_ids=b["input_ids"], attention_mask=b["attention_mask"], dna_tokenized=b["dna_tokenized"],
                     batch_idx_map=b["batch_idx_map"])
        u = torch.rand(C, G, generator=torch.Generator().manual_seed(5))
        kw = dict(max_new_tokens=C, do_sample=True, temperature=0.6, top_k=20, top_p=0.95, uniforms=u, eos_token_id=-1, pad_token_id=0)
        for th in (1.0, 1.1):
            m.generate(**batch, repetition_penalty=th, **kw)                 # warm-up: one captured graph per setting
        t = {1.0: [], 1.1: []}
        for _ in range(args.reps):
            for th in t:
                t[th].append(events_ms(lambda: m.generate(**batch, repetition_penalty=th, **kw))[1])
        res["rollout"] = {"P": b["input_ids"].shape[1], "rows": G, "C": C, "layers": tc.num_hidden_layers,
                          "ms_theta1": [round(x, 1) for x in t[1.0]], "ms_theta1.1": [round(x, 1) for x in t[1.1]],
                          "median_ms_theta1": round(median(t[1.0]), 1), "median_ms_theta1.1": round(median(t[1.1]), 1),
                          "per_step_extra_us": round((median(t[1.1]) - median(t[1.0])) / C * 1e3, 2)}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
