"""The linear layers of config (c) (Qwen3-4B widths) through br_gemm_bf16, timed with CUDA events after a warm-up: qkv, o, gate/up
and down as the forward runs them (o and down add the residual, gate/up writes the gated SiLU and its pre-activation copy), and the
backward's dX products with the transposed weights, plus the fused lm_head log-prob over 2048 completion rows.  Prints one JSON
object with TFLOP/s per shape from 2*M*N*K, and the card name and power limit it was measured on.

    python scripts/gemm_bench.py [--rows 9456 6368] [--iters 20] [--reps 5] [--lib PATH] [--out FILE]

--rows: token rows per call (9456 = the trainer's 4-row dense chunk at L = 2364, 6368 = the shared-prefix buffer).
--lib: time another build of libbioreason_b200.so (for instance the previous commit's) with the same script.
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


def shapes(tc):
    d, F = tc.hidden_size, tc.intermediate_size
    q, kv = tc.num_attention_heads * tc.head_dim, tc.num_key_value_heads * tc.head_dim
    # (name, N, K, epilogue)
    return [("qkv", q + 2 * kv, d, "plain"), ("o", d, q, "residual"), ("gate_up", 2 * F, d, "silu"), ("down", d, F, "residual"),
            ("qkv_dX", d, q + 2 * kv, "plain"), ("o_dX", q, d, "plain"), ("gate_up_dX", d, 2 * F, "plain"), ("down_dX", F, d, "plain")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[9456, 6368])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--text", default="qwen3-4b")
    ap.add_argument("--lib", default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "gemm_bench times the GPU kernels; it needs a CUDA device"
    from bioreason_b200 import _lib
    if args.lib:
        _lib._lib = _lib.ffi.dlopen(os.path.abspath(args.lib))
    else:
        from bioreason_b200.build import ensure_built
        ensure_built()
    from bioreason_b200 import ops
    from bioreason_b200.configs import text_config
    tc = text_config(args.text)
    g = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *s: (torch.randn(*s, device="cuda", generator=g) * 0.05).bfloat16()

    def time_ms(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        best = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            best.append(e0.elapsed_time(e1) / args.iters)
        best.sort()
        return best[len(best) // 2], best[0], best[-1]

    result = {"card": card(), "lib": args.lib or "tree", "iters": args.iters, "reps": args.reps, "shapes": []}
    for M in args.rows:
        for name, N, K, epi in shapes(tc):
            a, w = rnd(M, K), rnd(N, K)
            kw = {}
            if epi == "residual":
                kw["residual"] = rnd(M, N)
            elif epi == "silu":
                kw.update(act=1, aux_out=torch.empty(M, N, device="cuda", dtype=torch.bfloat16))
            out = torch.empty(M, N // 2 if epi == "silu" else N, device="cuda", dtype=torch.bfloat16)
            med, lo, hi = time_ms(lambda: ops.gemm(a, w, out=out, **kw))
            flop = 2.0 * M * N * K
            result["shapes"].append({"name": name, "M": M, "N": N, "K": K, "epilogue": epi, "ms": round(med, 4), "ms_min": round(lo, 4),
                                     "ms_max": round(hi, 4), "tflops": round(flop / med / 1e9, 1)})
            del a, w, kw, out
    M, V, K = 2048, tc.vocab_size, tc.hidden_size
    h, w = rnd(M, K), rnd(V, K)
    tgt = torch.randint(0, V, (M,), device="cuda", generator=g)
    med, lo, hi = time_ms(lambda: ops.lmhead_logprob(h, w, tgt))
    result["shapes"].append({"name": "lm_head_logprob", "M": M, "N": V, "K": K, "epilogue": "lse", "ms": round(med, 4), "ms_min": round(lo, 4),
                             "ms_max": round(hi, 4), "tflops": round(2.0 * M * V * K / med / 1e9, 1)})
    for s in result["shapes"]:
        print("%-16s M=%-5d N=%-6d K=%-5d %8.3f ms  %6.1f TFLOP/s" % (s["name"], s["M"], s["N"], s["K"], s["ms"], s["tflops"]), file=sys.stderr)
    line = json.dumps(result)
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
