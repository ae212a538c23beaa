"""Time the full-vocabulary sampler (ops.sample_next_full) against the two-stage top_k = 20 call, with CUDA events.  Settings alternate
in one process after a warm-up; each figure is the median over rounds of the mean over `--iters` back-to-back calls.  Prints the card
name and power limit of the same run, then one JSON line per setting.

  python scripts/sampler_full_bench.py [--rounds 15] [--iters 50]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:                                             # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    from bioreason_b200.build import ensure_built
    ensure_built()
    from bioreason_b200 import ops
    print("card:", card(), flush=True)
    V = 151936
    cases = []
    for R in (8, 32):
        for fam, scale in (("randn3", 3.0), ("flat", 0.05)):
            z = torch.randn(R, V, device="cuda", generator=torch.Generator("cuda").manual_seed(R)) * scale
            U = torch.rand(1, R, device="cuda")
            step = torch.zeros(1, device="cuda", dtype=torch.int32)
            tok = torch.zeros(R, 1, device="cuda", dtype=torch.int64)
            wsf = ops.sample_full_workspace(R, V, "cuda")
            ws2 = ops.sample_workspace(R, V, "cuda")
            for T, k, p in ((1.0, 0, 1.0), (1.0, 0, 0.95), (0.6, 0, 0.95)):
                cases.append((f"full R={R} {fam} T={T} top_k={k} top_p={p}",
                              lambda z=z, U=U, step=step, tok=tok, ws=wsf, T=T, k=k, p=p: ops.sample_next_full(
                                  z, workspace=ws, temperature=T, top_k=k, top_p=p, uniforms=U, step=step, tokens=tok)))
            cases.append((f"two-stage R={R} {fam} T=1.0 top_k=20 top_p=1.0",
                          lambda z=z, U=U, step=step, tok=tok, ws=ws2: ops.sample_next(
                              z, workspace=ws, temperature=1.0, top_k=20, top_p=1.0, uniforms=U, step=step, tokens=tok)))
    for _, f in cases:                                                 # warm-up
        for _ in range(5):
            f()
    torch.cuda.synchronize()
    times = {name: [] for name, _ in cases}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for name, f in cases:
            ev0.record()
            for _ in range(args.iters):
                f()
            ev1.record()
            ev1.synchronize()
            times[name].append(ev0.elapsed_time(ev1) * 1000.0 / args.iters)
    for name, _ in cases:
        print(json.dumps({"case": name, "median_us": round(statistics.median(times[name]), 2),
                          "min_us": round(min(times[name]), 2), "max_us": round(max(times[name]), 2)}), flush=True)


if __name__ == "__main__":
    main()
