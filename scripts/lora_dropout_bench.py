"""Cost of LoRA dropout at config (c) shapes (Qwen3-4B, 36 layers, r = 32; 8 rows x 2364 tokens, micro_rows chosen as the trainer
does): the policy forward + backward with p = 0 and p = 0.05, alternating in one process, and each masked kernel against its unmasked
counterpart (CUDA events).  Prints one JSON object, with the card name and power limit it was measured on.

    python scripts/lora_dropout_bench.py [--reps 3] [--out FILE]
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


def events_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernels(M, d, HqD, F, nqkv, r, reps=20):
    from bioreason_b200 import ops
    from bioreason_b200.engine import LoraDropout
    drop = LoraDropout(seed=7, pass_id=1, threshold=int(round(0.05 * 65536)), row_offset=0)
    bf = torch.bfloat16
    out = {}
    # (name, input width K, output width of the base linear, n_proj, first projection)
    for name, K, N, npj, j0 in (("qkv", d, nqkv, 3, 0), ("o", HqD, d, 1, 3), ("gate_up", d, 2 * F, 2, 4), ("down", F, d, 1, 6)):
        x = torch.randn(M, K, device="cuda").to(bf)
        a = (torch.randn(npj * r, K, device="cuda") * 0.02).to(bf)
        desc = ops.lora_dropout_desc(drop, 0, j0, r)
        plain = events_ms(lambda: ops.gemm(x, a, alpha=2.0), reps)
        masked = events_ms(lambda: ops.lora_down_dropout(x, a, 2.0, desc), reps)
        # dX of this linear: dy [M, N] @ W [N, K] + u [M, npj r] @ A [npj r, K]
        dy = torch.randn(M, N, device="cuda").to(bf)
        wT = (torch.randn(K, N, device="cuda") * 0.02).to(bf)
        u = torch.randn(M, npj * r, device="cuda").to(bf)
        aT = (torch.randn(K, npj * r, device="cuda") * 0.02).to(bf)
        dx_plain = events_ms(lambda: ops.gemm(dy, wT, a2=u, b2=aT), reps)
        dx_masked = events_ms(lambda: ops.gemm(dy, wT, a2=u, b2=aT, dropout=desc), reps)
        # dA of one adapter: u_j^T (x * m_j)
        g = torch.zeros(r, K, device="cuda")
        tn_plain = events_ms(lambda: ops.lora_grad_tn(x, u[:, :r], [(g, 0, K, 0, r)], mode=1), reps)
        tn_masked = events_ms(lambda: ops.lora_grad_tn(x, u[:, :r], [(g, 0, K, 0, r)], mode=1, dropout=desc), reps)
        out[name] = {"down_ms": [plain, masked], "dx_ms": [dx_plain, dx_masked], "dA_ms": [tn_plain, tn_masked],
                     "x_read_GBps_masked_down": M * K * 2 / masked / 1e6}
        del x, a, dy, wT, u, aT, g
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--text", default="qwen3-4b")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from bioreason_b200.build import ensure_built
    ensure_built()
    from bioreason_b200 import training
    from bioreason_b200.configs import dna_config, text_config
    from bioreason_b200.models import DNALLMModel
    from bioreason_b200.synth import synth_batch
    from bioreason_b200.trainer.grpo_trainer import DNALLMGRPOTrainer, _slice_mm
    tc, dc = text_config(args.text), dna_config("nt-v2-500m")
    G, C = 8, 512
    m = DNALLMModel(tc, dc, seed=1234)
    m.enable_lora(r=32, alpha=64.0, seed=3)
    with torch.no_grad():
        for p in m._lora.params[1::2]:
            p.normal_(0, 0.01)
    m.sync_adapters(rollout=False)
    b = synth_batch(tc, dc, batch=G, n_seq=2, dna_len=668, text_len=512, seed=8, same_prompt=True)
    comp = torch.randint(0, tc.eos_token_id, (G, C), generator=torch.Generator().manual_seed(9))
    ids = torch.cat([b["input_ids"], comp], 1).cuda()
    mask = torch.ones_like(ids)
    L = ids.shape[1]
    mm = dict(dna_tokenized={k: v.cuda() for k, v in b["dna_tokenized"].items()}, batch_idx_map=b["batch_idx_map"])
    wgt = torch.randn(G, C, device="cuda")
    mr = DNALLMGRPOTrainer._auto_micro_rows(m, G, L)

    def step(p):
        m.set_lora_dropout(p, seed=11)
        pid = m.new_lora_dropout_pass()
        m.zero_grad_buffers()
        for lo in range(0, G, mr):
            hi = min(G, lo + mr)
            mc = _slice_mm(mm, lo, hi)
            kw = dict(dropout=True, dropout_pass=pid, row_offset=lo) if pid is not None else {}
            lp, ctx = training.policy_forward(m, ids[lo:hi], mask[lo:hi], mc["dna_tokenized"], mc["batch_idx_map"], C, **kw)
            training.policy_backward(m, ctx, wgt[lo:hi])
            del ctx

    times = {0.0: [], 0.05: []}
    for p in (0.0, 0.05):                                                   # warm-up of both paths
        step(p)
    torch.cuda.synchronize()
    for _ in range(args.reps):
        for p in (0.0, 0.05):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            step(p)
            torch.cuda.synchronize()
            times[p].append(time.perf_counter() - t0)
    med = {p: sorted(v)[len(v) // 2] for p, v in times.items()}
    res = {"card": card(), "rows": G, "L": L, "layers": tc.num_hidden_layers, "micro_rows": mr, "r": 32,
           "policy_fwd_bwd_s": {"p0": times[0.0], "p0.05": times[0.05]}, "ratio_median": med[0.05] / med[0.0]}
    del m
    torch.cuda.empty_cache()
    Hq, Hkv, D = tc.num_attention_heads, tc.num_key_value_heads, tc.head_dim
    res["kernels_ms_plain_vs_masked"] = kernels(mr * L, tc.hidden_size, Hq * D, tc.intermediate_size, (Hq + 2 * Hkv) * D, 32)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
