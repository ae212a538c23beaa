"""What bounds the 5-launch decode layer chain?  Times variants of the chain (CUDA graph, PDL on) at config (c) shapes, R = 8:
  full      qkv -> fused attention -> o -> gate/up -> down           (the production layer)
  gemms     qkv -> o -> gate/up -> down                              (no attention)
  no_o      qkv -> attention -> gate/up -> down
  attn_x2   qkv -> attention -> attention -> o -> gate/up -> down
and prints each variant's time next to the sum of the isolated (same kernel back to back) launch times."""
import math, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from bioreason_b200 import ops
dev, bf = "cuda", torch.bfloat16
d, F, Hq, Hkv, D, R, G, P, gen = 2560, 9728, 32, 8, 128, 8, 8, 1848, 256
NL = 6
mk = lambda *s: (torch.randn(*s, device=dev) * 0.02).to(bf)
ws = [dict(qkv=mk((Hq + 2 * Hkv) * D, d), o=mk(d, Hq * D), gu=mk(2 * F, d), down=mk(d, F)) for _ in range(NL)]
scratch = ops.skinny_scratch(2 * F, dev)
PAGE = 64; T = P + gen; n_shared = P // PAGE; priv = math.ceil((T + 1 - n_shared * PAGE) / PAGE); max_pages = n_shared + priv
table = torch.zeros(R, max_pages, dtype=torch.int32); nxt = n_shared
for r in range(R):
    table[r, :n_shared] = torch.arange(n_shared, dtype=torch.int32); table[r, n_shared:] = torch.arange(nxt, nxt + priv, dtype=torch.int32); nxt += priv
table = table.to(dev)
kc = torch.randn(nxt, Hkv, PAGE, D, device=dev).to(bf); vc = torch.randn_like(kc)
qn = torch.ones(D, device=dev).to(bf); kn = torch.ones(D, device=dev).to(bf)
cur = torch.full((R,), T, dtype=torch.int32, device=dev)
rope = ops.rope_table(T + 8, D, 1e6, dev)
n_part = (d // 128) * 4
ssa = torch.ones(n_part, 32, device=dev); ssb = torch.ones(n_part, 32, device=dev)
SS, SP = 14, 3
wsf = ops.decode_fused_workspace(R, Hq, Hkv, D, SS + SP, dev)
attn_out = mk(R, Hq * D); x0 = mk(R, d); q0 = mk(R, (Hq + 2 * Hkv) * D); x2_0 = mk(R, d); a0 = mk(R, F)


def timed(fn, reps=30):
    fn(); torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (reps * NL)


def k_qkv(w, x): return ops.skinny_gemm(x, w["qkv"], scratch, sumsq_in=ssa, sumsq_in_n=n_part, eps=1e-6)
def k_attn(q): ops.decode_attn_fused(q, qn, kn, kc, vc, table, cur, G, Hq, Hkv, D, n_shared, SS, SP, 1e6, 1e-6, wsf, attn_out, rope=rope)
def k_o(w, x): return ops.skinny_gemm(attn_out, w["o"], scratch, mode=1, residual=x, sumsq_out=ssb)
def k_gu(w, x2): return ops.skinny_gemm(x2, w["gu"], scratch, mode=2, sumsq_in=ssb, sumsq_in_n=n_part, eps=1e-6)
def k_down(w, a, x2): return ops.skinny_gemm(a, w["down"], scratch, mode=1, residual=x2, sumsq_out=ssa)


def variant(name):
    def fn():
        x = x0
        for w in ws:
            q = k_qkv(w, x) if "qkv" in name else q0
            for _ in range(name.count("A")):
                k_attn(q)
            x2 = k_o(w, x) if "o" in name.split("-") else x2_0
            a = k_gu(w, x2) if "gu" in name else a0
            x = k_down(w, a, x2) if "down" in name else x
    return fn


iso = {}
for nm in ("qkv", "A", "o", "gu", "down"):
    iso[nm] = timed(variant(nm))
    print(f"isolated {nm:5s}: {iso[nm]:7.2f} us per launch")
for nm in ("qkv-A-o-gu-down", "qkv-o-gu-down", "qkv-A-gu-down", "qkv-A-A-o-gu-down", "o-gu-down", "gu-down", "qkv-A", "A-o", "o-gu", "qkv-o", "down-qkv"):
    t = timed(variant(nm))
    parts = [p_ for p_ in nm.split("-")]
    s = sum(iso[p_] for p_ in parts)
    print(f"chain {nm:20s}: {t:7.2f} us per layer   sum of isolated {s:7.2f}   diff {t - s:+6.2f}")

# ---- L2 staging from the fused attention ONLY (HBM is idle for the ~13 us it runs): units [6, 6 + m) of every gate/up chunk
print(f"gate/up chunk = {ops.skinny_chunk_units(ws[0]['gu'])} units of 16 KB per CTA, down {ops.skinny_chunk_units(ws[0]['down'])}, o {ops.skinny_chunk_units(ws[0]['o'])}")
for who, m in (("none", 0), ("attn->gu", 8), ("attn->gu", 16), ("attn->gu", 24), ("attn->gu", 39), ("attn->o", 3), ("attn->down", 15), ("qkv->gu", 16)):
    def fn():
        x = x0
        for w in ws:
            q = ops.skinny_gemm(x, w["qkv"], scratch, sumsq_in=ssa, sumsq_in_n=n_part, eps=1e-6, prefetch=(w["gu"], 6, 6 + m) if who == "qkv->gu" else None)
            tgt = {"attn->gu": "gu", "attn->o": "o", "attn->down": "down"}.get(who)
            ops.decode_attn_fused(q, qn, kn, kc, vc, table, cur, G, Hq, Hkv, D, n_shared, SS, SP, 1e6, 1e-6, wsf, attn_out, rope=rope,
                                  prefetch=(w[tgt], 6, 6 + m) if tgt and m > 0 else None)
            x2 = k_o(w, x); a = k_gu(w, x2); x = k_down(w, a, x2)
    print(f"staging {who:10s} m={m:2d}: {timed(fn):7.2f} us per layer")

# ---- stream gate (br_stream_gate): early weight loads start when the previous GEMM's weights are on chip
cnt = torch.zeros(1, device=dev, dtype=torch.int32); ep = torch.ones(1, device=dev, dtype=torch.int32)
grids = {k: ops.skinny_grid(ws[0][k]) for k in ("qkv", "o", "gu", "down")}
per_layer = sum(grids.values())
for mode in ("off", "on"):
    def fn():
        cnt.zero_()
        x = x0
        acc = 0
        def g(name, wait):
            nonlocal acc
            spec = None if mode == "off" else dict(counter=cnt, epoch=ep, epoch_base=1, per_step=NL * per_layer, wait=(acc if wait else None), signal=True)
            acc += grids[name]
            return spec
        for li, w in enumerate(ws):
            q = ops.skinny_gemm(x, w["qkv"], scratch, sumsq_in=ssa, sumsq_in_n=n_part, eps=1e-6, gate=g("qkv", li > 0))
            k_attn(q)
            x2 = ops.skinny_gemm(attn_out, w["o"], scratch, mode=1, residual=x, sumsq_out=ssb, gate=g("o", False))
            a = ops.skinny_gemm(x2, w["gu"], scratch, mode=2, sumsq_in=ssb, sumsq_in_n=n_part, eps=1e-6, gate=g("gu", True))
            x = ops.skinny_gemm(a, w["down"], scratch, mode=1, residual=x2, sumsq_out=ssa, gate=g("down", True))
    print(f"stream gate {mode:3s}: {timed(fn):7.2f} us per layer")
