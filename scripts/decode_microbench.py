"""Per-kernel timing of one decode step's launches at config (c) shapes, each captured in a CUDA graph (no host launch
overhead) and timed with CUDA events.  Prints us/launch and achieved GB/s for the weight-streaming GEMMs."""
import math, sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from bioreason_b200 import ops
from bioreason_b200.configs import text_config

torch.manual_seed(0)
tc = text_config(sys.argv[1] if len(sys.argv) > 1 else "qwen3-4b")
d, F, V = tc.hidden_size, tc.intermediate_size, tc.vocab_size
Hq, Hkv, D = tc.num_attention_heads, tc.num_key_value_heads, tc.head_dim
R, G, P, gen = 8, 8, 1848, 256
dev = "cuda"
NL = 6                                   # distinct weight sets so every launch streams from HBM, not L2
bf = torch.bfloat16


def timed_graph(fn, reps=20, inner=1):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(inner):
            fn()
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (reps * inner)


scratch = ops.skinny_scratch(max(V, 2 * F), dev)
res = {}
shapes = {"qkv": ((Hq + 2 * Hkv) * D, d, 0), "o": (d, Hq * D, 1), "gate_up": (2 * F, d, 2), "down": (d, F, 1), "lm_head": (V, d, 3)}
for name, (N, K, mode) in shapes.items():
    n_sets = NL if name != "lm_head" else 2
    ws = [torch.randn(N, K, device=dev).to(bf) * 0.02 for _ in range(n_sets)]
    x = torch.randn(R, K, device=dev).to(bf)
    r = torch.randn(R, N, device=dev).to(bf)
    ssq = torch.ones(32, device=dev)
    def fn():
        for w in ws:
            ops.skinny_gemm(x, w, scratch, mode=mode, residual=r if mode == 1 else None, sumsq_in=ssq if mode in (0, 2, 3) else None, eps=1e-6)
    us = timed_graph(fn) / n_sets
    gbs = N * K * 2 / (us * 1e-6) / 1e9
    res[name] = (us, gbs)
    print(f"skinny {name:8s} N={N:6d} K={K:5d}: {us:8.2f} us  {gbs:7.1f} GB/s")
    del ws

# fused attention at ctx = P + gen
PAGE = 64
T = P + gen
n_shared = P // PAGE
priv = math.ceil((T + 1 - n_shared * PAGE) / PAGE)
max_pages = n_shared + priv
n_pages = n_shared + R * priv
table = torch.zeros(R, max_pages, dtype=torch.int32)
nxt = n_shared
for r_ in range(R):
    table[r_, :n_shared] = torch.arange(n_shared, dtype=torch.int32)
    table[r_, n_shared:] = torch.arange(nxt, nxt + priv, dtype=torch.int32); nxt += priv
table = table.to(dev)
kc = torch.randn(n_pages, Hkv, PAGE, D, device=dev).to(bf); vc = torch.randn_like(kc)
qkv = torch.randn(R, (Hq + 2 * Hkv) * D, device=dev).to(bf)
qn = torch.ones(D, device=dev).to(bf); kn = torch.ones(D, device=dev).to(bf)
cur = torch.full((R,), T, dtype=torch.int32, device=dev)
rope = ops.rope_table(T + 8, D, 1e6, dev)
for ss, sp in ((8, 2), (14, 3), (16, 2), (28, 2), (4, 1)):       # <= 3 work items per SM on a 132-SM H100
    wsf = ops.decode_fused_workspace(R, Hq, Hkv, D, ss + sp, dev)
    out = torch.empty(R, Hq * D, device=dev, dtype=bf)
    us = timed_graph(lambda: ops.decode_attn_fused(qkv, qn, kn, kc, vc, table, cur, G, Hq, Hkv, D, n_shared, ss, sp, 1e6, 1e-6, wsf, out, rope=rope), inner=4)
    print(f"decode_attn_fused ctx={T} splits=({ss},{sp}): {us:8.2f} us")
    res[f"attn_fused_{ss}_{sp}"] = (us, 0)

# sampler
logits = torch.randn(R, V, device=dev)
tokens = torch.zeros(R, 4, dtype=torch.int64, device=dev); nx = torch.zeros(R, dtype=torch.int64, device=dev)
fin = torch.zeros(R, dtype=torch.int32, device=dev); step = torch.zeros(1, dtype=torch.int32, device=dev); uni = torch.rand(4, R, device=dev)
us = timed_graph(lambda: ops.sample_next(logits, temperature=0.6, top_k=20, top_p=0.95, do_sample=True, uniforms=uni, step=step, max_steps=4,
                                          finished=fin, tokens=tokens, next_ids=nx), inner=2)
print(f"sampler 1-stage: {us:8.2f} us")
if hasattr(ops, "sample_workspace"):
    sw = ops.sample_workspace(R, V, dev)
    us = timed_graph(lambda: ops.sample_next(logits, temperature=0.6, top_k=20, top_p=0.95, do_sample=True, uniforms=uni, step=step, max_steps=4,
                                              finished=fin, tokens=tokens, next_ids=nx, workspace=sw), inner=2)
    print(f"sampler 2-stage: {us:8.2f} us")
emb = torch.randn(V, d, device=dev).to(bf); h = torch.empty(R, d, device=dev, dtype=bf); ssq = torch.zeros(32, device=dev)
us = timed_graph(lambda: ops.embed_gather_sumsq(nx, emb, h, ssq), inner=4)
print(f"embed_gather_sumsq: {us:8.2f} us")
us = timed_graph(lambda: ops.decode_advance(step, cur), inner=4)
print(f"decode_advance: {us:8.2f} us")
tot = 36 * (res["qkv"][0] + res["o"][0] + res["gate_up"][0] + res["down"][0] + res["attn_fused_8_2"][0]) + res["lm_head"][0]
print(f"estimated token step (36 layers): {tot / 1e3:.3f} ms")

# ---- a real layer chain (qkv -> fused attention -> o -> gate/up -> down) x NL in one graph: what a token step actually costs
ws_l = [dict(qkv=torch.randn((Hq + 2 * Hkv) * D, d, device=dev).to(bf) * 0.02, o=torch.randn(d, Hq * D, device=dev).to(bf) * 0.02,
             gu=torch.randn(2 * F, d, device=dev).to(bf) * 0.02, down=torch.randn(d, F, device=dev).to(bf) * 0.02) for _ in range(NL)]
x0 = torch.randn(R, d, device=dev).to(bf)
cur.fill_(T); step.zero_()          # decode_advance above moved them
n_part = ((d + 127) // 128) * 4
ssa = torch.ones(n_part, 32, device=dev); ssb = torch.ones(n_part, 32, device=dev)
attn_out = torch.empty(R, Hq * D, device=dev, dtype=bf)
SS_, SP_ = 8, 2
wsf = ops.decode_fused_workspace(R, Hq, Hkv, D, SS_ + SP_, dev)
def chain():
    x = x0
    for w in ws_l:
        q = ops.skinny_gemm(x, w["qkv"], scratch, sumsq_in=ssa, sumsq_in_n=n_part, eps=1e-6)
        ops.decode_attn_fused(q, qn, kn, kc, vc, table, cur, G, Hq, Hkv, D, n_shared, SS_, SP_, 1e6, 1e-6, wsf, attn_out, rope=rope)
        x2 = ops.skinny_gemm(attn_out, w["o"], scratch, mode=1, residual=x, sumsq_out=ssb)
        a = ops.skinny_gemm(x2, w["gu"], scratch, mode=2, sumsq_in=ssb, sumsq_in_n=n_part, eps=1e-6)
        x = ops.skinny_gemm(a, w["down"], scratch, mode=1, residual=x2, sumsq_out=ssa)
us = timed_graph(chain) / NL
print(f"layer chain (5 launches, splits {SS_},{SP_}): {us:8.2f} us per layer  -> {36 * us / 1e3:.3f} ms per token (36 layers)   PDL={'off' if os.environ.get('BR_NO_PDL') else 'on'}")
