"""The training-pass GEMMs against float64 references with per-element error bounds (tests/gemm_ref.py has the error model): the
wgmma GEMM and its epilogues at both tile widths, the fused lm-head (log-prob, lse and every element of the softmax gradient) at the
Qwen3 vocabulary, and the LoRA-gradient GEMM at the trainer's Qwen3-4B calls and its split-K edges.  Outputs are NaN-prefilled and
strided with sentinel columns, so a tile that is never stored or a store past the row shows up; the LoRA-gradient destinations hold
data and sit inside larger buffers whose other rows and columns must keep their bits.  Each case asserts the tile width it runs on
(the rule of test_gpu_gemm_wide._is_wide).  Run with -s to see the worst err / bound ratio of every output."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gemm_ref as gr  # noqa: E402
from lora_dropout_ref import threshold  # noqa: E402
from test_gpu_gemm_wide import _is_wide  # noqa: E402
from test_gpu_train_kernels_fp64 import PAD, _bits, _check, _nan_buffer  # noqa: E402

pytestmark = pytest.mark.gpu

ROWS = 1024                     # float64 reference row block of the GEMM checks
LM_ROWS = 64                    # ... of the lm-head checks ([64, V] float64 buffers)
T_DROP = threshold(0.05)
INV_KEEP = 65536.0 / (65536 - T_DROP)


@pytest.fixture(scope="module")
def ops():
    from bioreason_b200 import ops
    return ops


def _n_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _fold(name, got, ref, bound, report):
    """_check one block of rows; report[name] keeps the worst ratio over the blocks."""
    rep = {}
    _check(name, got, ref, bound, rep)
    report[name] = max(report.get(name, 0.0), rep[name])


def _print(what, rep):
    print(f"\n{what}: worst err/bound " + " ".join(f"{n} {x:.3f}" for n, x in rep.items()))


def _desc(ops, proj, r, row_offset=77, layer=3):
    from bioreason_b200.engine import LoraDropout
    return ops.lora_dropout_desc(LoraDropout(seed=77, pass_id=3, threshold=T_DROP, row_offset=row_offset), layer, proj, r)


# ---------------------------------------------------------------------------------------------------------------------- lm-head
# (M, V, K, wide): V = 151 936 ends on a 256-wide tile holding one 128-column half, V = 152 000 on a half 64 columns wide; 4104 ends
# on a 128-wide tile holding 8 columns
LM_SHAPES = [(515, 151936, 2560, True), (300, 152000, 2560, True), (129, 4104, 256, False), (1, 1024, 2560, False), (64, 8, 64, False)]
LM_CASES = [s + (f, sc) for s in LM_SHAPES for f in gr.LM_FAMILIES for sc in (1.0, 1 / 0.6)]
_W = {}


def _lm_weight(V, K):
    """One lm-head weight at a time (the cases run shape by shape)."""
    if (V, K) not in _W:
        _W.clear()
        _W[(V, K)] = gr.make_lmhead_weight(V, K, seed=V + K, device="cuda")
    return _W[(V, K)]


def _lmhead_run(ops, M, V, K, family, scale):
    w = _lm_weight(V, K)
    h, tgt, same = gr.make_lmhead_inputs(family, w, M, gr.lmhead_targets(M, V, seed=M), scale=scale, seed=M + V)
    tgt = tgt.cuda()
    logp, lse = ops.lmhead_logprob(h, w, tgt, scale=scale)
    gs = torch.randn(M, generator=torch.Generator().manual_seed(M)).cuda()
    gs[3::5] *= 1e3                                                         # a spread of gradient scales
    buf = _nan_buffer(M, V, seed=5)
    sentinel = buf[:, V:].clone()
    ops.lmhead_dlogits(h, w, tgt, lse, gs, scale=scale, out=buf[:, :V])
    assert torch.equal(_bits(buf[:, V:]), _bits(sentinel)), "dlogits: write past the row"
    return w, h, tgt, same, gs, logp, lse, buf[:, :V]


@pytest.mark.parametrize("M,V,K,wide,family,scale", LM_CASES,
                         ids=[f"{M}x{V}x{K}-{f}-s{sc:.2f}" for M, V, K, _, f, sc in LM_CASES])
def test_lmhead_fp64(ops, M, V, K, wide, family, scale):
    assert _is_wide(M, V, K) == wide
    w, h, tgt, same, gs, logp, lse, d = _lmhead_run(ops, M, V, K, family, scale)
    rep = {}
    for r0 in range(0, M, LM_ROWS):
        r1 = min(M, r0 + LM_ROWS)
        r = gr.lmhead_ref(h[r0:r1], w, tgt[r0:r1], scale, lse_used=lse[r0:r1], gs=gs[r0:r1], same_sign=same)
        _fold("lse", lse[r0:r1], r["lse"], r["b_lse"], rep)
        _fold("logp", logp[r0:r1], r["logp"], r["b_logp"], rep)
        _fold("dlogits", d[r0:r1], r["d"], r["b_d"], rep)
        del r
    _print(f"lmhead {M}x{V}x{K} {'wide' if wide else 'narrow'} {family} scale {scale:.3f}", rep)


def test_lmhead_rejects_bug_variants(ops):
    """The kernel's own outputs against each lm-head bug variant: every one exceeds the bound >= 10x on the family built for it."""
    M, V, K = 300, 152000, 2560
    assert _is_wide(M, V, K)
    show = {"no_last_tile": "tail_max", "no_rescale": "tail_max", "tgt_neighbour": "random", "no_scale_dlogits": "random",
            "no_onehot_odd": "random"}
    rep = {}
    for family in sorted(set(show.values())):
        w, h, tgt, same, gs, logp, lse, d = _lmhead_run(ops, M, V, K, family, 1 / 0.6)
        sl = slice(0, LM_ROWS)
        kw = dict(lse_used=lse[sl], gs=gs[sl], same_sign=same)
        r = gr.lmhead_ref(h[sl], w, tgt[sl], 1 / 0.6, **kw)
        got = {"lse": lse[sl], "logp": logp[sl], "d": d[sl]}
        assert max(gr.worst_ratio(got[n], r[n], r["b_" + n]) for n in got) <= 1.0
        for variant in [v for v, f in show.items() if f == family]:
            m = gr.lmhead_ref(h[sl], w, tgt[sl], 1 / 0.6, variant=variant, **kw)
            rep[variant] = max(gr.worst_ratio(got[n], m[n], r["b_" + n]) for n in got)
    print("\nlmhead bug variants: err/bound " + " ".join(f"{n} {x:.3g}" for n, x in rep.items()))
    assert min(rep.values()) >= 10, rep


# ------------------------------------------------------------------------------------------------------------------------- GEMM
# (M, N, K, wide): the trainer's dense chunk (9456 rows) and shared-prefix buffer (6368) at Qwen3-4B widths, an N tail of 232
# (1000) and of 8 (2568) columns with a K tail of 8 (520); narrow: single-row / single-tile problems and partial M, N and K tiles
GEMM_SHAPES = [(9456, 2560, 2560, True), (9456, 6144, 2560, True), (6368, 19456, 2560, True), (9456, 2560, 9728, True),
               (9456, 1000, 2560, True), (9456, 2568, 520, True),
               (1, 8, 8, False), (127, 136, 72, False), (129, 264, 40, False), (300, 1000, 192, False)]


def _gemm_check(got, ref_fn, M, rep, names=("y",)):
    """got: name -> [M, n] output view; ref_fn(r0, r1): the gemm_ref dict of rows [r0, r1), checked one row block at a time."""
    for r0 in range(0, M, ROWS):
        r1 = min(M, r0 + ROWS)
        r = ref_fn(r0, r1)
        for n in names:
            _fold(n, got[n][r0:r1], r[n], r["b_" + n], rep)
        del r


@pytest.mark.parametrize("family", ("random", "tail_k", "tail_mn"))
@pytest.mark.parametrize("M,N,K,wide", GEMM_SHAPES)
def test_gemm_plain_fp64(ops, M, N, K, wide, family):
    assert _is_wide(M, N, K) == wide
    a, b = gr.make_gemm_inputs(family, M, N, K, seed=M + N + K, device="cuda")
    o32 = _nan_buffer(M, N, seed=1, dtype=torch.float32)
    o16 = _nan_buffer(M, N, seed=2)
    s32, s16 = o32[:, N:].clone(), o16[:, N:].clone()
    ops.gemm(a, b, out=o32[:, :N])
    ops.gemm(a, b, out=o16[:, :N])
    assert torch.equal(_bits(o32[:, N:]), _bits(s32)) and torch.equal(_bits(o16[:, N:]), _bits(s16)), "write past the row"
    rep = {}
    for r0 in range(0, M, ROWS):
        r1 = min(M, r0 + ROWS)
        r = gr.gemm_ref(a[r0:r1], b, out_f32=True)
        _fold("fp32", o32[r0:r1, :N], r["y"], r["b_y"], rep)
        _fold("bf16", o16[r0:r1, :N], r["y"], r["b_y"] + gr.SAFETY * gr.U_BF16 * r["y"].abs(), rep)     # + the output rounding
        del r
    _print(f"gemm {M}x{N}x{K} {'wide' if wide else 'narrow'} {family}", rep)


EPI_SHAPES = [(9456, 2560, 2560, True), (9456, 2568, 520, True), (129, 264, 40, False), (300, 1008, 192, False)]
EPILOGUES = ("bias_alpha_residual", "bias_f32_alpha", "residual_f32", "silu_aux", "row_map", "k2_32", "k2_96")


@pytest.mark.parametrize("epi", EPILOGUES)
@pytest.mark.parametrize("M,N,K,wide", EPI_SHAPES)
def test_gemm_epilogues_fp64(ops, M, N, K, wide, epi):
    assert _is_wide(M, N, K) == wide
    if epi == "silu_aux" and N % 16:
        pytest.skip("gated SiLU needs N % 16 == 0")
    a, b = gr.make_gemm_inputs("random", M, N, K, seed=M + 3 * N + K, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(N)
    bias = torch.randn(N, generator=gen, device="cuda").to(torch.bfloat16)
    rep = {}
    if epi in ("bias_alpha_residual", "residual_f32"):
        res = _nan_buffer(M, N, seed=3)
        res[:, :N] = torch.randn(M, N, generator=gen, device="cuda").to(torch.bfloat16)       # a strided residual
        f32 = epi == "residual_f32"
        out = _nan_buffer(M, N, seed=4, dtype=torch.float32 if f32 else torch.bfloat16)
        sent = out[:, N:].clone()
        kw = dict(residual=res[:, :N]) if f32 else dict(residual=res[:, :N], bias=bias, alpha=0.5)
        ops.gemm(a, b, out=out[:, :N], **kw)
        assert torch.equal(_bits(out[:, N:]), _bits(sent))
        _gemm_check({"y": out[:, :N]}, lambda r0, r1: gr.gemm_ref(a[r0:r1], b, out_f32=f32, **{**kw, "residual": kw["residual"][r0:r1]}),
                    M, rep)
    elif epi == "bias_f32_alpha":
        out = _nan_buffer(M, N, seed=4, dtype=torch.float32)
        sent = out[:, N:].clone()
        kw = dict(bias=bias.float() * 3, alpha=1.7)
        ops.gemm(a, b, out=out[:, :N], **kw)
        assert torch.equal(_bits(out[:, N:]), _bits(sent))
        _gemm_check({"y": out[:, :N]}, lambda r0, r1: gr.gemm_ref(a[r0:r1], b, out_f32=True, **kw), M, rep)
    elif epi == "silu_aux":
        out = _nan_buffer(M, N // 2, seed=4)
        aux = _nan_buffer(M, N, seed=5)
        so, sa = out[:, N // 2:].clone(), aux[:, N:].clone()
        kw = dict(bias=bias, alpha=0.8, act=1)
        ops.gemm(a, b, out=out[:, :N // 2], aux_out=aux[:, :N], **kw)
        assert torch.equal(_bits(out[:, N // 2:]), _bits(so)) and torch.equal(_bits(aux[:, N:]), _bits(sa))
        _gemm_check({"y": out[:, :N // 2], "aux": aux[:, :N]}, lambda r0, r1: gr.gemm_ref(a[r0:r1], b, **kw), M, rep,
                    names=("y", "aux"))
    elif epi == "row_map":
        g_ = torch.Generator().manual_seed(M)
        rm = torch.full((M,), -1, dtype=torch.int32)
        n_map = max(M - 20, M // 2)
        perm = torch.randperm(M + 80, generator=g_)[:n_map].int()
        rm[torch.randperm(M, generator=g_)[:n_map]] = perm
        rm = rm.cuda()
        dst = _nan_buffer(M + 80, N, seed=6)
        pre = dst.clone()
        ops.gemm(a, b, bias=bias, out=dst[:, :N], row_map=rm)
        hit = torch.zeros(M + 80, dtype=torch.bool, device="cuda")
        hit[rm[rm >= 0].long()] = True
        assert torch.equal(_bits(dst[~hit]), _bits(pre[~hit])), "rows no input maps to must keep their bits"
        assert torch.equal(_bits(dst[:, N:]), _bits(pre[:, N:]))
        for r0 in range(0, M, ROWS):
            r1 = min(M, r0 + ROWS)
            r = gr.gemm_ref(a[r0:r1], b, bias=bias)
            m = rm[r0:r1]
            keep = m >= 0
            _fold("y", dst[m[keep].long(), :N], r["y"][keep], r["b_y"][keep], rep)
            del r
    else:
        K2 = 32 if epi == "k2_32" else 96
        a2 = torch.randn(M, K2 + 8, generator=gen, device="cuda").to(torch.bfloat16)[:, :K2]               # strided operands
        b2 = torch.randn(N, K2 + 8, generator=gen, device="cuda").to(torch.bfloat16)[:, :K2]
        f32 = K2 == 32
        out = _nan_buffer(M, N, seed=4, dtype=torch.float32 if f32 else torch.bfloat16)
        sent = out[:, N:].clone()
        kw = dict(a2=a2, b2=b2) if f32 else dict(a2=a2, b2=b2, bias=bias.float())
        ops.gemm(a, b, out=out[:, :N], **kw)
        assert torch.equal(_bits(out[:, N:]), _bits(sent))
        _gemm_check({"y": out[:, :N]}, lambda r0, r1: gr.gemm_ref(a[r0:r1], b, out_f32=f32, **{**kw, "a2": a2[r0:r1]}), M, rep)
    _print(f"gemm {M}x{N}x{K} {'wide' if wide else 'narrow'} {epi}", rep)


def _masked_case(ops, M, N, K, r, n_proj, proj, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    dy = torch.randn(M, K, generator=gen, device="cuda").to(torch.bfloat16)
    w = (torch.randn(N, K, generator=gen, device="cuda") / K ** 0.5).to(torch.bfloat16)
    u = torch.randn(M, n_proj * r, generator=gen, device="cuda").to(torch.bfloat16)
    aT = torch.randn(N, n_proj * r, generator=gen, device="cuda").to(torch.bfloat16)
    bias = torch.randn(N, generator=gen, device="cuda").to(torch.bfloat16)
    masks = [ops.lora_dropout_mask(_desc(ops, proj + j, r), M, N, "cuda").bool() for j in range(n_proj)]
    out = _nan_buffer(M, N, seed=7, dtype=torch.float32)
    sent = out[:, N:].clone()
    ops.gemm(dy, w, a2=u, b2=aT, bias=bias, dropout=_desc(ops, proj, r), out=out[:, :N])
    assert torch.equal(_bits(out[:, N:]), _bits(sent))
    return dy, w, u, aT, bias, masks, out[:, :N]


# (M, N = dx width, K = dy width, r, n_proj, first projection): the qkv dX of one config (c) row at Qwen3-4B widths, and partial tiles
MASKED = [(2364, 2560, 6144, 32, 3, 0), (129, 136, 72, 16, 3, 4)]


@pytest.mark.parametrize("M,N,K,r,n_proj,proj", MASKED)
def test_gemm_masked_segment_fp64(ops, M, N, K, r, n_proj, proj):
    assert not _is_wide(M, N, K)                                           # the masked segment always runs 128-wide
    dy, w, u, aT, bias, masks, out = _masked_case(ops, M, N, K, r, n_proj, proj, seed=M)
    rep = {}
    _gemm_check({"y": out}, lambda r0, r1: gr.gemm_ref(dy[r0:r1], w, a2=u[r0:r1], b2=aT, bias=bias, out_f32=True,
                                                                   masks=[m[r0:r1] for m in masks], inv_keep=INV_KEEP), M, rep)
    _print(f"gemm masked LoRA segment {M}x{N}x{K} r={r} x{n_proj}", rep)


def test_gemm_rejects_bug_variants(ops):
    """The kernel's own outputs against each GEMM bug variant: every one exceeds the bound >= 10x."""
    rep = {}
    M, N, K = 9456, 2568, 520                                              # wide: bias halves of a 256-wide tile, K tail of 8
    assert _is_wide(M, N, K)
    bias = torch.randn(N, generator=torch.Generator(device="cuda").manual_seed(1), device="cuda").to(torch.bfloat16)
    for variant, family in (("bias_half", "random"), ("no_k_tail", "tail_k")):
        a, b = gr.make_gemm_inputs(family, M, N, K, seed=11, device="cuda")
        out = ops.gemm(a, b, bias=bias, out_dtype=torch.float32)
        r = gr.gemm_ref(a[:ROWS], b, bias=bias, out_f32=True)
        assert gr.worst_ratio(out[:ROWS], r["y"], r["b_y"]) <= 1.0
        m = gr.gemm_ref(a[:ROWS], b, bias=bias, out_f32=True, variant=variant)
        rep[variant] = gr.worst_ratio(out[:ROWS], m["y"], r["b_y"])
    dy, w, u, aT, bias, masks, out = _masked_case(ops, 129, 136, 72, 16, 3, 4, seed=2)
    kw = dict(a2=u, b2=aT, bias=bias, out_f32=True, masks=masks, inv_keep=INV_KEEP)
    r = gr.gemm_ref(dy, w, **kw)
    assert gr.worst_ratio(out, r["y"], r["b_y"]) <= 1.0
    rep["wrong_mask"] = gr.worst_ratio(out, gr.gemm_ref(dy, w, variant="wrong_mask", **kw)["y"], r["b_y"])
    print("\ngemm bug variants: err/bound " + " ".join(f"{n} {x:.3g}" for n, x in rep.items()))
    assert min(rep.values()) >= 10, rep


# ---------------------------------------------------------------------------------------------------------------- LoRA gradient
def _dst(rows, cols, seed):
    """fp32 [rows + 2, cols + PAD] holding data, and the [rows, cols] destination view inside it (one row above and below)."""
    buf = torch.randn(rows + 2, cols + PAD, generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda") * 5
    return buf, buf[1:rows + 1, :cols]


def _lora_run(ops, big, small, segs, mode, *, dropout=None, mask=None, what, rep, variants=()):
    """segs: [(row_lo, row_hi, col_lo, n_cols)]; runs ops.lora_grad_tn into fresh data-holding destinations and checks them."""
    M, P = big.shape
    N = small.shape[1]
    shapes = [(N, P) if mode == 1 else (P // 2, nc) if mode == 2 else (hi - lo, nc) for lo, hi, _, nc in segs]
    bufs = [_dst(rr, cc, seed=i + 1) for i, (rr, cc) in enumerate(shapes)]
    pre = [b.clone() for b, _ in bufs]
    ops.lora_grad_tn(big, small, [(v,) + tuple(s) for (_, v), s in zip(bufs, segs)], mode=mode, dropout=dropout)
    kw = dict(mask=mask, inv_keep=INV_KEEP if mask is not None else 1.0, n_sms=_n_sms())
    refs = gr.lora_grad_ref(big, small, segs, mode, [p[1:rr + 1, :cc] for p, (rr, cc) in zip(pre, shapes)], **kw)
    for i, ((buf, view), (ref, bound), p, (rr, cc)) in enumerate(zip(bufs, refs, pre, shapes)):
        outside = torch.ones_like(buf, dtype=torch.bool)
        outside[1:rr + 1, :cc] = False
        assert torch.equal(_bits(buf[outside]), _bits(p[outside])), f"{what} segment {i}: write outside the destination"
        _fold(f"seg{i}", view, ref, bound, rep)
    out = {}
    for variant in variants:
        m = gr.lora_grad_ref(big, small, segs, mode, [p[1:rr + 1, :cc] for p, (rr, cc) in zip(pre, shapes)], variant=variant, **kw)
        out[variant] = max(gr.worst_ratio(v, mr, b) for (_, v), (mr, _), (_, b) in zip(bufs, m, refs))
    return out


# The trainer's calls (training.policy_backward) at Qwen3-4B widths (d 2560, Hq*D 4096, F 9728, qkv 6144), r = 32, on the tokens of
# a 2-row config (c) chunk
TOK, RK = 4728, 32
LORA_TRAINER = {
    "qkv_dB": (6144, 3 * RK, 0, [(0, 4096, 0, RK), (4096, 5120, RK, RK), (5120, 6144, 2 * RK, RK)], None),      # 48 tiles: 2 splits
    "gate_up_dB": (19456, 2 * RK, 2, [(0, 19456, 0, RK), (0, 19456, RK, RK)], None),                          # 152 tiles: no exchange
    "down_dA": (9728, RK, 1, [(0, 9728, 0, RK)], None),                                                         # 76 tiles: 1 split
    "o_dA_dropout": (4096, RK, 1, [(0, 4096, 0, RK)], 3),
    "k_dA_dropout_strided_u": (2560, RK, 1, [(0, 2560, 0, RK)], 1),                                             # u[:, r:2r] of [M, 3r]
}


@pytest.mark.parametrize("name", list(LORA_TRAINER))
def test_lora_grad_trainer_calls_fp64(ops, name):
    P, N, mode, segs, proj = LORA_TRAINER[name]
    big, small = gr.make_lora_inputs("random", TOK, P, 3 * N if name.endswith("strided_u") else N, n_sms=_n_sms(), seed=P, device="cuda")
    if name.endswith("strided_u"):
        small = small[:, RK:2 * RK]
        assert not small.is_contiguous()
    dropout = mask = None
    if proj is not None:
        dropout = _desc(ops, proj, RK, row_offset=2364, layer=5)
        mask = ops.lora_dropout_mask(dropout, TOK, P, "cuda").bool()
    rep = {}
    _lora_run(ops, big, small, segs, mode, dropout=dropout, mask=mask, what=name, rep=rep)
    _print(f"lora_grad {name} M={TOK} P={P} N={N} splits={len(gr.lora_splits(TOK, P, _n_sms()))}", rep)


LORA_EDGES = [(M, P, N, mode) for M in (1, 63, 65, 1088) for P in (8, 136) for N in (8, 64, 72, 128) for mode in (0, 1)]


@pytest.mark.parametrize("M,P,N,mode", LORA_EDGES)
def test_lora_grad_edges_fp64(ops, M, P, N, mode):
    big, small = gr.make_lora_inputs("random", M, P, N, n_sms=_n_sms(), seed=M * P + N, device="cuda")
    h = N // 2
    segs = [(0, P, 0, N)] if mode == 1 else [(0, P // 2, 0, h), (P // 2, P, h, N - h)]
    rep = {}
    _lora_run(ops, big, small, segs, mode, what="edge", rep=rep)
    _print(f"lora_grad M={M} P={P} N={N} mode {mode} splits={len(gr.lora_splits(M, P, _n_sms()))}", rep)


@pytest.mark.parametrize("family", gr.LORA_FAMILIES)
@pytest.mark.parametrize("M,P,N,mode", [(1000, 136, 72, 0), (1088, 8, 64, 1), (65, 144, 72, 2), (1000, 144, 64, 2)])
def test_lora_grad_families_fp64(ops, M, P, N, mode, family):
    big, small = gr.make_lora_inputs(family, M, P, N, n_sms=_n_sms(), seed=M + P, device="cuda")
    segs = {0: [(0, 64, 8, 24), (64, P, 40, 32)], 1: [(0, P, 0, N)], 2: [(0, P, 0, N // 2), (0, P, N // 2, N // 2)]}[mode]
    rep = {}
    _lora_run(ops, big, small, segs, mode, what=family, rep=rep)
    _print(f"lora_grad M={M} P={P} N={N} mode {mode} {family}", rep)


def test_lora_grad_rejects_bug_variants(ops):
    """The kernel's own outputs against each LoRA-gradient bug variant: every one exceeds the bound >= 10x."""
    rep, junk = {}, {}
    M = 1000                                                               # 16 token blocks, the last one 40 tokens
    big, small = gr.make_lora_inputs("tail_split", M, 136, 72, n_sms=_n_sms(), seed=1, device="cuda")
    rep.update(_lora_run(ops, big, small, [(0, 136, 0, 72)], 1, what="split", rep=junk, variants=("no_last_split",)))
    big, small = gr.make_lora_inputs("tail_token", M, 136, 72, n_sms=_n_sms(), seed=2, device="cuda")
    rep.update(_lora_run(ops, big, small, [(0, 136, 0, 72)], 1, what="tail", rep=junk, variants=("no_token_tail",)))
    big, small = gr.make_lora_inputs("random", M, 144, 64, n_sms=_n_sms(), seed=3, device="cuda")
    rep.update(_lora_run(ops, big, small, [(0, 144, 0, 32), (0, 144, 32, 32)], 2, what="gate/up", rep=junk,
                         variants=("gate_up_swapped",)))
    print("\nlora_grad bug variants: err/bound " + " ".join(f"{n} {x:.3g}" for n, x in rep.items()))
    assert min(rep.values()) >= 10, rep
