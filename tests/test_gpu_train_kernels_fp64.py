"""Training attention (dense and shared-prefix forward / backward) and the backward row kernels (RMSNorm, SwiGLU, q/k-norm + RoPE)
against float64 references with per-element error bounds (tests/attn_ref.py has the attention model), at the shapes and mask edges
where these kernels go wrong.  Outputs are NaN-prefilled and strided with sentinel columns, so a tile that is never stored or a
store past the row shows up.  Run with -s to see the worst err / bound ratio of every output."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attn_ref as ar  # noqa: E402

pytestmark = pytest.mark.gpu

D = 128
PAD = 64                                           # sentinel columns after every strided output
U, W_ACC, SAFETY = ar.U_BF16, ar.W_ACC, ar.SAFETY


@pytest.fixture(scope="module")
def ops():
    from bioreason_b200 import ops
    return ops


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _nan_buffer(rows, width, seed, dtype=torch.bfloat16):
    """[rows, width + PAD] (bf16 or fp32), NaN in the first `width` columns and a seeded sentinel pattern after them."""
    buf = torch.full((rows, width + PAD), math.nan, dtype=dtype, device="cuda")
    buf[:, width:] = torch.randn(rows, PAD, generator=torch.Generator().manual_seed(seed)).to(dtype).cuda()
    return buf


def _check(name, got, ref, bound, report):
    got = got.to(torch.float64)
    assert torch.isfinite(got).all(), f"{name}: {int((~torch.isfinite(got)).sum())} non-finite elements"
    worst = ar.worst_ratio(got, ref, bound)
    report[name] = worst
    assert worst <= 1.0, f"{name}: err / bound = {worst:.3g}"


def _check_lse(lse, r, report):
    fin = torch.isfinite(r["lse"])
    assert torch.equal(torch.isfinite(lse), fin), "lse must be finite exactly where a key is visible"
    assert (lse[~fin] == math.inf).all(), "lse of a row with no visible key must be +inf"
    _check("lse", lse[fin], r["lse"][fin], r["b_lse"][fin], report)


# ------------------------------------------------------------------------------------------------------------ dense attention
# (Hq, Hkv, B, L, windows)
DENSE = [
    (32, 8, 2, 2364, [(0, 2364), (188, 2327)]),          # config (c): Qwen3-4B heads, left pad off the tile grid, post-EOS tail
    (16, 8, 3, 129, [(0, 129), (64, 129), (63, 65)]),    # Qwen3-1.7B heads; windows on and one off a tile edge
    (4, 2, 2, 1, [(0, 1), (0, 1)]),
    (4, 2, 2, 63, [(0, 63), (62, 63)]),
    (4, 2, 2, 64, [(0, 64), (63, 64)]),
    (4, 2, 2, 65, [(0, 65), (64, 65)]),
    (4, 2, 3, 65, [(0, 65), (64, 65), (0, 0)]),          # the empty window of an all-pad row (engine.mask_window)
    (8, 2, 2, 200, [(65, 130), (65, 130)]),              # GQA 4:1, a window inside the row
]
FAMILIES = ("random", "decoy", "first_key")


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("Hq,Hkv,B,L,windows", DENSE, ids=lambda x: str(x).replace(" ", "") if isinstance(x, list) else None)
def test_attn_dense_fp64(ops, Hq, Hkv, B, L, windows, family):
    q, k, v, do = ar.make_inputs(family, B, L, Hq, Hkv, windows, seed=L + B, device="cuda")
    W = (Hq + 2 * Hkv) * D
    qo, ko, vo = 0, Hq * D, (Hq + Hkv) * D
    qkv = torch.cat([q.reshape(B * L, Hq * D), k.reshape(B * L, Hkv * D), v.reshape(B * L, Hkv * D)], 1)     # one fused buffer
    ks = torch.tensor([w[0] for w in windows], dtype=torch.int32, device="cuda")
    ke = torch.tensor([w[1] for w in windows], dtype=torch.int32, device="cuda")
    o = torch.full((B * L, Hq * D), math.nan, dtype=torch.bfloat16, device="cuda")
    o, lse = ops.attn_fwd(qkv[:, qo:ko], qkv[:, ko:vo], qkv[:, vo:], B, L, Hq, Hkv, D, kv_start=ks, kv_end=ke, causal=True,
                          want_lse=True, out=o)
    dob = do.reshape(B * L, Hq * D)

    def bwd():
        g = _nan_buffer(B * L, W, seed=1)
        sentinel = g[:, W:].clone()
        ops.attn_bwd(qkv[:, qo:ko], qkv[:, ko:vo], qkv[:, vo:], o, dob, lse, g[:, qo:ko], g[:, ko:vo], g[:, vo:W], B, L, Hq, Hkv, D,
                     kv_start=ks, kv_end=ke)
        assert torch.equal(_bits(g[:, W:]), _bits(sentinel)), "write past the dq / dk / dv columns"
        return g
    g = bwd()
    assert torch.equal(_bits(bwd()), _bits(g)), "backward not bit-reproducible"
    r = ar.attn_ref(q, k, v, do, windows, o_used=o.view(B, L, Hq, D))
    rep = {}
    _check("O", o.view(B, L, Hq, D), r["o"], r["b_o"], rep)
    _check_lse(lse, r, rep)
    _check("dQ", g[:, qo:ko].reshape(B, L, Hq, D), r["dq"], r["b_dq"], rep)
    _check("dK", g[:, ko:vo].reshape(B, L, Hkv, D), r["dk"], r["b_dk"], rep)
    _check("dV", g[:, vo:W].reshape(B, L, Hkv, D), r["dv"], r["b_dv"], rep)
    print(f"\ndense {Hq}/{Hkv} B={B} L={L} {family}: worst err/bound " + " ".join(f"{n} {x:.3f}" for n, x in rep.items()))


# ---------------------------------------------------------------------------------------------------- shared-prefix attention
# (U, G, Lp, Ls, Hq, Hkv, kv_start per group, kv_end per row)
SHARED = [
    (1, 8, 1792, 572, 32, 8, [0], [2364, 2364 - 37, 1853, 2364, 1900, 2364, 2364, 2000]),     # config (c)
    (2, 4, 128, 70, 8, 2, [0, 30], [198, 150, 198, 129, 198, 198, 140, 175]),
]


@pytest.mark.parametrize("Uu,G,Lp,Ls,Hq,Hkv,kv_start,kv_end", SHARED)
def test_attn_shared_fp64(ops, Uu, G, Lp, Ls, Hq, Hkv, kv_start, kv_end):
    R, L = Uu * G, Lp + Ls
    windows = [(kv_start[r // G], kv_end[r]) for r in range(R)]
    q, k, v, do = ar.make_inputs("decoy", R, L, Hq, Hkv, windows, seed=L, device="cuda", group=(G, Lp))
    do = do.clone()
    do[torch.arange(R) % G != 0, :Lp] = 0                      # prefix dO lives once per group: row g = 0 of the dense equivalent
    fold = lambda t, prefix="sum": ar.fold_shared(t, Uu, G, Lp, Ls, prefix=prefix)
    W = (Hq + 2 * Hkv) * D
    qo, ko, vo = 0, Hq * D, (Hq + Hkv) * D
    N = Uu * Lp + R * Ls
    buf = torch.cat([fold(t, "first").reshape(N, -1) for t in (q, k, v)], 1)
    do_buf = fold(do).reshape(N, Hq * D)
    ks = torch.tensor(kv_start, dtype=torch.int32, device="cuda")
    ke = torch.tensor(kv_end, dtype=torch.int32, device="cuda")
    o = torch.full((N, Hq * D), math.nan, dtype=torch.bfloat16, device="cuda")
    o, (lse_p, lse_s) = ops.attn_fwd_shared(buf[:, qo:ko], buf[:, ko:vo], buf[:, vo:], Uu, G, Lp, Ls, Hq, Hkv, D, ks, ke, want_lse=True, out=o)

    def bwd():
        g = _nan_buffer(N, W, seed=2)
        sentinel = g[:, W:].clone()
        ops.attn_bwd_shared(buf[:, qo:ko], buf[:, ko:vo], buf[:, vo:], o, do_buf, (lse_p, lse_s), g[:, qo:ko], g[:, ko:vo], g[:, vo:W],
                            Uu, G, Lp, Ls, Hq, Hkv, D, ks, ke)
        assert torch.equal(_bits(g[:, W:]), _bits(sentinel)), "write past the dq / dk / dv columns"
        return g
    g = bwd()
    assert torch.equal(_bits(bwd()), _bits(g)), "backward not bit-reproducible"
    o_dense = ar.expand_shared(o.view(N, Hq, D), Uu, G, Lp, Ls)
    r = ar.attn_ref(q, k, v, do, windows, o_used=o_dense)
    rep = {}
    _check("O", o.view(N, Hq, D), fold(r["o"], "first"), fold(r["b_o"], "first"), rep)
    lse = torch.cat([lse_p.repeat_interleave(G, 0), lse_s], 2)                                # [R, Hq, L] dense equivalent
    _check_lse(lse, r, rep)
    for name, sl, key, H in (("dQ", slice(qo, ko), "dq", Hq), ("dK", slice(ko, vo), "dk", Hkv), ("dV", slice(vo, W), "dv", Hkv)):
        _check(name, g[:, sl].reshape(N, H, D), fold(r[key]), fold(r["b_" + key]), rep)
    print(f"\nshared U={Uu} G={G} Lp={Lp} Ls={Ls} {Hq}/{Hkv} decoy: worst err/bound " + " ".join(f"{n} {x:.3f}" for n, x in rep.items()))


# ------------------------------------------------------------------------------------------------------------------ row kernels
def _strided(rows, width, gen, scale=1.0):
    """bf16 [rows, width] view with row stride width + PAD."""
    return (torch.randn(rows, width + PAD, generator=gen) * scale).to(torch.bfloat16).cuda()[:, :width]


def _row_check(name, got_full, width, prefill, ref, bound, report):
    """got_full: the whole strided output buffer; its sentinel columns must be untouched."""
    assert torch.equal(_bits(got_full[:, width:]), _bits(prefill[:, width:])), f"{name}: write past the row"
    _check(name, got_full[:, :width], ref, bound, report)


@pytest.mark.parametrize("d", [128, 512, 1024, 2048, 2560, 4096])         # VEC_ITERS 1, 4, 4, 8, 16, 16
@pytest.mark.parametrize("M", [1, 9, 4733])
def test_rmsnorm_bwd_fp64(ops, d, M):
    gen = torch.Generator().manual_seed(d + M)
    x, dy, dres = _strided(M, d, gen, 2.0), _strided(M, d, gen), _strided(M, d, gen)
    w = (1 + 0.1 * torch.randn(d, generator=gen)).to(torch.bfloat16).cuda()
    eps = 1e-6
    _, rstd = ops.rmsnorm(x, w, eps, want_rstd=True)
    xr = x.double().requires_grad_(True)
    (w.double() * xr * torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + eps)).backward(dy.double())
    # dx = r (w o dy) - x r^3 mean(x o w o dy) (+ dres): bound 2u times the sum of the absolute terms
    rr = torch.rsqrt(x.double().pow(2).mean(-1, keepdim=True) + eps)
    wd = (w.double() * dy.double()).abs()
    T = rr * wd + x.double().abs() * rr ** 3 * (x.double().abs() * wd).mean(-1, keepdim=True)
    rep = {}
    for with_res in (False, True):
        out = _nan_buffer(M, d, seed=3)
        prefill = out.clone()
        ops.rmsnorm_bwd(x, w, rstd, dy, dres=dres if with_res else None, out=out[:, :d])
        ref = xr.grad + (dres.double() if with_res else 0.0)
        bound = SAFETY * (2 * U * (T + (dres.double().abs() if with_res else 0.0)) + 1e-6)
        _row_check("dx+dres" if with_res else "dx", out, d, prefill, ref, bound, rep)
    print(f"\nrmsnorm_bwd d={d} M={M}: worst err/bound " + " ".join(f"{n} {x:.3f}" for n, x in rep.items()))


def test_rmsnorm_bwd_rejects_wide_rows(ops):
    x = torch.zeros(1, 4104, dtype=torch.bfloat16, device="cuda")
    rstd = torch.ones(1, device="cuda")
    with pytest.raises(RuntimeError, match="rmsnorm_bwd"):
        ops.rmsnorm_bwd(x, x[0], rstd, x)


@pytest.mark.parametrize("F", [512, 1536, 6144, 9728])
def test_swiglu_bwd_fp64(ops, F):
    M = 37
    gen = torch.Generator().manual_seed(F)
    g = torch.rand(M, F, generator=gen) * 60 - 30                       # saturated on both sides
    g.view(-1)[::97] = 0.0
    g.view(-1)[1::97] = 1e-3
    g.view(-1)[2::97] = -1e-3
    g = g.to(torch.bfloat16)
    up = torch.randn(M, F, generator=gen).to(torch.bfloat16)
    dact_s = torch.randn(M, F + PAD, generator=gen)
    dact_s[:, :F][torch.rand(M, F, generator=gen) < 0.1] = 0.0           # zeros in the incoming gradient
    dact = dact_s.to(torch.bfloat16).cuda()[:, :F]
    gu_full = torch.randn(M, 2 * F + PAD, generator=gen).to(torch.bfloat16)
    blk = gu_full[:, :2 * F].view(M, F // 8, 2, 8)
    blk[:, :, 0] = g.view(M, F // 8, 8)
    blk[:, :, 1] = up.view(M, F // 8, 8)
    gu = gu_full.cuda()[:, :2 * F]
    out = _nan_buffer(M, 2 * F, seed=4)
    prefill = out.clone()
    ops.swiglu_bwd(gu, dact, out=out[:, :2 * F])
    gr, ur = g.double().cuda().requires_grad_(True), up.double().cuda().requires_grad_(True)
    (torch.nn.functional.silu(gr) * ur).backward(dact.double())
    gd, ud, dd = g.double().cuda(), up.double().cuda(), dact.double()
    s = torch.sigmoid(gd)
    Tg = (dd * ud * s).abs() + (dd * ud * s * gd * (1 - s)).abs()        # d u s (1 + g (1 - s))
    Tu = (dd * gd * s).abs()                                             # d g s
    ref = torch.stack([gr.grad.view(M, F // 8, 8), ur.grad.view(M, F // 8, 8)], 2).view(M, 2 * F)
    bound = SAFETY * (2 * U * torch.stack([Tg.view(M, F // 8, 8), Tu.view(M, F // 8, 8)], 2).view(M, 2 * F) + 1e-6)
    rep = {}
    _row_check("dgu", out, 2 * F, prefill, ref, bound, rep)
    print(f"\nswiglu_bwd F={F}: worst err/bound {rep['dgu']:.3f}")


def _ulp32(x):
    """Unit in the last place of fp32 values (float64 result)."""
    _, e = torch.frexp(x.to(torch.float32).abs())
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), (e - 24).to(torch.int64))


POSITIONS = list(range(2364)) + [4095, 4096, 40959]


@pytest.mark.parametrize("nq,nk", [(32, 8), (16, 8), (4, 2)])
def test_qk_rope_bwd_fp64(ops, nq, nk):
    gen = torch.Generator().manual_seed(nq)
    M, H = len(POSITIONS), nq + nk
    W = (nq + 2 * nk) * D
    theta, eps = 1e6, 1e-6
    pos = torch.tensor(POSITIONS, dtype=torch.int32, device="cuda")
    pre = _strided(M, W, gen)
    qw = (1 + 0.1 * torch.randn(D, generator=gen)).to(torch.bfloat16).cuda()
    kw = (1 + 0.1 * torch.randn(D, generator=gen)).to(torch.bfloat16).cuda()
    dfull = torch.randn(M, W + PAD, generator=gen).to(torch.bfloat16).cuda()
    dy = dfull.clone()
    ops.qk_rope_bwd_(dfull[:, :W], pre, nq, nk, D, qw, kw, pos, theta, eps)
    assert torch.equal(_bits(dfull[:, H * D:]), _bits(dy[:, H * D:])), "the V and sentinel columns must come back untouched"
    # fp64 autograd of y = rot(pos) (w o x rstd), exact angles
    x = pre[:, :H * D].double().view(M, H, D).requires_grad_(True)
    w = torch.cat([qw[None].expand(nq, D), kw[None].expand(nk, D)]).double()[None]
    rstd = torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps)
    xn = w * x * rstd
    j = torch.arange(D // 2, device="cuda", dtype=torch.float64)
    ang = pos.double()[:, None] * theta ** (-2 * j / D)[None]
    c, s = torch.cat([ang.cos(), ang.cos()], -1)[:, None], torch.cat([ang.sin(), ang.sin()], -1)[:, None]
    y = xn * c + torch.cat([-xn[..., D // 2:], xn[..., :D // 2]], -1) * s
    g = dy[:, :H * D].double().view(M, H, D)
    y.backward(g)
    # bound: the kernel rotates dy back with bf16 cos / sin of an fp32 angle.  2u covers the cos / sin and output roundings; the
    # angle itself is off by up to 2 pos ulp(inv_freq) (powf + reciprocal) + ulp(angle) (the product) + 2^-21 (sincosf)
    inv32 = (1.0 / torch.pow(torch.tensor(theta, dtype=torch.float32), (2 * j / D).float())).cuda()
    dth = 2 * pos.double()[:, None] * _ulp32(inv32)[None] + _ulp32(pos.float()[:, None] * inv32[None]) + 2.0 ** -21
    dth = torch.cat([dth, dth], -1)[:, None]
    gl, gh = g[..., :D // 2], g[..., D // 2:]
    ca, sa = c[..., :D // 2].abs(), s[..., :D // 2].abs()
    Dabs = torch.cat([gl.abs() * ca + gh.abs() * sa, gl.abs() * sa + gh.abs() * ca], -1)      # |terms| of the rotated dy
    Eang = torch.cat([gl.abs() + gh.abs()] * 2, -1) * dth                                    # its error from the angle
    r = rstd.detach()
    wx = (w * x.detach()).abs()
    norm_t = lambda t: r * w.abs() * t + x.detach().abs() * r ** 3 * (wx * t).mean(-1, keepdim=True)
    bound = SAFETY * (2 * U * norm_t(Dabs) + norm_t(Eang) + 1e-6)
    rep = {}
    _check("dqk", dfull[:, :H * D].view(M, H, D), x.grad, bound, rep)
    print(f"\nqk_rope_bwd {nq}/{nk}: worst err/bound {rep['dqk']:.3f}")


def test_qk_rope_table_matches_inline(ops):
    """The training forward's cos / sin table path equals the inline path bit for bit, below the table length and past it (the
    inline fallback), and out= leaves the input untouched."""
    gen = torch.Generator().manual_seed(5)
    nq, nk = 32, 8
    W = (nq + 2 * nk) * D
    table = ops.rope_table(4096, D, 1e6, "cuda")
    pos = torch.tensor(list(range(0, 4096, 7)) + [4095, 4096, 4097, 40959], dtype=torch.int32, device="cuda")
    M = pos.numel()
    qkv = torch.randn(M, W, generator=gen).to(torch.bfloat16).cuda()
    qw = (1 + 0.1 * torch.randn(D, generator=gen)).to(torch.bfloat16).cuda()
    kw = (1 + 0.1 * torch.randn(D, generator=gen)).to(torch.bfloat16).cuda()
    before = qkv.clone()
    kw_ = dict(q_norm_w=qw, k_norm_w=kw, eps=1e-6, mode=0)
    o_tab = ops.qk_rope_(qkv, nq, nk, D, pos, 1e6, out=torch.empty(M, (nq + nk) * D, dtype=torch.bfloat16, device="cuda"), rope=table, **kw_)
    assert torch.equal(_bits(qkv), _bits(before)), "out= must leave the input untouched"
    o_inl = ops.qk_rope_(qkv, nq, nk, D, pos, 1e6, out=torch.empty_like(o_tab), **kw_)
    assert torch.equal(_bits(o_tab), _bits(o_inl))
    ops.qk_rope_(qkv, nq, nk, D, pos, 1e6, rope=table, **kw_)                                  # in place
    assert torch.equal(_bits(qkv[:, :(nq + nk) * D]), _bits(o_tab)) and torch.equal(_bits(qkv[:, (nq + nk) * D:]), _bits(before[:, (nq + nk) * D:]))


def test_rope_table_matches_hf_rotary(ops):
    """ops.rope_table against transformers' Qwen3RotaryEmbedding (qwen3-4b config, every position up to 40959): per entry at most one
    bf16 ulp plus the angle change of one fp32 ulp of inv_freq_j (pos ulp(inv_freq_j)) and of the rounded product (ulp(angle))."""
    pytest.importorskip("transformers")
    from transformers.models.qwen3.modeling_qwen3 import Qwen3RotaryEmbedding
    from bioreason_b200.configs import text_config
    cfg = text_config("qwen3-4b")
    n = 40960
    rot = Qwen3RotaryEmbedding(cfg)
    pos = torch.arange(n)[None]
    cos_hf, sin_hf = rot(torch.zeros(1, dtype=torch.bfloat16), pos)
    half = D // 2
    hf = torch.stack([cos_hf[0, :, :half], sin_hf[0, :, :half]], -1).double()                # [n, 64, 2]
    assert torch.equal(cos_hf[0, :, :half], cos_hf[0, :, half:])
    tab = ops.rope_table(n, D, 1e6, "cuda").cpu().double()
    inv = rot.inv_freq.float()
    ang = pos[0].float()[:, None] * inv[None]
    slack = (torch.arange(n, dtype=torch.float64)[:, None] * _ulp32(inv)[None] + _ulp32(ang))[..., None]
    mag = torch.maximum(tab.abs(), hf.abs()).to(torch.bfloat16).float()
    _, e = torch.frexp(mag)
    ulp_bf16 = torch.where(mag > 0, torch.ldexp(torch.ones_like(mag), (e - 8).to(torch.int64)), 2.0 ** -133).double()
    diff = (tab - hf).abs()
    ratio = (diff / (ulp_bf16 + slack)).max().item()
    neq = (diff > 0).double().mean().item()
    print(f"\nrope_table vs HF Qwen3RotaryEmbedding: {neq:.2e} of entries not bit-equal; worst diff / allowed {ratio:.3f}")
    assert ratio <= 1.0
