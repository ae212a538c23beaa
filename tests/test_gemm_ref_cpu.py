"""The fp64 GEMM, lm-head and LoRA-gradient references and their error bounds (tests/gemm_ref.py), checked without a GPU: each reference
equals a direct float64 formula (autograd for dlogits), an fp32 emulation of each kernel's arithmetic stays inside the bound, and a
reference carrying one typical kernel bug breaks the bound by >= 10x on at least one input family, so the GPU tests built on it would
catch that bug."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gemm_ref as gr  # noqa: E402
from lora_dropout_ref import keep_mask, threshold  # noqa: E402

N_SMS = 132
P_DROP = 0.05
T_DROP = threshold(P_DROP)
INV_KEEP = 65536.0 / (65536 - T_DROP)


def _close(a, b):
    torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)


def _bf(x):
    return x.to(torch.bfloat16).float()


def _masks(M, N, n_proj, proj=0, row0=77):
    return [torch.from_numpy(keep_mask(5, 3, 2, proj + j, np.arange(row0, row0 + M), N, T_DROP)) for j in range(n_proj)]


# ------------------------------------------------------------------------------------------------------------ fp32 emulations
def _chunks(a, b, acc=None):
    """acc (+)= a b^T in fp32, one exact k16 chunk product after another (the contraction runs over the columns)."""
    if acc is None:
        acc = torch.zeros(a.shape[0], b.shape[0], dtype=torch.float32)
    for k in range(0, a.shape[1], 16):
        acc += (a[:, k:k + 16].double() @ b[:, k:k + 16].double().T).float()
    return acc


def gemm_emul(a, b, *, alpha=1.0, bias=None, residual=None, act=0, out_f32=False, a2=None, b2=None, masks=None, inv_keep=1.0):
    acc = _chunks(a, b)
    if a2 is not None and masks is None:
        acc = _chunks(a2, b2, acc)
    elif a2 is not None:
        r = a2.shape[1] // len(masks)
        for j, m in enumerate(masks):
            tmp = _chunks(a2[:, j * r:(j + 1) * r], b2[:, j * r:(j + 1) * r])
            acc += torch.where(m, tmp * torch.tensor(inv_keep, dtype=torch.float32), 0.0)
    v = acc * torch.tensor(alpha, dtype=torch.float32)
    if bias is not None:
        v = v + bias.float()
    M, N = v.shape
    if act == 1:
        g = _bf(v.view(M, N // 16, 2, 8)[:, :, 0].reshape(M, N // 2))
        u = _bf(v.view(M, N // 16, 2, 8)[:, :, 1].reshape(M, N // 2))
        return {"y": _bf(_bf(g / (1 + torch.exp(-g))) * u), "aux": _bf(v)}
    if residual is not None:
        v = _bf(v) + residual.float()
    return {"y": v if out_f32 else _bf(v)}


def lmhead_emul(h, w, tgt, scale, gs):
    z = _chunks(h, w) * torch.tensor(scale, dtype=torch.float32)
    M, V = z.shape
    nt = math.ceil(V / gr.TILE)
    zp = torch.nn.functional.pad(z, (0, nt * gr.TILE - V), value=-math.inf).view(M, nt, gr.TILE)
    mt = zp.amax(2)
    st = torch.exp(zp - mt[..., None]).sum(2)
    gmax = mt.amax(1)
    lse = torch.log((st * torch.exp(mt - gmax[:, None])).sum(1)) + gmax
    has = tgt >= 0
    logp = torch.where(has, z.gather(1, tgt.clamp(min=0)[:, None])[:, 0] - lse, 0.0)
    onehot = torch.zeros_like(z)
    onehot[torch.nonzero(has)[:, 0], tgt[has]] = 1.0
    d = _bf(gs.float()[:, None] * (onehot - torch.exp(z - lse[:, None])))
    return logp, lse, d


def lora_emul(big, small, segs, mode, prev, *, mask=None, inv_keep=1.0):
    M, P = big.shape
    N = small.shape[1]
    x = big.float() * mask.float() if mask is not None else big.float()
    v = torch.zeros(P, N, dtype=torch.float32)
    for lo, hi in gr.lora_splits(M, P, N_SMS):
        part = _chunks(x[lo:hi].T.contiguous(), small[lo:hi].float().T.contiguous())
        if mask is not None:
            part = part * torch.tensor(inv_keep, dtype=torch.float32)
        v += part
    out = []
    for i, (row_lo, row_hi, col_lo, n_cols) in enumerate(segs):
        if mode == 1:
            inc = v.T
        elif mode == 2:
            inc = v.view(P // 16, 2, 8, N)[:, i].reshape(P // 2, N)[:, col_lo:col_lo + n_cols]
        else:
            inc = v[row_lo:row_hi, col_lo:col_lo + n_cols]
        out.append(prev[i].float() + inc)
    return out


# ------------------------------------------------------------------------------------------------------------------------- GEMM
GM, GN, GK, R, NP = 130, 272, 200, 16, 3          # K % 64 = 8, N = 272: a 256-wide tile plus 16 columns, 3 projections of r = 16


def _gemm_case(family, seed=1):
    a, b = gr.make_gemm_inputs(family, GM, GN, GK, seed=seed)
    gen = torch.Generator().manual_seed(seed + 7)
    bias = torch.randn(GN, generator=gen).to(torch.bfloat16)
    res = torch.randn(GM, GN, generator=gen).to(torch.bfloat16)
    a2 = torch.randn(GM, NP * R, generator=gen).to(torch.bfloat16)
    b2 = torch.randn(GN, NP * R, generator=gen).to(torch.bfloat16)
    return a, b, bias, res, a2, b2


EPILOGUES = {
    "plain_f32": dict(out_f32=True),
    "bias_alpha_residual": dict(bias=True, alpha=0.5, residual=True),
    "bias_f32_out_f32": dict(bias="f32", out_f32=True, alpha=1.7),
    "residual_f32": dict(residual=True, out_f32=True),
    "silu": dict(act=1, bias=True, alpha=0.8),
    "k2": dict(k2=True),
    "masked": dict(k2=True, masked=True, bias=True),
}


def _kw(spec, bias, res, a2, b2):
    kw = dict(alpha=spec.get("alpha", 1.0), act=spec.get("act", 0))
    if "out_f32" in spec:
        kw["out_f32"] = True
    if spec.get("bias"):
        kw["bias"] = bias.float() if spec["bias"] == "f32" else bias
    if spec.get("residual"):
        kw["residual"] = res
    if spec.get("k2"):
        kw.update(a2=a2, b2=b2)
    if spec.get("masked"):
        kw.update(masks=_masks(GM, GN, NP), inv_keep=INV_KEEP)
    return kw


@pytest.mark.parametrize("epi", list(EPILOGUES))
def test_gemm_reference_matches_direct(epi):
    a, b, bias, res, a2, b2 = _gemm_case("random")
    kw = _kw(EPILOGUES[epi], bias, res, a2, b2)
    r = gr.gemm_ref(a, b, **kw)
    lin = torch.nn.functional.linear(a.double(), b.double())
    if "a2" in kw:
        if "masks" in kw:
            for j, m in enumerate(kw["masks"]):
                lin = lin + m.double() * INV_KEEP * torch.nn.functional.linear(a2[:, j * R:(j + 1) * R].double(), b2[:, j * R:(j + 1) * R].double())
        else:
            lin = lin + torch.nn.functional.linear(a2.double(), b2.double())
    lin = kw["alpha"] * lin + (kw["bias"].double() if "bias" in kw else 0.0)
    if kw["act"] == 1:
        blk = lin.view(GM, GN // 16, 2, 8)
        want = (torch.nn.functional.silu(blk[:, :, 0]) * blk[:, :, 1]).reshape(GM, GN // 2)
        _close(r["aux"], lin)
    else:
        want = lin + (res.double() if "residual" in kw else 0.0)
    _close(r["y"], want)
    assert (r["b_y"] > 0).all()


@pytest.mark.parametrize("family", ("random", "tail_k", "tail_mn"))
@pytest.mark.parametrize("epi", list(EPILOGUES))
def test_gemm_emulation_within_bound(epi, family):
    a, b, bias, res, a2, b2 = _gemm_case(family)
    kw = _kw(EPILOGUES[epi], bias, res, a2, b2)
    r = gr.gemm_ref(a, b, **kw)
    em = gemm_emul(a, b, **kw)
    worst = {n: gr.worst_ratio(em[n], r[n], r["b_" + n]) for n in em}
    print(f"{epi} {family}: " + " ".join(f"{n} {x:.3g}" for n, x in worst.items()))
    assert max(worst.values()) <= 1.0, worst
    if family == "tail_mn" and not {"bias", "residual", "a2"} & set(kw):
        zero = r["b_y"] == 0                                  # outside the corner tile every output is an exact zero
        assert zero.any() and (r["y"][zero] == 0).all()


@pytest.mark.parametrize("variant", gr.GEMM_VARIANTS)
def test_gemm_variants_break_the_bound(variant):
    """bias_half on random, no_k_tail on tail_k (every product term lives in the K tail), wrong_mask on random (a LoRA segment that
    outweighs the main product)."""
    worst = {}
    for family in ("random", "tail_k", "tail_mn"):
        a, b, bias, res, a2, b2 = _gemm_case(family)
        kw = _kw(EPILOGUES["masked"], bias, res, a2, b2)
        kw["out_f32"] = True
        r = gr.gemm_ref(a, b, **kw)
        m = gr.gemm_ref(a, b, variant=variant, **kw)
        worst[family] = gr.worst_ratio(m["y"], r["y"], r["b_y"])
    print(f"{variant}: " + " ".join(f"{f} {x:.3g}" for f, x in worst.items()))
    assert max(worst.values()) >= 10, worst


# ---------------------------------------------------------------------------------------------------------------------- lm-head
LM, LV, LK = 30, 1000, 128                         # 8 column tiles, the last one 104 wide


@pytest.fixture(scope="module")
def lm_weight():
    return gr.make_lmhead_weight(LV, LK, seed=3)


def _lm_case(w, family, scale):
    h, tgt, same = gr.make_lmhead_inputs(family, w, LM, gr.lmhead_targets(LM, LV, seed=4), scale=scale, seed=5)
    gs = torch.randn(LM, generator=torch.Generator().manual_seed(6))
    return h, tgt, same, gs


@pytest.mark.parametrize("family", gr.LM_FAMILIES)
def test_lmhead_reference_matches_direct_and_autograd(lm_weight, family):
    scale = 1 / 0.6
    h, tgt, same, gs = _lm_case(lm_weight, family, scale)
    zf = (scale * (h.double() @ lm_weight.double().T)).requires_grad_(True)
    lse = torch.logsumexp(zf, 1)
    has = tgt >= 0
    logp = torch.where(has, torch.log_softmax(zf, 1).gather(1, tgt.clamp(min=0)[:, None])[:, 0], 0.0)
    (gs.double() * torch.where(has, zf.gather(1, tgt.clamp(min=0)[:, None])[:, 0], 0.0) - gs.double() * lse).sum().backward()
    r = gr.lmhead_ref(h, lm_weight, tgt, scale, lse_used=lse.detach(), gs=gs, same_sign=same)
    _close(r["lse"], lse.detach())
    _close(r["logp"], logp.detach())
    _close(r["d"], zf.grad)
    assert (r["b_logp"][~has] == 0).all() and (r["logp"][~has] == 0).all() and (r["b_logp"][has] > 0).all()


def test_lmhead_families_have_their_edges(lm_weight):
    V, lo = LV, (math.ceil(LV / gr.TILE) - 1) * gr.TILE
    for family in gr.LM_FAMILIES:
        h, tgt, same, gs = _lm_case(lm_weight, family, 1.0)
        z = h.double() @ lm_weight.double().T
        lse = torch.logsumexp(z, 1)
        top2 = z.topk(2, 1)
        if family == "zero_row":
            assert (z[::2] == 0).all()
            _close(lse[::2], torch.full_like(lse[::2], math.log(V)))
        elif family == "peaked":
            assert (top2.values[:, 0] - top2.values[:, 1] >= 30).all()
            rows = tgt >= 0
            assert (top2.indices[rows, 0] == tgt[rows]).all()
        elif family == "tail_max":
            assert (top2.values[:, 0] - top2.values[:, 1] >= 8).all() and (top2.indices[:, 0] >= lo).all()
            assert (z[:, :gr.TILE].amax(1) > z[:, gr.TILE:lo].amax(1)).double().mean() >= 0.75     # a second cluster in tile 0
            assert ((tgt == top2.indices[:, 0]).sum() >= LM // 4)
        elif family == "far_negative":
            assert ((z - lse[:, None]) < -87).double().mean() > 0.5
    assert {0, 1, V - 1, V - 2, lo, lo - 1, lo - gr.TILE} <= set(tgt.tolist()) and (tgt[::7] == -1).all()


@pytest.mark.parametrize("scale", [1.0, 1 / 0.6])
@pytest.mark.parametrize("family", gr.LM_FAMILIES)
def test_lmhead_emulation_within_bound(lm_weight, family, scale):
    h, tgt, same, gs = _lm_case(lm_weight, family, scale)
    logp, lse, d = lmhead_emul(h, lm_weight, tgt, scale, gs)
    r = gr.lmhead_ref(h, lm_weight, tgt, scale, lse_used=lse, gs=gs, same_sign=same)
    worst = {n: gr.worst_ratio(x, r[n], r["b_" + n]) for n, x in (("lse", lse), ("logp", logp), ("d", d))}
    print(f"{family} scale {scale:.3f}: " + " ".join(f"{n} {x:.3g}" for n, x in worst.items()))
    assert max(worst.values()) <= 1.0, worst


@pytest.mark.parametrize("variant", gr.LMHEAD_VARIANTS)
def test_lmhead_variants_break_the_bound(lm_weight, variant):
    scale = 1 / 0.6
    worst = {}
    for family in gr.LM_FAMILIES:
        h, tgt, same, gs = _lm_case(lm_weight, family, scale)
        _, lse, _ = lmhead_emul(h, lm_weight, tgt, scale, gs)
        r = gr.lmhead_ref(h, lm_weight, tgt, scale, lse_used=lse, gs=gs, same_sign=same)
        m = gr.lmhead_ref(h, lm_weight, tgt, scale, lse_used=lse, gs=gs, same_sign=same, variant=variant)
        worst[family] = max(gr.worst_ratio(m[n], r[n], r["b_" + n]) for n in ("lse", "logp", "d"))
    print(f"{variant}: " + " ".join(f"{f} {x:.3g}" for f, x in worst.items()))
    assert max(worst.values()) >= 10, worst


# ---------------------------------------------------------------------------------------------------------------- LoRA gradient
LORA_CASES = {   # name: (M, P, N, mode, segs, masked)
    "mode0_3seg": (1000, 136, 72, 0, [(0, 64, 0, 24), (64, 100, 24, 24), (100, 136, 48, 24)], False),
    "mode1": (1000, 136, 72, 1, [(0, 136, 0, 72)], False),
    "mode1_dropout": (1000, 136, 32, 1, [(0, 136, 0, 32)], True),
    "mode2": (1000, 144, 64, 2, [(0, 144, 0, 32), (0, 144, 32, 32)], False),
    "mode0_one_token": (1, 8, 8, 0, [(0, 8, 0, 8)], False),
}


def _lora_case(name, family):
    M, P, N, mode, segs, masked = LORA_CASES[name]
    big, small = gr.make_lora_inputs(family, M, P, N, n_sms=N_SMS, seed=M + P)
    gen = torch.Generator().manual_seed(N)
    shapes = [(N, P) if mode == 1 else (P // 2, nc) if mode == 2 else (hi - lo, nc) for lo, hi, _, nc in segs]
    prev = [torch.randn(*s, generator=gen) * 5 for s in shapes]
    mask = torch.from_numpy(keep_mask(9, 1, 4, 3, np.arange(500, 500 + M), P, T_DROP)) if masked else None
    return big, small, segs, mode, prev, mask


@pytest.mark.parametrize("name", list(LORA_CASES))
def test_lora_reference_matches_direct(name):
    big, small, segs, mode, prev, mask = _lora_case(name, "random")
    r = gr.lora_grad_ref(big, small, segs, mode, prev, mask=mask, inv_keep=INV_KEEP if mask is not None else 1.0, n_sms=N_SMS)
    x = big.double() * (mask.double() * INV_KEEP if mask is not None else 1.0)
    prod = x.T @ small.double()
    P, N = prod.shape
    for i, (lo, hi, c0, nc) in enumerate(segs):
        want = prev[i].double().clone()
        if mode == 1:
            want += prod.T
        elif mode == 2:
            for p in range(P):
                if (p // 8) % 2 == i:
                    want[(p // 16) * 8 + p % 8] += prod[p, c0:c0 + nc]
        else:
            want += prod[lo:hi, c0:c0 + nc]
        _close(r[i][0], want)


@pytest.mark.parametrize("family", gr.LORA_FAMILIES)
@pytest.mark.parametrize("name", list(LORA_CASES))
def test_lora_emulation_within_bound(name, family):
    big, small, segs, mode, prev, mask = _lora_case(name, family)
    ik = INV_KEEP if mask is not None else 1.0
    r = gr.lora_grad_ref(big, small, segs, mode, prev, mask=mask, inv_keep=ik, n_sms=N_SMS)
    em = lora_emul(big, small, segs, mode, prev, mask=mask, inv_keep=ik)
    worst = max(gr.worst_ratio(e, ref, b) for e, (ref, b) in zip(em, r))
    print(f"{name} {family}: {worst:.3g}")
    assert worst <= 1.0


def test_lora_splits_follow_the_host_rule():
    assert gr.lora_splits(1088, 8, 132) == [(128 * s, 128 * s + 128) for s in range(8)] + [(1024, 1088)]   # 7 of 16 splits get no block
    assert gr.lora_splits(4728, 6144, 132) == [(0, 2368), (2368, 4728)]                                   # qkv dB: 48 tiles, 2 splits
    assert gr.lora_splits(4728, 19456, 132) == [(0, 4728)]                                                # gate/up dB: 152 tiles > SMs
    assert gr.lora_splits(4728, 9728, 132) == [(0, 4728)]                                                 # down dA: 76 tiles, 1 split


@pytest.mark.parametrize("variant", gr.LORA_VARIANTS)
def test_lora_variants_break_the_bound(variant):
    name = "mode2" if variant == "gate_up_swapped" else "mode1"
    worst = {}
    for family in gr.LORA_FAMILIES:
        big, small, segs, mode, prev, mask = _lora_case(name, family)
        r = gr.lora_grad_ref(big, small, segs, mode, prev, n_sms=N_SMS)
        m = gr.lora_grad_ref(big, small, segs, mode, prev, n_sms=N_SMS, variant=variant)
        worst[family] = max(gr.worst_ratio(mm[0], rr[0], rr[1]) for mm, rr in zip(m, r))
    print(f"{variant}: " + " ".join(f"{f} {x:.3g}" for f, x in worst.items()))
    assert max(worst.values()) >= 10, worst
