"""The encoder references and their bounds (tests/encoder_ref.py, the causal=False mode of tests/attn_ref.py), checked without a GPU:
one reference encoder layer equals HF's EsmLayer in float64, a CPU emulation of each kernel's rounding points (bf16 storage, fp32
math) stays inside its bound at the GPU test's shapes, and a reference carrying one typical kernel bug breaks the bound by a stated
factor, so the GPU tests built on them would catch that bug."""
import math
import os
import sys
from types import SimpleNamespace

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attn_ref as ar  # noqa: E402
import encoder_ref as er  # noqa: E402

BF = torch.bfloat16


# ------------------------------------------------------------------------------------------------------------ HF EsmLayer parity
def _kernel_layout(layer, dtype=torch.float64):
    """The weights of one HF EsmLayer (NT-v2 patched) in packing.pack_encoder's layout, without moving the model's parameters."""
    from bioreason_b200.packing import gu_views
    sa, inter = layer.attention.self, layer.intermediate.dense
    F = inter.weight.shape[0] // 2
    c = lambda t: None if t is None else t.detach().to(dtype).clone()
    w_gu = torch.empty(2 * F, inter.weight.shape[1], dtype=dtype)
    gv, uv = gu_views(w_gu)
    gv.copy_(inter.weight[:F].detach().view(F // 8, 8, -1))
    uv.copy_(inter.weight[F:].detach().view(F // 8, 8, -1))
    return SimpleNamespace(
        ln1_w=c(layer.attention.LayerNorm.weight), ln1_b=c(layer.attention.LayerNorm.bias),
        ln2_w=c(layer.LayerNorm.weight), ln2_b=c(layer.LayerNorm.bias),
        w_qkv=torch.cat([c(sa.query.weight), c(sa.key.weight), c(sa.value.weight)]),
        b_qkv=torch.cat([c(sa.query.bias), c(sa.key.bias), c(sa.value.bias)]),
        w_o=c(layer.attention.output.dense.weight), b_o=c(layer.attention.output.dense.bias),
        w_gu=w_gu, b_gu=None, w_down=c(layer.output.dense.weight), b_down=c(layer.output.dense.bias))


def test_encoder_layer_matches_hf_esm_layer():
    """Pins the semantics the kernels claim: q scaled before the rotary, rotate-half pairs, key-only masking (pad queries still
    attend), SiLU on the first half of the gated FFN, biased LayerNorm variance.  Valid rows only: HF's pad rows are not used."""
    from bioreason_b200.configs import dna_config
    from oracle.models import build_dna_model
    cfg = dna_config("small")
    cfg._attn_implementation = "eager"
    model = build_dna_model(cfg).double()
    layer = model.esm.encoder.layer[1]
    nh, d = cfg.num_attention_heads, cfg.hidden_size
    D = d // nh
    # exact angles: HF computes inv_freq in fp32, the reference in fp64
    layer.attention.self.rotary_embeddings.inv_freq = er.ROPE_THETA ** (-torch.arange(0, D, 2, dtype=torch.float64) / D)
    B, S = 3, 70
    lens = [70, 41, 1]
    gen = torch.Generator().manual_seed(0)
    x = torch.randn(B, S, d, generator=gen, dtype=torch.float64) * 0.5 + 0.1
    mask = (torch.arange(S)[None] < torch.tensor(lens)[:, None])
    add = torch.zeros(B, 1, 1, S, dtype=torch.float64).masked_fill(~mask[:, None, None], torch.finfo(torch.float64).min)
    with torch.no_grad():
        want = layer(x, attention_mask=add)
    want = want[0] if isinstance(want, tuple) else want
    got = er.encoder_layer(x.reshape(B * S, d), _kernel_layout(layer), B, S, nh, [(0, n) for n in lens], cfg.layer_norm_eps)
    got = got["down"][0].view(B, S, d)
    for b, n in enumerate(lens):
        torch.testing.assert_close(got[b, :n], want[b, :n], rtol=1e-10, atol=1e-10)


# ---------------------------------------------------------------------------------------------- CPU emulation of the kernels
def _row_sum32(t):
    """fp32 row sums of t [M, d] in the row kernels' order: lane l adds the elements of its vectors l, l + 32, ... one by one, then
    a 5-step xor butterfly (br::warp_sum)."""
    M, d = t.shape
    nv = d // 8
    iters = -(-nv // 32)
    tp = torch.zeros(M, iters * 32, 8, dtype=torch.float32)
    tp[:, :nv] = t.reshape(M, nv, 8)
    tp = tp.view(M, iters, 32, 8)
    s = torch.zeros(M, 32, dtype=torch.float32)
    for i in range(iters):
        for j in range(8):
            s = s + tp[:, i, :, j]
    lanes = torch.arange(32)
    for off in (16, 8, 4, 2, 1):
        s = s + s[:, lanes ^ off]
    return s[:, 0]


def _layernorm32(x, w, b, eps):
    xf = x.float()
    mean = _row_sum32(xf) / x.shape[1]
    t = xf - mean[:, None]
    r = torch.rsqrt(_row_sum32(t * t) / x.shape[1] + eps)
    return (t * r[:, None] * w.float() + b.float()).to(BF)


def _rmsnorm32(x, w, eps):
    xf = x.float()
    r = torch.rsqrt(_row_sum32(xf * xf) / x.shape[1] + eps)
    return (w.float() * (xf * r[:, None]).to(BF).float()).to(BF), r


def _rope32(qk, pos, n_q, n_k, D, q_scale):
    M = qk.shape[0]
    x = qk[:, :(n_q + n_k) * D].view(M, n_q + n_k, D).float()
    j = torch.arange(D // 2, dtype=torch.float32)
    inv = 1.0 / torch.pow(torch.tensor(er.ROPE_THETA, dtype=torch.float32), 2 * j / D)
    ang = pos.float()[:, None] * inv[None]
    c, s = ang.cos()[:, None], ang.sin()[:, None]
    sc = torch.tensor([q_scale] * n_q + [1.0] * n_k, dtype=torch.float32)[None, :, None]
    a = (x * sc).to(BF).float()
    lo, hi = a[..., :D // 2], a[..., D // 2:]
    return torch.cat([lo * c - hi * s, hi * c + lo * s], -1).to(BF)


def _attn32(q, k, v, windows, scale):
    """Bidirectional flash forward as attn_fwd_tc5 computes it: fp32 scores, running maximum in the log2 domain over 64-key tiles,
    P rounded to bf16 for P V, fp32 accumulators; O rounded to bf16, lse = m ln 2 + log l."""
    B, L, H, D = q.shape
    o = torch.zeros(B, L, H, D, dtype=BF)
    lse = torch.full((B, H, L), math.inf)
    sl2 = torch.tensor(scale * 1.4426950408889634, dtype=torch.float32)
    for b in range(B):
        ks, ke = windows[b]
        if ke <= ks:
            continue
        for h in range(H):
            S = q[b, :, h].float() @ k[b, :, h].float().T
            m = torch.full((L,), -math.inf)
            l = torch.zeros(L)
            acc = torch.zeros(L, D)
            for t0 in range((ks // 64) * 64, ke, 64):
                j = torch.arange(t0, min(t0 + 64, L))
                st = S[:, j].masked_fill(((j < ks) | (j >= ke))[None], -math.inf)
                m_new = torch.maximum(m, st.amax(1) * sl2)
                alpha = torch.where(torch.isinf(m), 0.0, torch.exp2(m - m_new))
                p = torch.exp2(st * sl2 - m_new[:, None])
                l = l * alpha + p.sum(1)
                acc = acc * alpha[:, None] + p.to(BF).float() @ v[b, j, h].float()
                m = m_new
            o[b, :, h] = (acc / l[:, None]).to(BF)
            lse[b, h] = m * 0.6931471805599453 + torch.log(l)
    return o, lse


LN_D = [128, 256, 1024, 1032, 2048]
@pytest.mark.parametrize("family", er.LN_FAMILIES)
@pytest.mark.parametrize("eps", [1e-12, 1e-5])
def test_layernorm_emulation_within_bound(family, eps):
    for d in LN_D:
        x, w, b = er.layernorm_inputs(family, 9, d, seed=d)
        r = er.layernorm_ref(x, w, b, eps)
        worst = ar.worst_ratio(_layernorm32(x, w, b, eps), r["y"], r["b_y"])
        assert worst <= 1.0, (d, worst)
        ref_torch = torch.nn.functional.layer_norm(x.double(), (d,), w.double(), b.double(), eps)
        torch.testing.assert_close(r["y"], ref_torch, rtol=1e-12, atol=1e-12)


RMS_D = [128, 512, 1032, 2048, 2560, 4096, 9728, 10240]


@pytest.mark.parametrize("d", RMS_D)
def test_rmsnorm_emulation_within_bound(d):
    gen = torch.Generator().manual_seed(d)
    x = (torch.randn(9, d, generator=gen) * 3).to(BF)
    w = (1 + 0.1 * torch.randn(d, generator=gen)).to(BF)
    r = er.rmsnorm_ref(x, w, 1e-6)
    y, rstd = _rmsnorm32(x, w, 1e-6)
    assert ar.worst_ratio(y, r["y"], r["b_y"]) <= 1.0
    assert ar.worst_ratio(rstd, r["rstd"], r["b_rstd"]) <= 1.0


def test_rope_emulation_within_bound():
    gen = torch.Generator().manual_seed(1)
    nh, D = 4, 64
    pos = torch.arange(2048, dtype=torch.int32)
    qkv = torch.randn(2048, 3 * nh * D, generator=gen).to(BF)
    r = er.rope_esm_ref(qkv, pos, nh, nh, D, D ** -0.5)
    got = _rope32(qkv, pos, nh, nh, D, D ** -0.5)
    assert ar.worst_ratio(got, r["y"], r["b_y"]) <= 1.0


# the GPU test's NT-v2 row edges, at 4 heads
ENC_L = 668
ENC_WINDOWS = [(0, 668), (0, 641), (0, 640), (0, 65), (0, 1), (0, 0)]


@pytest.mark.parametrize("family", ["random", "first_key", "window_decoy"])
def test_noncausal_attention_emulation_within_bound(family):
    H, D = 4, 64
    B = len(ENC_WINDOWS)
    q, k, v, _ = ar.make_inputs(family, B, ENC_L, H, H, ENC_WINDOWS, D=D, seed=3, causal=False)
    qs = (q * D ** -0.5).to(BF)                                     # encoder_forward's pre-scaled q, attention at scale 1
    r = ar.attn_ref(qs, k, v, None, ENC_WINDOWS, scale=1.0, causal=False)
    o, lse = _attn32(qs, k, v, ENC_WINDOWS, 1.0)
    assert ar.worst_ratio(o, r["o"], r["b_o"]) <= 1.0
    fin = torch.isfinite(r["lse"])
    assert torch.equal(torch.isfinite(lse), fin)
    assert ar.worst_ratio(lse[fin], r["lse"][fin], r["b_lse"][fin]) <= 1.0
    assert (o[-1] == 0).all()                                        # the all-pad row


# -------------------------------------------------------------------------------------------------------------------- mutants
MUT_THRESHOLD = 10.0


def _variant_ratio(variant):
    """(worst err / bound of the variant against the correct reference, label) at a shape where the bug is live."""
    gen = torch.Generator().manual_seed(11)
    if variant.startswith("ln_"):
        x, w, b = er.layernorm_inputs("normal", 16, 1032, seed=5)               # 1032: the tail vector is live
        r = er.layernorm_ref(x, w, b, 1e-12)
        m = er.layernorm_ref(x, w, b, 1e-12, variant=variant)
        return ar.worst_ratio(m["y"], r["y"], r["b_y"])
    if variant.startswith("rope_"):
        nh, D = 4, 64
        pos = torch.arange(700, dtype=torch.int32)
        qkv = torch.randn(700, 3 * nh * D, generator=gen).to(BF)
        r = er.rope_esm_ref(qkv, pos, nh, nh, D, D ** -0.5)
        m = er.rope_esm_ref(qkv, pos, nh, nh, D, D ** -0.5, variant=variant)
        return ar.worst_ratio(m["y"], r["y"], r["b_y"])
    x = (torch.randn(16, 1024, generator=gen) * 3).to(BF)
    w = (1 + 0.1 * torch.randn(1024, generator=gen)).to(BF)
    r = er.rmsnorm_ref(x, w, 1e-6)
    m = er.rmsnorm_ref(x, w, 1e-6, variant=variant)
    return max(ar.worst_ratio(m["y"], r["y"], r["b_y"]), ar.worst_ratio(m["rstd"], r["rstd"], r["b_rstd"]))


@pytest.mark.parametrize("variant", er.VARIANTS)
def test_encoder_mutants_break_the_bound(variant):
    worst = _variant_ratio(variant)
    print(f"{variant}: worst err/bound {worst:.3g}")
    assert worst >= MUT_THRESHOLD, worst


NC_B, NC_L, NC_H = 4, 300, 4
NC_WINDOWS = [(0, 300), (0, 250), (37, 250), (0, 131)]          # a full row, ragged tails off the tile grid, a left edge


@pytest.fixture(scope="module", params=["first_key", "window_decoy"])
def nc_family_ref(request):
    q, k, v, _ = ar.make_inputs(request.param, NC_B, NC_L, NC_H, NC_H, NC_WINDOWS, D=64, seed=7, causal=False)
    return request.param, (q, k, v), ar.attn_ref(q, k, v, None, NC_WINDOWS, causal=False)


def test_noncausal_reference_is_within_its_own_bound(nc_family_ref):
    family, (q, k, v), r = nc_family_ref
    m = ar.attn_ref(q, k, v, None, NC_WINDOWS, variant="online", bounds=False, causal=False)
    worst = max(ar.worst_ratio(m[n], r[n], r["b_" + n]) for n in ("o", "lse"))
    assert worst < 1e-6, worst


@pytest.mark.parametrize("variant", ar.NONCAUSAL_VARIANTS)
def test_noncausal_mutants_break_the_bound(nc_family_ref, variant):
    """Each one-bug variant exceeds the O / lse bound by >= 10x.  On first_key the row maximum sits in the first key tile, so a
    skipped rescale is invisible there by construction; window_decoy puts it in the last tile and catches it."""
    family, (q, k, v), r = nc_family_ref
    m = ar.attn_ref(q, k, v, None, NC_WINDOWS, variant=variant, bounds=False, causal=False)
    worst = {n: ar.worst_ratio(m[n], r[n], r["b_" + n]) for n in ("o", "lse")}
    print(f"{family} {variant}: " + " ".join(f"{n} {x:.3g}" for n, x in worst.items()))
    if family == "first_key" and variant == "no_rescale":
        assert max(worst.values()) < 1e-6
        return
    assert max(worst.values()) >= MUT_THRESHOLD, worst
