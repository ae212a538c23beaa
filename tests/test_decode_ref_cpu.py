"""The float64 references of tests/decode_ref.py, without a GPU: each equals a direct formula, an fp32 emulation of each kernel stays
inside its bound, and each one-bug variant breaks the bound by at least 10x on the family that exposes it."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import decode_ref as dr  # noqa: E402

D, THETA, EPS = 128, 1e6, 1e-6
bf = torch.bfloat16


def rb(x):
    return x.float().to(bf).float()


# ------------------------------------------------------------------------------------------------------------------- skinny GEMM
def _skinny_inputs(R, N, K, seed, n_part=3):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(R, K, generator=g).to(bf)
    w = (torch.randn(N, K, generator=g) * K ** -0.5).to(bf)
    res = torch.randn(R, N, generator=g).to(bf)
    ssq = torch.rand(n_part, 32, generator=g) * K / n_part + 0.1
    return x, w, res, ssq


def _skinny_emul(x, w, mode, res, ssq, n, eps, K):
    """fp32 emulation: fp32 accumulation in k16 chunks, fp32 rstd, the epilogue's bf16 roundings."""
    R = x.shape[0]
    acc = torch.zeros(R, w.shape[0])
    for k0 in range(0, K, 16):
        acc += x[:, k0:k0 + 16].float() @ w[:, k0:k0 + 16].float().T
    rs = torch.rsqrt(ssq[:n, :R].float().sum(0) / K + eps)[:, None] if ssq is not None else torch.ones(R, 1)
    v = acc * rs
    if mode == 3:
        return v
    if mode == 0:
        return rb(v)
    if mode == 1:
        return rb(rb(v) + res.float())
    G, U = rb(v.view(R, -1, 2, 8)[:, :, 0]), rb(v.view(R, -1, 2, 8)[:, :, 1])
    return rb(rb(G / (1 + torch.exp(-G))) * U).reshape(R, -1)


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
@pytest.mark.parametrize("norm", [False, True])
def test_skinny_ref_formula_and_emulation(mode, norm):
    R, N, K = 5, 272, 200
    x, w, res, ssq = _skinny_inputs(R, N, K, seed=mode + 10 * norm)
    kw = dict(residual=res, sumsq_in=ssq if norm else None, sumsq_in_n=3, eps=EPS)
    ref, bound = dr.skinny_ref(x, w, mode, **kw)
    y = x.double() @ w.double().T
    if norm:
        y = y / torch.sqrt(ssq[:3, :R].double().sum(0) / K + EPS)[:, None]
    if mode == 1:
        y = y + res.double()
    if mode == 2:
        y = (torch.nn.functional.silu(y.view(R, -1, 2, 8)[:, :, 0]) * y.view(R, -1, 2, 8)[:, :, 1]).reshape(R, -1)
    assert (ref - y).abs().max().item() <= 1e-12 * (1 + y.abs().max().item())
    got = _skinny_emul(x, w, mode, res, ssq if norm else None, 3, EPS, K)
    assert dr.worst_ratio(got, ref, bound) <= 1.0


def test_skinny_variants_break_the_bound():
    x, w, res, ssq = _skinny_inputs(8, 256, 4096, seed=3, n_part=7)
    worst = {}
    for variant in dr.SKINNY_VARIANTS:
        mode = 2 if variant == "gate_up_swapped" else 0
        kw = dict(residual=res, sumsq_in=ssq, sumsq_in_n=7, eps=EPS, n_sms=132)
        ref, bound = dr.skinny_ref(x, w, mode, **kw)
        bad, _ = dr.skinny_ref(x, w, mode, variant=variant, **kw)
        worst[variant] = dr.worst_ratio(bad, ref, bound)
    print("skinny variants, err / bound:", {k: round(v, 1) for k, v in worst.items()})
    assert all(v >= 10 for v in worst.values()), worst


def test_streamk_plan_spans_more_than_8_contributors():
    chunk, KB = dr.streamk_plan(128, 9728, 132)                   # one tile of 152 k blocks over 132 CTAs
    assert KB == 152 and chunk == 2 and (KB - 1) // chunk + 1 > 8


def test_sumsq_out_ref():
    g = torch.Generator().manual_seed(0)
    y = torch.randn(3, 144, generator=g).to(bf)
    ref, bound = dr.sumsq_out_ref(y, 144)
    assert ref.shape == (8, 3)
    want = torch.zeros(8, 3, dtype=torch.float64)
    for f in range(144):
        want[f // 32] += y[:, f].double() ** 2
    assert torch.equal(ref[5:], torch.zeros(3, 3, dtype=torch.float64)) and (ref - want).abs().max() <= 1e-12
    sq = (y.float() ** 2)
    sq = torch.cat([sq, torch.zeros(3, 256 - 144)], 1).view(3, 8, 32)
    for step in (16, 8, 4, 2, 1):                                  # the warp tree in fp32
        sq = sq[..., :step] + sq[..., step:2 * step]
    assert dr.worst_ratio(sq[..., 0].T, ref, bound) <= 1.0


# --------------------------------------------------------------------------------------------------------------- q/k norm + RoPE
def _prep_direct(x, g, pos, rope, eps):
    """The HF rounding points written out element by element (a handful of vectors)."""
    y = torch.zeros_like(x, dtype=torch.float64)
    M, H, _ = x.shape
    for m in range(M):
        for h in range(H):
            v = x[m, h].double()
            rstd = 1.0 / math.sqrt(float((v * v).sum()) / D + eps)
            t = [dr.bf16(torch.tensor(float(v[i]) * rstd)) * float(g[i]) for i in range(D)]
            a = [float(dr.bf16(ti)) for ti in t]
            c, s = rope[int(pos[m]), :, 0].double(), rope[int(pos[m]), :, 1].double()
            c, s = [torch.tensor(float(z), dtype=torch.float64) for z in c], [torch.tensor(float(z), dtype=torch.float64) for z in s]
            for j in range(D // 2):
                p1, p2 = dr.bf16(a[j] * c[j]), dr.bf16(-a[j + 64] * s[j])
                p3, p4 = dr.bf16(a[j + 64] * c[j]), dr.bf16(a[j] * s[j])
                y[m, h, j], y[m, h, j + 64] = dr.bf16(p1 + p2), dr.bf16(p3 + p4)
    return y


def _prep_emul(x, g, pos, rope, eps):
    """fp32 emulation of the kernels (fp32 sum of squares in another order, rsqrt)."""
    xf = x.float()
    ss = (xf * xf).flip(-1).cumsum(-1)[..., -1:]
    rstd = torch.rsqrt(ss / D + eps)
    a = rb(g.float() * rb(xf * rstd))
    cs = rope[pos.long()]
    c, s = cs[..., 0][:, None], cs[..., 1][:, None]
    lo, hi = a[..., :64], a[..., 64:]
    return torch.cat([rb(rb(lo * c) + rb(-hi * s)), rb(rb(hi * c) + rb(lo * s))], -1)


def test_qk_prep_ref_formula():
    g = torch.Generator().manual_seed(1)
    rope = dr.rope_table_ref(4200, D, THETA)
    x = torch.randn(3, 2, D, generator=g).to(bf)
    w = (1 + 0.1 * torch.randn(D, generator=g)).to(bf)
    pos = torch.tensor([0, 1851, 4095])
    y, allow, risk = dr.qk_prep_ref(x, w, pos, rope, EPS)
    assert torch.equal(y, _prep_direct(x, w, pos, rope, EPS))
    assert torch.equal(allow == 0, ~risk)


def test_qk_prep_emulation_within_allowance():
    g = torch.Generator().manual_seed(2)
    rope = dr.rope_table_ref(41000, D, THETA)
    M, H = 512, 12
    x = (torch.randn(M, H, D, generator=g) * torch.rand(M, H, 1, generator=g) * 4).to(bf)
    w = (1 + 0.1 * torch.randn(D, generator=g)).to(bf)
    pos = torch.randint(0, 41000, (M,), generator=g)
    y, allow, risk = dr.qk_prep_ref(x, w, pos, rope, EPS)
    got = _prep_emul(x, w, pos, rope, EPS).double()
    frac = risk.double().mean().item()
    print(f"q/k prep: at-risk fraction {frac:.4%}, emulation differs on {(got != y).sum().item()} of {y.numel()}")
    assert frac < 0.01
    assert torch.equal(got[~risk], y[~risk])
    assert ((got - y).abs() <= allow).all()


# ----------------------------------------------------------------------------------------------------------- fused decode attention
def _emul_decode(case, Hq, Hkv, G, SS, SP, rope):
    """fp32 emulation of br_decode_attn_fused: q / k prep in fp32, the append, each slot's online softmax over its 64-key tiles (bf16
    P into the P V product), the partials (o / l, m ln2 + log l) and the slot merge with exp weights; bf16 output."""
    qkv, kc, vc, table, cur = case["qkv"], case["kc"].clone(), case["vc"].clone(), case["table"].long(), case["cur"].long()
    R, GQ = qkv.shape[0], Hq // Hkv
    raw = qkv[:, :(Hq + 2 * Hkv) * D].reshape(R, Hq + 2 * Hkv, D)
    q = _prep_emul(raw[:, :Hq], case["qw"], cur, rope, EPS)
    k = _prep_emul(raw[:, Hq:Hq + Hkv], case["kw"], cur, rope, EPS)
    for r in range(R):
        T = int(cur[r])
        kc[table[r, T // 64], :, T % 64] = k[r].to(bf)
        vc[table[r, T // 64], :, T % 64] = raw[r, Hq + Hkv:]
    n_sh, SSe = dr.decode_slots(case["n_shared"], SS, SP)
    n_slots = SSe + SP
    sl2 = D ** -0.5 * 1.4426950408889634
    out = torch.zeros(R, Hq, D)
    for r in range(R):
        T = int(cur[r])
        kv_len = T + 1
        for h in range(Hq):
            hk = h // GQ
            qv = q[r, h]
            po, pl = [], []
            for s in range(n_slots):
                pages = range(s, n_sh, SSe) if s < SSe else range(n_sh + s - SSe, -(-kv_len // 64), SP)
                m, l, o = -math.inf, 0.0, torch.zeros(D)
                for pg in pages:
                    K, V = kc[table[r, pg], hk].float(), vc[table[r, pg], hk].float()
                    sc = (K @ qv) * sl2
                    j = pg * 64 + torch.arange(64)
                    sc = torch.where(j < kv_len, sc, torch.tensor(-math.inf))
                    mn = max(m, sc.max().item())
                    p = torch.exp2(sc - mn)
                    a = 2.0 ** (m - mn) if m > -math.inf else 0.0
                    l = l * a + p.sum().item()
                    o = o * a + rb(p) @ V
                    m = mn
                po.append(o / l if l > 0 else torch.zeros(D))
                pl.append(m * math.log(2) + math.log(l) if l > 0 else -math.inf)
            lse = torch.tensor(pl)
            wts = torch.where(torch.isfinite(lse), torch.exp(lse - lse.max()), torch.tensor(0.0))
            wts = wts / wts.sum()
            out[r, h] = rb(sum(wts[s] * po[s] for s in range(n_slots)))
    return out.reshape(R, Hq * D), kc, vc


# (plen per group, G, cur per row, Hq, Hkv, SS, SP)
ATTN_CASES = [
    ([130], 2, [200, 140], 4, 2, 2, 2),          # shared pages, newest page of row 0 in the last slot, row 1 in the first private slot
    ([70], 1, [127], 4, 2, 0, 3),                # no sharing: the newest position is the last slot of a page
    ([64, 150], 2, [64, 100, 260, 151], 8, 2, 1, 2),   # two groups, n_shared = min = 1, the new token in the first private slot
]


def _case(family, plen, G, cur, Hq, Hkv, seed=0):
    rope = dr.rope_table_ref(max(cur) + 2, D, THETA)
    return dr.make_decode_case(family, plen, G, cur, Hq, Hkv, rope, seed=seed), rope


def _ref(case, Hq, Hkv, G, SS, SP, rope, variant=None):
    return dr.decode_step_ref(case["qkv"], Hq, Hkv, case["qw"], case["kw"], case["kc"], case["vc"], case["table"], case["cur"], G,
                              case["n_shared"], SS, SP, rope, EPS, variant=variant, bounds=variant is None)


@pytest.mark.parametrize("plen,G,cur,Hq,Hkv,SS,SP", ATTN_CASES)
def test_decode_ref_equals_dense_softmax(plen, G, cur, Hq, Hkv, SS, SP):
    case, rope = _case("random", plen, G, cur, Hq, Hkv)
    r = _ref(case, Hq, Hkv, G, SS, SP, rope)
    R, GQ = len(cur), Hq // Hkv
    raw = case["qkv"][:, :(Hq + 2 * Hkv) * D].reshape(R, Hq + 2 * Hkv, D)
    q, _, _ = dr.qk_prep_ref(raw[:, :Hq], case["qw"], case["cur"], rope, EPS)
    for row in range(R):
        T = int(case["cur"][row])
        Kd = torch.zeros(T + 1, Hkv, D, dtype=torch.float64); Vd = torch.zeros_like(Kd)
        for t in range(T):                                          # gathered through the table one position at a time
            p = int(case["table"][row, t // 64])
            Kd[t], Vd[t] = case["kc"][p, :, t % 64].double(), case["vc"][p, :, t % 64].double()
        Kd[T], Vd[T] = r["k_new"][row], r["v_new"][row]
        for h in range(Hq):
            P = torch.softmax(D ** -0.5 * (Kd[:, h // GQ] @ q[row, h]), 0)
            o = P @ Vd[:, h // GQ]
            assert (r["o"][row, h * D:(h + 1) * D] - o).abs().max().item() <= 1e-12


@pytest.mark.parametrize("family", dr.FAMILIES)
@pytest.mark.parametrize("plen,G,cur,Hq,Hkv,SS,SP", ATTN_CASES)
def test_decode_emulation_within_bound(family, plen, G, cur, Hq, Hkv, SS, SP):
    case, rope = _case(family, plen, G, cur, Hq, Hkv, seed=len(family))
    r = _ref(case, Hq, Hkv, G, SS, SP, rope)
    o, kc, vc = _emul_decode(case, Hq, Hkv, G, SS, SP, rope)
    ratio = dr.worst_ratio(o, r["o"], r["b_o"])
    print(f"{family} {cur}: emulated O err / bound {ratio:.3f}")
    assert ratio <= 1.0


def test_attention_variants_break_the_bound():
    worst = {v: 0.0 for v in dr.ATTN_VARIANTS}
    for plen, G, cur, Hq, Hkv, SS, SP in ATTN_CASES:
        for variant in dr.ATTN_VARIANTS:
            case, rope = _case(dr.EXPOSED_BY[variant], plen, G, cur, Hq, Hkv, seed=1)
            ref = _ref(case, Hq, Hkv, G, SS, SP, rope)
            bad = _ref(case, Hq, Hkv, G, SS, SP, rope, variant=variant)
            worst[variant] = max(worst[variant], dr.worst_ratio(bad["o"], ref["o"], ref["b_o"]))
    print("attention variants, err / bound:", {k: round(v, 1) for k, v in worst.items()})
    assert all(v >= 10 for v in worst.values()), worst
