"""The rollout's decode step against float64 references with per-element error bounds (tests/decode_ref.py has the models): the skinny
GEMM on bf16 weights with its folded RMSNorm and sum-of-squares partials, the fused paged decode attention (q/k prep, KV append, shared
and private split passes, slot merge), and the helpers that fill the cache and fold the weights.  Outputs are NaN-prefilled and
strided with sentinel columns.  Every case stays within the fused attention's co-residency check (work items <= 3 per SM).  Run with
-s to see the worst err / bound of every output."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import decode_ref as dr  # noqa: E402
from test_gpu_train_kernels_fp64 import _bits, _nan_buffer  # noqa: E402

pytestmark = pytest.mark.gpu

D, THETA, EPS = 128, 1e6, 1e-6
bf = torch.bfloat16
REPORT = {}


@pytest.fixture(scope="module")
def ops():
    from bioreason_b200.build import ensure_built
    ensure_built()
    from bioreason_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def n_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _note(name, ratio):
    REPORT[name] = max(REPORT.get(name, 0.0), ratio)


def _check(name, got, ref, bound):
    got = got.to(torch.float64)
    assert torch.isfinite(got).all(), f"{name}: {int((~torch.isfinite(got)).sum())} non-finite elements"
    worst = dr.worst_ratio(got, ref, bound)
    _note(name, worst)
    assert worst <= 1.0, f"{name}: err / bound = {worst:.3g}"
    return worst


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    for k, v in sorted(REPORT.items()):
        print(f"worst err/bound  {k:40s} {v:.4f}")


# ------------------------------------------------------------------------------------------------------------------- skinny GEMM
QWEN3_4B = [(6144, 2560), (2560, 4096), (19456, 2560), (2560, 9728)]
QWEN3_1P7B = [(4096, 2048), (2048, 2048), (12288, 2048), (2048, 6144)]
LM_HEAD = [(151936, 2560), (152000, 2560)]
TAILS = [(16, 512), (144, 1024), (2576, 512), (256, 8), (512, 72), (384, 1000)]
STREAMK = [(128, 9728), (1664, 2560)]            # one tile over ~76 CTAs (> one batch of 8); 13 tiles x 40 k blocks: chunks straddle tiles
R_SET = (1, 2, 7, 8, 9, 16, 17, 31, 32)


def _strided(t, extra=64):
    """A copy of t [rows, cols] living in a wider buffer (ld = cols + extra)."""
    buf = torch.full((t.shape[0], t.shape[1] + extra), float("nan"), dtype=t.dtype, device="cuda")
    buf[:, :t.shape[1]] = t
    return buf[:, :t.shape[1]]


def _skinny_case(ops, scratch, x, w, mode, norm, seed, n_sms, variants=False):
    R, K = x.shape
    N = w.shape[0]
    g = torch.Generator(device="cuda").manual_seed(seed)
    res = _strided(torch.randn(R, N, device="cuda", generator=g).to(bf)) if mode == 1 else None
    n_part = {None: 1, "embed": 1, "mid": 7}[norm]
    ssq = None
    if norm:
        ssq = torch.rand(n_part, 32, device="cuda", generator=g) * K / n_part + 0.1        # [n, 32]: the kernel's fixed layout
    ncol = N // 2 if mode == 2 else N
    out_buf = _nan_buffer(R, ncol, seed, dtype=torch.float32 if mode == 3 else bf)
    sent = out_buf[:, ncol:].clone()
    want_ssq = mode <= 1 and seed % 2 == 0
    tiles = -(-N // 128)
    ssq_out = torch.full((tiles * 4, 32), float("nan"), device="cuda") if want_ssq else None
    ops.skinny_gemm(x, w, scratch, mode=mode, residual=res, out=out_buf[:, :ncol], sumsq_in=ssq, sumsq_in_n=n_part,
                    sumsq_out=ssq_out, eps=EPS)
    assert torch.equal(_bits(out_buf[:, ncol:]), _bits(sent)), "write past the output columns"
    got = out_buf[:, :ncol]
    kw = dict(residual=res, sumsq_in=ssq, sumsq_in_n=n_part, eps=EPS, n_sms=n_sms)
    ref, bound = dr.skinny_ref(x, w, mode, **kw)
    tag = "skinny " + ("lm_head" if N >= 151936 else f"mode {mode}")
    _check(tag, got, ref, bound)
    if want_ssq:
        sref, sb = dr.sumsq_out_ref(got, N)
        _check("skinny sumsq_out", ssq_out[:, :R], sref, sb)
    if variants:
        for v in dr.SKINNY_VARIANTS:
            if (v == "gate_up_swapped") != (mode == 2) or (v.startswith("rstd") and not norm):
                continue
            bad, _ = dr.skinny_ref(x, w, mode, variant=v, **kw)
            if torch.equal(bad, ref):
                continue                                                # no tile of this shape spans several CTAs
            r = dr.worst_ratio(got, bad, bound)
            REPORT[f"(variant {v})"] = max(REPORT.get(f"(variant {v})", 0.0), r)
            # rstd / N instead of / K scales every output by sqrt(K / N); where that is within a factor 2 of 1 (2560 x 4096: 1.26) it is
            # only ~50x the bf16-dominated bound, a larger one (128 x 9728: 8.7) shows > 1000x
            want = 10 if v == "rstd_over_n" and abs(math.sqrt(K / N) - 1) < 1 else 100
            assert r > want, (v, r)


@pytest.mark.parametrize("N,K", QWEN3_4B + QWEN3_1P7B + LM_HEAD + TAILS + STREAMK)
def test_skinny_gemm_vs_fp64(ops, n_sms, N, K):
    scratch = ops.skinny_scratch(max(N, 2 * 19456), "cuda")
    g = torch.Generator(device="cuda").manual_seed(N + K)
    w = _strided((torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).to(bf))
    big = N >= 151936
    for i, R in enumerate(R_SET if not big else (1, 8, 9, 17, 32)):
        x = _strided((torch.randn(R, K, device="cuda", generator=g)).to(bf), extra=8)
        for mode in ((3, 0) if big else (0, 1, 2, 3)):
            norm = (None, "embed", "mid")[(i + mode) % 3]
            _skinny_case(ops, scratch, x, w, mode, norm, seed=R * 131 + mode * 7 + N, n_sms=n_sms,
                         variants=(R in (8, 17) and not big))
    assert scratch.view(torch.int32)[n_sms * 32 * 128:].abs().sum().item() == 0          # arrival counters self-reset


def test_skinny_layer_chain_vs_fp64(ops, n_sms):
    """The decode layer's GEMM sequence, each GEMM checked from the exact bf16 inputs and statistics it received."""
    torch.manual_seed(7)
    R, d, F, nqkv, V = 8, 2560, 9728, 6144, 151936
    mk = lambda *s_: (torch.randn(*s_, device="cuda") * s_[-1] ** -0.5).to(bf)
    w_o, w_gu, w_down, w_qkv, w_lm = mk(d, 4096), mk(2 * F, d), mk(d, F), mk(nqkv, d), mk(V, d)
    attn = torch.randn(R, 4096, device="cuda").to(bf); h0 = torch.randn(R, d, device="cuda").to(bf)
    n_part = ((d + 127) // 128) * 4
    scratch = ops.skinny_scratch(V, "cuda")
    ssa = torch.full((n_part, 32), float("nan"), device="cuda"); ssb = ssa.clone()
    x2 = ops.skinny_gemm(attn, w_o, scratch, mode=1, residual=h0, sumsq_out=ssb)
    act = ops.skinny_gemm(x2, w_gu, scratch, mode=2, sumsq_in=ssb, sumsq_in_n=n_part, eps=EPS)
    hn = ops.skinny_gemm(act, w_down, scratch, mode=1, residual=x2, sumsq_out=ssa)
    qkv = ops.skinny_gemm(hn, w_qkv, scratch, sumsq_in=ssa, sumsq_in_n=n_part, eps=EPS)
    lg = ops.skinny_gemm(hn, w_lm, scratch, mode=3, sumsq_in=ssa, sumsq_in_n=n_part, eps=EPS)
    steps = [("o_proj", attn, w_o, 1, dict(residual=h0), x2), ("gate_up", x2, w_gu, 2, dict(sumsq_in=ssb, sumsq_in_n=n_part), act),
             ("down", act, w_down, 1, dict(residual=x2), hn), ("qkv", hn, w_qkv, 0, dict(sumsq_in=ssa, sumsq_in_n=n_part), qkv),
             ("lm_head", hn, w_lm, 3, dict(sumsq_in=ssa, sumsq_in_n=n_part), lg)]
    for name, xin, w, mode, kw, got in steps:
        ref, bound = dr.skinny_ref(xin, w, mode, eps=EPS, **kw)
        _check(f"layer chain {name}", got, ref, bound)
    for ss, y in ((ssb, x2), (ssa, hn)):
        sref, sb = dr.sumsq_out_ref(y, d)
        _check("layer chain sumsq_out", ss[:, :R], sref, sb)


# ----------------------------------------------------------------------------------------------------------- fused decode attention
def _cases(n_sms):
    """(name, Hq, Hkv, G, plen per group, cur per row, (SS, SP) or None for the rollout's own) -- all within 3 items per SM."""
    from bioreason_b200.generation import decode_splits
    cap = 3 * n_sms
    out = [("config_c", 32, 8, 8, [1852], [1852, 1852 + 63, 2363, 1852, 1852 + 63, 2363, 1852, 2000], None),
           ("gq_g_32", 16, 8, 16, [128], [128] * 16, None),
           ("two_groups", 32, 8, 4, [200, 70], [205, 263, 200, 255, 70, 127, 128, 300], None),
           ("second_tile", 32, 8, 4, [640], [832, 850, 895, 870], None),
           ("gq_1", 8, 8, 32, [128], [128 + (r % 5) for r in range(32)], None),
           ("gq_16", 32, 2, 2, [300], [300, 420], None)]
    for sp in (1, 8, 32):
        cur = [0, 63, 64, 127, 40959]
        while len(cur) * 8 * sp > cap:
            cur = cur[1:]
        out.append((f"no_sharing_sp{sp}", 32, 8, 1, list(cur), list(cur), (0, sp)))
    for ss, sp in ((16, 8), (17, 8), (28, 4)):
        if 8 * ss + 16 * sp <= cap:
            out.append((f"slots_{ss + sp}", 32, 8, 2, [1852], [2400, 2363], (ss, sp)))
    res = []
    for name, Hq, Hkv, G, plen, cur, splits in out:
        R = len(cur)
        n_sh = min(p // 64 for p in plen) if G > 1 else 0
        ss, sp = splits if splits else decode_splits(R, G, Hkv, n_sh, n_sms)
        assert (R // G) * Hkv * (ss if n_sh else 0) + R * Hkv * sp <= cap, name
        res.append((name, Hq, Hkv, G, plen, cur, ss, sp))
    return res


def _run_attn(ops, case, Hq, Hkv, G, SS, SP, rope, reps=1):
    R = case["qkv"].shape[0]
    qkv = case["qkv"].cuda()
    qkv_before = qkv.clone()
    kc, vc = case["kc"].cuda(), case["vc"].cuda()
    table, cur = case["table"].cuda(), case["cur"].cuda()
    qw, kw = case["qw"].cuda(), case["kw"].cuda()
    n_slots = (SS if case["n_shared"] else 0) + SP
    ws = ops.decode_fused_workspace(R, Hq, Hkv, D, n_slots, "cuda")
    n_f = R * Hq * n_slots * (D + 1)
    ws.view(torch.float32)[:n_f] = float("nan")                         # partials: NaN; the counters stay zero
    outs = []
    for _ in range(reps):
        buf = _nan_buffer(R, Hq * D, seed=R)
        sent = buf[:, Hq * D:].clone()
        ops.decode_attn_fused(qkv[:, :(Hq + 2 * Hkv) * D], qw, kw, kc, vc, table, cur, G, Hq, Hkv, D, case["n_shared"], SS, SP, THETA, EPS,
                              ws, buf[:, :Hq * D], rope=rope)
        assert torch.equal(_bits(buf[:, Hq * D:]), _bits(sent)), "write past the output columns"
        outs.append(buf[:, :Hq * D].clone())
    assert torch.equal(_bits(qkv), _bits(qkv_before)), "the raw projection must not change"
    return outs, kc, vc


@pytest.mark.parametrize("family", dr.FAMILIES)
def test_decode_attn_fused_vs_fp64(ops, n_sms, family):
    cases = _cases(n_sms)
    rope = ops.rope_table(40960, D, THETA, "cuda")
    risk_n = risk_tot = 0
    for name, Hq, Hkv, G, plen, cur, SS, SP in cases:
        case = dr.make_decode_case(family, plen, G, cur, Hq, Hkv, rope.cpu(), extra_width=64, seed=len(name) + len(family))
        R = len(cur)
        width = (Hq + 2 * Hkv) * D
        outs, kc, vc = _run_attn(ops, case, Hq, Hkv, G, SS, SP, rope, reps=3)
        for o in outs[1:]:
            assert torch.equal(_bits(o), _bits(outs[0])), f"{name}: repeated launches differ"
        got = outs[0]
        ref = dr.decode_step_ref(case["qkv"].cuda(), Hq, Hkv, case["qw"], case["kw"], case["kc"].cuda(), case["vc"].cuda(), case["table"],
                                 case["cur"], G, case["n_shared"], SS, SP, rope, EPS)
        _check(f"attn O ({family})", got, ref["o"], ref["b_o"])
        # K / V: the appended K is qk_rope_'s output bit for bit and within the prep allowance; V is the raw projection; nothing else moves
        rq = case["qkv"].cuda()[:, :width].clone()
        ops.qk_rope_(rq, Hq, Hkv, D, case["cur"].cuda(), THETA, q_norm_w=case["qw"].cuda(), k_norm_w=case["kw"].cuda(), eps=EPS, rope=rope)
        want_kc, want_vc = case["kc"].cuda().clone(), case["vc"].cuda().clone()
        tab = case["table"].long()
        for r in range(R):
            T = int(cur[r])
            p = int(tab[r, T // 64])
            want_kc[p, :, T % 64] = rq[r, Hq * D:(Hq + Hkv) * D].view(Hkv, D)
            want_vc[p, :, T % 64] = case["qkv"].cuda()[r, (Hq + Hkv) * D:width].view(Hkv, D)
            kn = kc[p, :, T % 64].double()
            assert ((kn - ref["k_new"][r].cuda()).abs() <= ref["k_allow"][r].cuda()).all(), f"{name}: appended K beyond the prep allowance"
        assert torch.equal(_bits(kc), _bits(want_kc)), f"{name}: K cache"
        assert torch.equal(_bits(vc), _bits(want_vc)), f"{name}: V cache"
        risk_n += int((ref["k_allow"] > 0).sum()); risk_tot += ref["k_allow"].numel()
        # the kernel against the bug variants this family exposes
        for v, fam in dr.EXPOSED_BY.items():
            if fam != family:
                continue
            bad = dr.decode_step_ref(case["qkv"].cuda(), Hq, Hkv, case["qw"], case["kw"], case["kc"].cuda(), case["vc"].cuda(), case["table"],
                                     case["cur"], G, case["n_shared"], SS, SP, rope, EPS, variant=v, bounds=False)
            if torch.equal(bad["o"], ref["o"]):
                continue                                                # the case lacks the structure (no shared pages, G = 1, ...)
            REPORT[f"(variant {v})"] = max(REPORT.get(f"(variant {v})", 0.0), dr.worst_ratio(got, bad["o"], ref["b_o"]))
    print(f"{family}: appended-K at-risk fraction {risk_n / max(risk_tot, 1):.4%}")
    for v, fam in dr.EXPOSED_BY.items():
        if fam == family:
            # doubling the weight of the shared keys moves O by at most a third of P|V|: 1 / (3 * 4u) = 21x of the bound at best
            want = 10 if v == "private_from_0" else 100
            assert REPORT.get(f"(variant {v})", 0.0) > want, (v, REPORT.get(f"(variant {v})"))


def test_decode_attn_refuses_past_coresidency(ops, n_sms):
    """One case just past 3 items per SM: the host refuses it (an argument check, before any launch)."""
    R = (3 * n_sms) // (8 * 32) + 1
    qkv = torch.zeros(R, 48 * D, dtype=bf, device="cuda")
    kc = torch.zeros(R, 8, 64, D, dtype=bf, device="cuda")
    table = torch.arange(R, dtype=torch.int32, device="cuda")[:, None]
    cur = torch.zeros(R, dtype=torch.int32, device="cuda")
    nw = torch.ones(D, dtype=bf, device="cuda")
    ws = ops.decode_fused_workspace(R, 32, 8, D, 32, "cuda")
    out = torch.empty(R, 32 * D, dtype=bf, device="cuda")
    with pytest.raises(RuntimeError, match="co-resident"):
        ops.decode_attn_fused(qkv, nw, nw, kc, kc.clone(), table, cur, 1, 32, 8, D, 0, 0, 32, THETA, EPS, ws, out,
                              rope=ops.rope_table(4, D, THETA, "cuda"))


# ----------------------------------------------------------------------------------------------------- prefill half and the helpers
@pytest.mark.parametrize("Hq,Hkv", [(32, 8), (16, 8)])
def test_qk_rope_mode0_vs_prep_ref(ops, Hq, Hkv):
    pos = torch.tensor(list(range(0, 2365)) + [4095, 4096, 40959], dtype=torch.int32)
    M = pos.numel()
    g = torch.Generator().manual_seed(Hq)
    width = (Hq + 2 * Hkv) * D
    x = (torch.randn(M, width, generator=g) * torch.rand(M, 1, generator=g) * 3).to(bf).cuda()
    qw, kw = [(1 + 0.1 * torch.randn(D, generator=g)).to(bf).cuda() for _ in range(2)]
    rope = ops.rope_table(40960, D, THETA, "cuda")
    raw = x.view(M, Hq + 2 * Hkv, D)
    yq, aq, rq = dr.qk_prep_ref(raw[:, :Hq], qw, pos, rope, EPS)
    yk, ak, rk = dr.qk_prep_ref(raw[:, Hq:Hq + Hkv], kw, pos, rope, EPS)
    for path in ("table", "inline"):
        buf = _nan_buffer(M, width, seed=3)
        buf[:, :width] = x
        sent = buf[:, width:].clone()
        ops.qk_rope_(buf[:, :width], Hq, Hkv, D, pos.cuda(), THETA, q_norm_w=qw, k_norm_w=kw, eps=EPS, rope=rope if path == "table" else None)
        got = buf[:, :width].view(M, Hq + 2 * Hkv, D).double()
        for nm, y, a in (("q", yq, aq), ("k", yk, ak)):
            sl = slice(0, Hq) if nm == "q" else slice(Hq, Hq + Hkv)
            _check(f"qk_rope_ {nm} ({path}), err / allowance", got[:, sl], y, a)
        assert torch.equal(_bits(buf[:, (Hq + Hkv) * D:]), _bits(torch.cat([x[:, (Hq + Hkv) * D:], sent], 1))), "V or sentinels changed"
    print(f"qk_rope_ {Hq}/{Hkv}: at-risk fraction q {rq.double().mean().item():.4%}, k {rk.double().mean().item():.4%}")


@pytest.mark.parametrize("n_tok", [1, 63, 64, 65, 1852])
def test_kv_write_pages_bit_exact(ops, n_tok):
    Hq, Hkv = 32, 8
    width = (Hq + 2 * Hkv) * D
    g = torch.Generator().manual_seed(n_tok)
    qkv = _strided(torch.randn(n_tok, width, generator=g).to(bf).cuda())
    n_pg = -(-n_tok // 64)
    n_pages = n_pg + 5
    pages = torch.randperm(n_pages, generator=g)[:n_pg].to(torch.int32)
    kc = torch.randn(n_pages, Hkv, 64, D, generator=g).to(bf).cuda(); vc = torch.randn(n_pages, Hkv, 64, D, generator=g).to(bf).cuda()
    want_k, want_v = kc.clone(), vc.clone()
    for t in range(n_tok):
        p = int(pages[t // 64])
        want_k[p, :, t % 64] = qkv[t, Hq * D:(Hq + Hkv) * D].view(Hkv, D)
        want_v[p, :, t % 64] = qkv[t, (Hq + Hkv) * D:].view(Hkv, D)
    ops.kv_write_pages(qkv, n_tok, Hq, Hkv, D, pages.cuda(), kc, vc)
    assert torch.equal(_bits(kc), _bits(want_k)) and torch.equal(_bits(vc), _bits(want_v))


def test_embed_gather_sumsq(ops):
    V, d = 151936, 2560
    g = torch.Generator().manual_seed(0)
    table = _strided((torch.randn(V, d, generator=g) * 0.05).to(bf).cuda())
    ids = torch.tensor([0, 1, V - 1, V, -1, 12345, 151935, -7, 2 ** 40], dtype=torch.int64)
    M = ids.numel()
    out = _nan_buffer(M, d, seed=1)
    sent = out[:, d:].clone()
    ss = torch.full((M,), float("nan"), device="cuda")
    ops.embed_gather_sumsq(ids.cuda(), table, out[:, :d], ss)
    torch.cuda.synchronize()
    ok = (ids >= 0) & (ids < V)
    want = torch.zeros(M, d, dtype=bf, device="cuda")
    want[ok.cuda()] = table[ids[ok].cuda()]
    assert torch.equal(_bits(out[:, :d]), _bits(want)) and torch.equal(_bits(out[:, d:]), _bits(sent))
    sq = (want.double() ** 2).sum(1)
    bound = dr.SAFETY * ((d / 32 + 5) * dr.E32 * sq + 2.0 ** -140)
    assert (ss[~ok.cuda()] == 0).all()
    _check("embed_gather_sumsq sumsq", ss, sq, bound)


def test_scale_columns_bit_exact(ops):
    N, K = 1000, 2560
    g = torch.Generator().manual_seed(4)
    buf = _nan_buffer(N, K, seed=5)
    W = torch.randn(N, K, generator=g).to(bf).cuda()
    buf[:, :K] = W
    sent = buf[:, K:].clone()
    s = (1 + 0.3 * torch.randn(K, generator=g)).to(bf).cuda()
    ops.scale_columns_(buf[:, :K], s)
    assert torch.equal(_bits(buf[:, :K]), _bits((W.float() * s.float()).to(bf)))
    assert torch.equal(_bits(buf[:, K:]), _bits(sent))
