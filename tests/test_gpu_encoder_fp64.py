"""The NT-v2 encoder's forward kernels -- bidirectional D = 64 attention, LayerNorm, the ESM rotary, the embedding gather, one encoder
layer at NT-v2-500m width through the shipped engine.encoder_forward -- and the decoder's RMSNorm forward against float64 references
with per-element error bounds (tests/encoder_ref.py, tests/attn_ref.py), at the shapes and edges where these kernels go wrong.
Outputs are NaN-prefilled and strided with sentinel columns.  Run with -s to see the worst err / bound ratio of every output."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attn_ref as ar  # noqa: E402
import encoder_ref as er  # noqa: E402
from test_gpu_train_kernels_fp64 import PAD, _bits, _check, _check_lse, _nan_buffer  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from bioreason_b200 import ops
    return ops


def _strided(x):
    """x [M, d] copied into a [M, d + PAD] buffer with a seeded tail; returns the [M, d] view."""
    buf = torch.randn(x.shape[0], x.shape[1] + PAD, generator=torch.Generator().manual_seed(x.shape[1])).to(x.dtype).to(x.device)
    buf[:, :x.shape[1]] = x
    return buf[:, :x.shape[1]]


def _report(tag, rep):
    print(f"\n{tag}: worst err/bound " + " ".join(f"{n} {x:.3f}" for n, x in rep.items()))


# ---------------------------------------------------------------------------------------------------------------- attention
# (B, L, H, kv_end per row); kv_start = 0 (right padding).  NT-v2 heads at the bench's --dna-len 668 (a 28-key tail tile), then the
# tile edges with two sequences each.  kv_end = 0 is an all-pad row.
NT_ENDS = [668, 667, 641, 640, 639, 65, 64, 1, 0]
ENC = [
    (16, 668, 16, NT_ENDS + [668, 600, 333, 128, 127, 2, 668]),
    (2, 1, 16, [1, 0]),
    (2, 63, 16, [63, 62]),
    (2, 64, 16, [64, 1]),
    (2, 65, 16, [65, 64]),
    (2, 2048, 16, [2048, 1985]),
]


def _run_attn(ops, q, k, v, windows, *, causal, scale):
    """ops.attn_fwd on one fused, strided QKV buffer into a NaN-prefilled strided O; twice, and the runs must be bit-identical."""
    B, L, Hq, D = q.shape
    Hkv = k.shape[2]
    qkv = torch.cat([q.reshape(B * L, -1), k.reshape(B * L, -1), v.reshape(B * L, -1)], 1)
    qkv = _strided(qkv)
    qo, ko, W = Hq * D, (Hq + Hkv) * D, (Hq + 2 * Hkv) * D
    ks = torch.tensor([w[0] for w in windows], dtype=torch.int32, device="cuda")
    ke = torch.tensor([w[1] for w in windows], dtype=torch.int32, device="cuda")
    runs = []
    for seed in (1, 2):
        o = _nan_buffer(B * L, qo, seed=seed)
        sentinel = o[:, qo:].clone()
        _, lse = ops.attn_fwd(qkv[:, :qo], qkv[:, qo:ko], qkv[:, ko:W], B, L, Hq, Hkv, D, kv_start=ks, kv_end=ke, scale=scale,
                              causal=causal, want_lse=True, out=o[:, :qo])
        assert torch.equal(_bits(o[:, qo:]), _bits(sentinel)), "write past the O columns"
        runs.append((o[:, :qo], lse))
    assert torch.equal(_bits(runs[0][0]), _bits(runs[1][0])) and torch.equal(_bits(runs[0][1]), _bits(runs[1][1])), \
        "attention forward not bit-reproducible"
    return runs[0]


@pytest.mark.parametrize("family", ["random", "first_key", "window_decoy"])
@pytest.mark.parametrize("B,L,H,ends", ENC, ids=lambda x: str(x).replace(" ", "") if isinstance(x, list) else None)
def test_attn_encoder_fp64(ops, B, L, H, ends, family):
    D = 64
    windows = [(0, e) for e in ends]
    q, k, v, _ = ar.make_inputs(family, B, L, H, H, windows, D=D, seed=L + B, device="cuda", causal=False)
    if L == 668:                    # as encoder_forward calls it: q already scaled by D^-0.5 (ESM scales before the rotary)
        q, scale = (q * D ** -0.5).to(torch.bfloat16), 1.0
    else:
        scale = None
    o, lse = _run_attn(ops, q, k, v, windows, causal=False, scale=scale)
    r = ar.attn_ref(q, k, v, None, windows, scale=scale, causal=False)
    rep = {}
    _check("O", o.reshape(B, L, H, D), r["o"], r["b_o"], rep)
    _check_lse(lse, r, rep)
    for b, e in enumerate(ends):
        if e == 0:
            assert (o.reshape(B, L, H, D)[b] == 0).all() and (lse[b] == math.inf).all(), "an all-pad row must give O = 0, lse = +inf"
    _report(f"attn D=64 non-causal B={B} L={L} H={H} {family}{' prescaled' if scale == 1.0 else ''}", rep)


@pytest.mark.parametrize("D,causal,family", [(64, True, "decoy"), (128, False, "window_decoy")])
def test_attn_other_branches_fp64(ops, D, causal, family):
    """The two other (head_dim, causal) instances br_attn_fwd dispatches to: D = 64 causal, D = 128 bidirectional."""
    B, L, Hq, Hkv = 3, 200, 8, 2
    windows = [(0, 200), (37, 131), (0, 0)]
    q, k, v, _ = ar.make_inputs(family, B, L, Hq, Hkv, windows, D=D, seed=D, device="cuda", causal=causal)
    o, lse = _run_attn(ops, q, k, v, windows, causal=causal, scale=None)
    r = ar.attn_ref(q, k, v, None, windows, causal=causal)
    rep = {}
    _check("O", o.reshape(B, L, Hq, D), r["o"], r["b_o"], rep)
    _check_lse(lse, r, rep)
    _report(f"attn D={D} causal={causal} {family}", rep)


# ---------------------------------------------------------------------------------------------------------------- LayerNorm
@pytest.mark.parametrize("eps", [1e-12, 1e-5])
@pytest.mark.parametrize("M", [1, 9, 4733])
@pytest.mark.parametrize("d", [128, 256, 1024, 1032, 2048])           # VEC_ITERS 1, 1, 4, 8 (a partial last vector), 8
def test_layernorm_fp64(ops, d, M, eps):
    rep = {}
    for family in er.LN_FAMILIES:
        x, w, b = er.layernorm_inputs(family, M, d, seed=d + M, device="cuda")
        xs = _strided(x)
        out = _nan_buffer(M, d, seed=5)
        prefill = out.clone()
        ops.layernorm(xs, w, b, eps, out=out[:, :d])
        assert torch.equal(_bits(out[:, d:]), _bits(prefill[:, d:])), f"{family}: write past the row"
        y = out[:, :d]
        if family == "zero":
            assert torch.equal(_bits(y), _bits(b[None].expand(M, d))), "a zero row must give y = b bit for bit"
        r = er.layernorm_ref(x, w, b, eps)
        _check(family, y, r["y"], r["b_y"], rep)
    _report(f"layernorm d={d} M={M} eps={eps:g}", rep)


@pytest.mark.parametrize("d", [2056, 1028])
def test_layernorm_refuses_bad_widths(ops, d):
    x = torch.zeros(2, d, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="layernorm"):
        ops.layernorm(x, x[0], x[0], 1e-5)


# ------------------------------------------------------------------------------------------------------------------ RMSNorm
@pytest.mark.parametrize("M", [1, 9, 4733])
@pytest.mark.parametrize("d", [128, 512, 1032, 2048, 2560, 4096, 9728, 10240])    # VEC_ITERS 1, 4, 8, 8, 16, 16, 40, 40
def test_rmsnorm_fp64(ops, d, M):
    gen = torch.Generator().manual_seed(d + M)
    x = (torch.randn(M, d, generator=gen) * 3 + 0.5).to(torch.bfloat16).cuda()
    w = (1 + 0.1 * torch.randn(d, generator=gen)).to(torch.bfloat16).cuda()
    out = _nan_buffer(M, d, seed=6)
    prefill = out.clone()
    _, rstd = ops.rmsnorm(_strided(x), w, 1e-6, out=out[:, :d], want_rstd=True)
    assert torch.equal(_bits(out[:, d:]), _bits(prefill[:, d:])), "write past the row"
    r = er.rmsnorm_ref(x, w, 1e-6)
    rep = {}
    _check("y", out[:, :d], r["y"], r["b_y"], rep)
    _check("rstd", rstd, r["rstd"], r["b_rstd"], rep)
    _report(f"rmsnorm d={d} M={M}", rep)


def test_rmsnorm_refuses_wide_rows(ops):
    x = torch.zeros(1, 10248, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="rmsnorm"):
        ops.rmsnorm(x, x[0], 1e-6)


# ------------------------------------------------------------------------------------------------------------- ESM rotary
@pytest.mark.parametrize("nh", [16, 4, 2])
def test_qk_rope_esm_fp64(ops, nh):
    D, M = 64, 2048
    pos = torch.arange(M, dtype=torch.int32, device="cuda")
    gen = torch.Generator().manual_seed(nh)
    W = 3 * nh * D
    QK = 2 * nh * D
    qkv = _strided(torch.randn(M, W, generator=gen).to(torch.bfloat16).cuda())
    before = qkv.clone()
    full = qkv.as_strided((M, W + PAD), qkv.stride())
    full_before = full.clone()
    r = er.rope_esm_ref(before, pos, nh, nh, D, D ** -0.5)
    rep = {}
    # out=: the input (and its tail) is left untouched
    out = _nan_buffer(M, QK, seed=7)
    prefill = out.clone()
    ops.qk_rope_(qkv, nh, nh, D, pos, er.ROPE_THETA, q_scale=D ** -0.5, mode=1, out=out[:, :QK])
    assert torch.equal(_bits(full), _bits(full_before)), "out= must leave the input untouched"
    assert torch.equal(_bits(out[:, QK:]), _bits(prefill[:, QK:])), "write past the q | k columns of out"
    _check("out=", out[:, :QK].reshape(M, 2 * nh, D), r["y"], r["b_y"], rep)
    # in place: the V columns and the tail come back bit-unchanged, q | k equal the out= result
    ops.qk_rope_(qkv, nh, nh, D, pos, er.ROPE_THETA, q_scale=D ** -0.5, mode=1)
    assert torch.equal(_bits(full[:, QK:]), _bits(full_before[:, QK:])), "the V and sentinel columns must come back untouched"
    assert torch.equal(_bits(qkv[:, :QK]), _bits(out[:, :QK]))
    _check("in place", qkv[:, :QK].reshape(M, 2 * nh, D), r["y"], r["b_y"], rep)
    _report(f"qk_rope mode 1 heads {nh}/{nh}", rep)


# ----------------------------------------------------------------------------------------------------------- embedding gather
def test_embed_gather_exact(ops):
    vocab, d, M = 4107, 1024, 700
    gen = torch.Generator().manual_seed(8)
    table = _strided(torch.randn(vocab, d, generator=gen).to(torch.bfloat16).cuda())
    ids = torch.randint(0, vocab, (M,), generator=gen)
    ids[:6] = torch.tensor([-1, vocab, vocab + 5, 0, vocab - 1, 1])
    keep = (torch.rand(M, generator=gen) > 0.2).to(torch.int32)
    keep[:6] = 1
    ids, keep = ids.cuda(), keep.cuda()
    out = _nan_buffer(M, d, seed=9)
    prefill = out.clone()
    ops.embed_gather(ids, table, keep=keep, out=out[:, :d])
    assert torch.equal(_bits(out[:, d:]), _bits(prefill[:, d:])), "write past the row"
    valid = (ids >= 0) & (ids < vocab) & (keep != 0)
    ref = torch.where(valid[:, None], table[ids.clamp(0, vocab - 1)], torch.zeros((), dtype=torch.bfloat16, device="cuda"))
    assert torch.equal(_bits(out[:, :d]), _bits(ref)), "embed_gather must equal table[ids] * keep, and +0 rows for ids outside [0, vocab)"
    assert (out[:3, :d] == 0).all()


# ------------------------------------------------------------------------------------------------ encoder layers, NT-v2-500m
def test_encoder_layer_chain_fp64(ops):
    """Two NT-v2-500m layers launched step by step as engine.encoder_forward launches them, each step checked from the bf16 tensor it
    received; encoder_forward itself must give the same bits, so the check covers the shipped path."""
    from bioreason_b200 import engine
    from bioreason_b200.configs import dna_config
    from bioreason_b200.packing import pack_encoder
    from oracle.models import build_dna_model
    cfg = dna_config("nt-v2-500m")
    cfg.num_hidden_layers = 2
    W = pack_encoder(build_dna_model(cfg), "cuda")
    nh, d, eps = cfg.num_attention_heads, cfg.hidden_size, cfg.layer_norm_eps
    D = d // nh
    n, S = 4, 668
    lens = [668, 600, 65, 1]
    gen = torch.Generator().manual_seed(12)
    mask = (torch.arange(S)[None] < torch.tensor(lens)[:, None]).to(torch.int64)
    ids = torch.where(mask.bool(), torch.randint(4, cfg.vocab_size, (n, S), generator=gen), cfg.pad_token_id)
    ids, mask = ids.cuda(), mask.cuda()
    windows = [(0, m) for m in lens]

    x = ops.embed_gather(ids, W.embed, keep=mask)
    assert torch.equal(_bits(x), _bits(torch.where(mask.reshape(-1, 1).bool(), W.embed[ids.reshape(-1)], torch.zeros((), dtype=torch.bfloat16, device="cuda"))))
    ks, ke = engine.mask_window(mask)
    pos = torch.arange(S, device="cuda", dtype=torch.int32).repeat(n)
    for li, Lw in enumerate(W.layers):
        got = {"ln1": ops.layernorm(x, Lw.ln1_w, Lw.ln1_b, eps)}
        qkv = ops.gemm(got["ln1"], Lw.w_qkv, bias=Lw.b_qkv)
        got["qkv"] = qkv.clone()
        ops.qk_rope_(qkv, nh, nh, D, pos, 10000.0, q_scale=D ** -0.5, mode=1)
        got["rope"] = qkv[:, :2 * d]
        got["attn"] = ops.attn_fwd(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], n, S, nh, nh, D, kv_start=ks, kv_end=ke, scale=1.0,
                                   causal=False)
        got["o"] = ops.gemm(got["attn"], Lw.w_o, bias=Lw.b_o, residual=x)
        got["ln2"] = ops.layernorm(got["o"], Lw.ln2_w, Lw.ln2_b, eps)
        got["gu"] = ops.gemm(got["ln2"], Lw.w_gu, bias=Lw.b_gu, act=1)
        got["down"] = ops.gemm(got["gu"], Lw.w_down, bias=Lw.b_down, residual=got["o"])
        refs = er.encoder_layer(x, Lw, n, S, nh, windows, eps, got=got)
        rep = {}
        for step in er.STEPS:
            _check(step, got[step], *refs[step], rep)
        del refs
        _report(f"encoder layer {li}", rep)
        x = got["down"]
    final = ops.layernorm(x, W.final_ln_w, W.final_ln_b, eps)
    r = er.layernorm_ref(x, W.final_ln_w, W.final_ln_b, eps)
    rep = {}
    _check("final_ln", final, r["y"], r["b_y"], rep)
    _report("encoder final LayerNorm", rep)
    shipped = engine.encoder_forward(W, ids, mask)
    assert torch.equal(_bits(shipped), _bits(final)), "engine.encoder_forward differs from the step chain"
