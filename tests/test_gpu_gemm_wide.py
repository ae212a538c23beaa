"""The 128 x 256 GEMM tile (chosen for N >= 256, K >= 512 and two waves of 256-wide tiles) against fp64 references, and bit for
bit against the 128 x 128 tile: the same rows computed in chunks too small for the wide tile must give identical outputs."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from bioreason_b200 import ops, _lib
    assert _lib.lib().br_device_ok() == 1, _lib.last_error()
    return ops


def _n_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _is_wide(M, N, K):
    return N >= 256 and K >= 512 and ((M + 127) // 128) * ((N + 255) // 256) >= 2 * _n_sms()


def _randn(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * scale).bfloat16()


def _ref_mm(a, b):
    return a.double() @ b.double().T


NARROW_ROWS = 384           # 3 row tiles: fewer than two waves of 256-wide tiles for every N up to 19 456


def _chunked(fn, M, N, K):
    """fn(i0, i1) computes rows [i0, i1) into the caller's output, in chunks that run on 128-wide tiles."""
    assert not _is_wide(NARROW_ROWS, N, K)
    for i0 in range(0, M, NARROW_ROWS):
        fn(i0, min(M, i0 + NARROW_ROWS))


# M = 9456 is the trainer's 4-row dense chunk of config (c), 6368 the shared-prefix buffer; N = 1000 leaves a 232-column tail tile
SHAPES = [(9456, 2560, 2560), (9456, 6144, 2560), (9456, 2560, 4096), (9456, 2560, 9728), (6368, 19456, 2560), (9456, 1000, 2560),
          (300, 1000, 192), (9456, 2560, 256)]


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_plain_wide(ops, M, N, K):
    a = _randn((M, K), M + N + K); b = _randn((N, K), 7 * K + N)
    ref = _ref_mm(a, b)
    out = ops.gemm(a, b, out_dtype=torch.float32)
    err = (out.double() - ref).abs().max().item()
    assert err < 1e-3 * K ** 0.5 + 1e-2, f"max err {err}"
    out16 = ops.gemm(a, b)
    torch.testing.assert_close(out16.float(), ref.float(), rtol=1e-2, atol=1e-2 * K ** 0.5)
    if _is_wide(M, N, K):
        narrow = torch.empty_like(out)
        _chunked(lambda i0, i1: ops.gemm(a[i0:i1], b, out=narrow[i0:i1]), M, N, K)
        assert torch.equal(out, narrow)
        for _ in range(3):
            assert torch.equal(ops.gemm(a, b, out_dtype=torch.float32), out)


@pytest.mark.parametrize("M,N,K", [(9456, 2560, 4096), (9456, 6144, 2560), (6368, 19456, 2560), (333, 512, 256)])
def test_gemm_epilogues_wide(ops, M, N, K):
    wide = _is_wide(M, N, K)
    a = _randn((M, K), 4 + K); b = _randn((N, K), 5 + N, 0.1)
    bias = _randn((N,), 6); res = _randn((M, N), 7)
    acc = _ref_mm(a, b).float()

    def check_narrow(full, run):
        """`run(i0, i1, out)` writes rows [i0, i1) of the same product into out; the row chunks run 128-wide."""
        if not wide:
            return
        got = torch.empty_like(full)
        _chunked(lambda i0, i1: run(i0, i1, got[i0:i1]), M, N, K)
        assert torch.equal(full, got)
        for _ in range(3):
            again = torch.empty_like(full)
            run(0, M, again)
            assert torch.equal(full, again)

    # bias (bf16) + residual + alpha, bf16 out
    out = ops.gemm(a, b, bias=bias, residual=res, alpha=0.5)
    ref = (acc * 0.5 + bias.float()).bfloat16().float() + res.float()
    torch.testing.assert_close(out.float(), ref, rtol=1e-2, atol=3e-2)
    check_narrow(out, lambda i0, i1, o: ops.gemm(a[i0:i1], b, bias=bias, residual=res[i0:i1], alpha=0.5, out=o))
    # fp32 bias, fp32 out
    out = ops.gemm(a, b, bias=bias.float(), out_dtype=torch.float32)
    torch.testing.assert_close(out, acc + bias.float(), rtol=1e-3, atol=1e-2)
    check_narrow(out, lambda i0, i1, o: ops.gemm(a[i0:i1], b, bias=bias.float(), out=o))
    # gated SiLU on interleaved (gate, up) column blocks + aux copy of the pre-activation
    aux = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    out = ops.gemm(a, b, act=1, aux_out=aux)
    a4 = acc.view(M, N // 16, 2, 8)
    g, u = a4[:, :, 0].reshape(M, N // 2).bfloat16().float(), a4[:, :, 1].reshape(M, N // 2).bfloat16().float()
    torch.testing.assert_close(out.float(), torch.nn.functional.silu(g).bfloat16().float() * u, rtol=2e-2, atol=2e-2)
    torch.testing.assert_close(aux.float(), acc, rtol=1e-2, atol=3e-2)
    aux2 = torch.empty_like(aux)
    check_narrow(out, lambda i0, i1, o: ops.gemm(a[i0:i1], b, act=1, aux_out=aux2[i0:i1], out=o))
    if wide:
        assert torch.equal(aux, aux2)
    # row scatter (projector epilogue): rows land where row_map says, -1 rows are dropped
    g_ = torch.Generator().manual_seed(M)
    rm = torch.full((M,), -1, dtype=torch.int32); perm = torch.randperm(M + 80, generator=g_)[:M - 20].int(); rm[:M - 20] = perm
    rm = rm.cuda()
    dst = torch.zeros(M + 80, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm(a, b, bias=bias, out=dst, row_map=rm)
    ref = torch.zeros(M + 80, N, device="cuda"); ref[perm.long().cuda()] = (acc + bias.float())[:M - 20]
    torch.testing.assert_close(dst.float(), ref, rtol=1e-2, atol=3e-2)
    if wide:
        dst2 = torch.zeros_like(dst)
        _chunked(lambda i0, i1: ops.gemm(a[i0:i1], b, bias=bias, out=dst2, row_map=rm[i0:i1]), M, N, K)
        assert torch.equal(dst, dst2)
    # second K segment (LoRA delta): K2 = 32 (less than one 64-wide box) and K2 = 96 (three projections of r = 32)
    for K2 in (32, 96):
        a2 = _randn((M, K2), 8 + K2); b2 = _randn((N, K2), 9 + K2)
        out = ops.gemm(a, b, a2=a2, b2=b2, out_dtype=torch.float32)
        torch.testing.assert_close(out, acc + _ref_mm(a2, b2).float(), rtol=1e-3, atol=2e-2)
        check_narrow(out, lambda i0, i1, o: ops.gemm(a[i0:i1], b, a2=a2[i0:i1], b2=b2, out=o))


# V = 151 936 (Qwen3) ends on a 256-wide tile with one 128-column half; V = 152 000 ends on a half 64 columns wide
@pytest.mark.parametrize("M,V", [(2048, 151936), (1000, 152000)])
def test_lmhead_wide(ops, M, V):
    K = 2560
    assert _is_wide(M, V, K)
    h = _randn((M, K), 10); w = _randn((V, K), 11, 3.0 / K ** 0.5)
    g_ = torch.Generator().manual_seed(M)
    tgt = torch.randint(0, V, (M,), generator=g_); tgt[::7] = -1; tgt[1] = V - 1; tgt[2] = V - 2
    tgt = tgt.cuda()
    logp, lse = ops.lmhead_logprob(h, w, tgt)
    logits = h.float() @ w.float().T
    ref_lse = torch.logsumexp(logits, dim=-1)
    ref_lp = torch.where(tgt >= 0, logits.gather(1, tgt.clamp(min=0)[:, None])[:, 0] - ref_lse, torch.zeros_like(ref_lse))
    torch.testing.assert_close(lse, ref_lse, rtol=1e-4, atol=2e-3)
    torch.testing.assert_close(logp, ref_lp, rtol=1e-4, atol=3e-3)
    gs = torch.randn(M, device="cuda")
    d = ops.lmhead_dlogits(h, w, tgt, lse, gs)
    onehot = torch.zeros_like(logits); rows = torch.nonzero(tgt >= 0)[:, 0]; onehot[rows, tgt[rows]] = 1
    torch.testing.assert_close(d.float(), gs[:, None] * (onehot - torch.softmax(logits, -1)), rtol=2e-2, atol=2e-3)
    del logits, onehot
    for _ in range(3):
        lp2, lse2 = ops.lmhead_logprob(h, w, tgt)
        assert torch.equal(lp2, logp) and torch.equal(lse2, lse)
        assert torch.equal(ops.lmhead_dlogits(h, w, tgt, lse, gs), d)
