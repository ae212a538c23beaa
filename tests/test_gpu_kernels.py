"""GPU parity tests for the C-ABI kernels (run with -m gpu on an H100)."""
import os, ctypes
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from bioreason_b200 import ops, _lib
    assert _lib.lib().br_device_ok() == 1, _lib.last_error()
    return ops


# ---------------------------------------------------------------- GRPO
@pytest.mark.parametrize("case,beta,lo,hi,use_old", [("mu1", 0.04, 0.2, 0.2, False), ("mu2", 0.04, 0.2, 0.2, True),
                                                     ("mu2_nokl", 0.0, 0.2, 0.2, True), ("mu2_asym", 0.1, 0.1, 0.3, True)])
def test_grpo_loss_golden(ops, golden, case, beta, lo, hi, use_old):
    G = golden["G"]; ref = G[case]
    dev = "cuda"
    out3, dlp = ops.grpo_loss_raw(G["lp"].to(dev), G["old"].to(dev) if use_old else None,
                                  G["ref"].to(dev) if beta > 0 else None, G["adv"].to(dev), G["mask"].to(dev), beta, lo, hi)
    out3, dlp = out3.cpu(), dlp.cpu()
    assert abs(out3[0].item() - ref["loss"].item()) <= 2e-6 * max(1, abs(ref["loss"].item()))
    assert abs(out3[2].item() - ref["clip_ratio"].item()) < 1e-6
    if beta > 0:
        assert abs(out3[1].item() - ref["kl"].item()) <= 2e-6
    torch.testing.assert_close(dlp, ref["dlp"], rtol=2e-5, atol=1e-8)


def test_grpo_loss_autograd_and_sizes(ops):
    from oracle import grpo as og
    torch.manual_seed(0)
    for B, C in [(8, 512), (1, 7), (40, 33), (64, 800)]:
        lp = -torch.rand(B, C) * 4
        old = lp + torch.randn(B, C) * 0.3
        ref = lp + torch.randn(B, C) * 0.2
        adv = torch.randn(B)
        mask = (torch.arange(C)[None] < torch.randint(1, C + 1, (B, 1))).int()
        lpc = lp.clone().requires_grad_(True)
        loss_o, kl_o, clip_o = og.grpo_loss(lpc, old, ref, adv, mask, 0.04, 0.2, 0.2)
        loss_o.backward()
        lpg = lp.cuda().requires_grad_(True)
        loss_g, out3 = ops.grpo_loss(lpg, old.cuda(), ref.cuda(), adv.cuda(), mask.cuda(), 0.04, 0.2, 0.2)
        (loss_g * 3.0).backward()
        assert abs(loss_g.item() - loss_o.item()) < 1e-5 * max(1, abs(loss_o.item()))
        assert abs(out3[1].item() - kl_o.item()) < 1e-5 and abs(out3[2].item() - clip_o.item()) < 1e-6
        torch.testing.assert_close(lpg.grad.cpu() / 3.0, lpc.grad, rtol=1e-4, atol=1e-8)


def test_advantages_and_eos_mask(ops, golden):
    from oracle import grpo as og
    F = golden["F"]
    adv = ops.grpo_advantages(F["rewards_per_func"].cuda(), F["G"]).cpu()
    torch.testing.assert_close(adv, F["advantages"], rtol=2e-5, atol=1e-6)
    torch.manual_seed(1)
    for rows, nf, G in [(8, 5, 8), (64, 1, 4), (48, 3, 16), (128, 2, 64)]:
        r = torch.randn(rows, nf)
        torch.testing.assert_close(ops.grpo_advantages(r.cuda(), G).cpu(), og.group_advantages(r, G), rtol=2e-5, atol=1e-6)
    E = golden["E"]
    eos = 1020
    assert torch.equal(ops.eos_mask(E["completion_ids"].cuda(), eos).cpu(), E["completion_mask"])
    ids = torch.randint(0, 50, (37, 129))
    assert torch.equal(ops.eos_mask(ids.cuda(), 7).cpu(), og.completion_mask_from_eos(ids, 7))
    ids = torch.randint(8, 50, (3, 5))   # no EOS at all
    assert torch.equal(ops.eos_mask(ids.cuda(), 7).cpu(), og.completion_mask_from_eos(ids, 7))


# ---------------------------------------------------------------- GEMM
def _ref_mm(a, b):
    return a.double() @ b.double().T


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (128, 256, 128), (256, 512, 256), (300, 1000, 192), (77, 136, 40),
                                   (1336, 3072, 1024), (4096, 2560, 9728), (2048, 6144, 2560), (8, 2560, 2560), (129, 24, 32)])
def test_gemm_plain(ops, M, N, K):
    torch.manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(M, K).bfloat16(); b = torch.randn(N, K).bfloat16()
    out = ops.gemm(a.cuda(), b.cuda(), out_dtype=torch.float32).cpu()
    ref = _ref_mm(a.float(), b.float())
    err = (out.double() - ref).abs().max().item()
    assert err < 1e-3 * K ** 0.5 + 1e-2, f"max err {err}"
    out16 = ops.gemm(a.cuda(), b.cuda()).cpu()
    torch.testing.assert_close(out16.float(), ref.float(), rtol=1e-2, atol=1e-2 * K ** 0.5)


def test_gemm_strided_and_tails(ops):
    torch.manual_seed(3)
    big_a = torch.randn(200, 328).bfloat16().cuda(); big_b = torch.randn(264, 328).bfloat16().cuda()
    a = big_a[:, 8:8 + 200]; b = big_b[:, 16:16 + 200]                       # lda != K
    outbuf = torch.zeros(200, 512, device="cuda", dtype=torch.bfloat16)
    out = outbuf[:, 64:64 + 264]
    ops.gemm(a, b, out=out)
    ref = _ref_mm(a.float().cpu(), b.float().cpu())
    torch.testing.assert_close(out.float().cpu(), ref.float(), rtol=1e-2, atol=0.2)
    assert outbuf[:, :64].abs().max().item() == 0 and outbuf[:, 64 + 264:].abs().max().item() == 0


def test_gemm_epilogues(ops):
    torch.manual_seed(4)
    M, N, K = 333, 512, 256
    a = torch.randn(M, K).bfloat16(); b = (torch.randn(N, K) * 0.1).bfloat16()
    bias = torch.randn(N).bfloat16(); res = torch.randn(M, N).bfloat16()
    acc = _ref_mm(a.float(), b.float()).float()
    out = ops.gemm(a.cuda(), b.cuda(), bias=bias.cuda(), residual=res.cuda(), alpha=0.5).cpu().float()
    ref = (acc * 0.5 + bias.float()).bfloat16().float() + res.float()
    torch.testing.assert_close(out, ref, rtol=1e-2, atol=3e-2)
    out = ops.gemm(a.cuda(), b.cuda(), bias=bias.float().cuda(), out_dtype=torch.float32).cpu()
    torch.testing.assert_close(out, acc + bias.float(), rtol=1e-3, atol=1e-2)
    # gated SiLU on interleaved (gate, up) column pairs + aux copy of the pre-activation
    aux = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    out = ops.gemm(a.cuda(), b.cuda(), act=1, aux_out=aux).cpu().float()
    a4 = acc.view(M, N // 16, 2, 8)
    g, u = a4[:, :, 0].reshape(M, N // 2).bfloat16().float(), a4[:, :, 1].reshape(M, N // 2).bfloat16().float()
    ref = torch.nn.functional.silu(g).bfloat16().float() * u
    torch.testing.assert_close(out, ref, rtol=2e-2, atol=2e-2)
    torch.testing.assert_close(aux.cpu().float(), acc, rtol=1e-2, atol=3e-2)
    # row scatter (projector epilogue): rows land where row_map says, -1 rows are dropped
    rm = torch.full((M,), -1, dtype=torch.int32); perm = torch.randperm(400)[:M - 20].int(); rm[:M - 20] = perm
    dst = torch.zeros(400, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm(a.cuda(), b.cuda(), bias=bias.cuda(), out=dst, row_map=rm.cuda())
    ref = torch.zeros(400, N); ref[perm.long()] = (acc + bias.float())[:M - 20]
    torch.testing.assert_close(dst.cpu().float(), ref, rtol=1e-2, atol=3e-2)
    # second K segment (LoRA delta) -- K2 = 32 < one 64-wide box
    a2 = torch.randn(M, 32).bfloat16(); b2 = torch.randn(N, 32).bfloat16()
    out = ops.gemm(a.cuda(), b.cuda(), a2=a2.cuda(), b2=b2.cuda(), out_dtype=torch.float32).cpu()
    torch.testing.assert_close(out, acc + _ref_mm(a2.float(), b2.float()).float(), rtol=1e-3, atol=2e-2)


@pytest.mark.parametrize("M,V,K", [(64, 1024, 256), (300, 4096, 512), (515, 151936, 2560)])
def test_lmhead_logprob_and_dlogits(ops, M, V, K):
    torch.manual_seed(5)
    h = torch.randn(M, K).bfloat16(); w = (torch.randn(V, K) * (3.0 / K ** 0.5)).bfloat16()
    tgt = torch.randint(0, V, (M,)); tgt[::7] = -1
    logp, lse = ops.lmhead_logprob(h.cuda(), w.cuda(), tgt.cuda())
    logits = (h.cuda().float() @ w.cuda().float().T)                     # torch fp32 checker on the same device
    ref_lse = torch.logsumexp(logits, dim=-1)
    ref_lp = torch.where(tgt.cuda() >= 0, logits.gather(1, tgt.clamp(min=0).cuda()[:, None])[:, 0] - ref_lse, torch.zeros_like(ref_lse))
    torch.testing.assert_close(lse, ref_lse, rtol=1e-4, atol=2e-3)
    torch.testing.assert_close(logp, ref_lp, rtol=1e-4, atol=3e-3)
    gs = torch.randn(M).cuda()
    d = ops.lmhead_dlogits(h.cuda(), w.cuda(), tgt.cuda(), lse, gs).float()
    onehot = torch.zeros_like(logits); rows = torch.nonzero(tgt >= 0)[:, 0].cuda(); onehot[rows, tgt.cuda()[rows]] = 1
    ref_d = gs[:, None] * (onehot - torch.softmax(logits, -1))
    torch.testing.assert_close(d, ref_d, rtol=2e-2, atol=2e-3)


# ---------------------------------------------------------------- row kernels
@pytest.mark.parametrize("M,d", [(5, 128), (300, 1024), (1000, 2560), (64, 2048), (17, 9728)])
def test_rmsnorm(ops, M, d):
    torch.manual_seed(d)
    x = (torch.randn(M, d) * 3).bfloat16(); w = (1 + 0.1 * torch.randn(d)).bfloat16()
    y, rstd = ops.rmsnorm(x.cuda(), w.cuda(), 1e-6, want_rstd=True)
    xf = x.float()
    r = torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6)
    ref = (w.float() * (xf * r).bfloat16().float()).bfloat16()                 # HF Qwen3RMSNorm rounding points
    torch.testing.assert_close(rstd.cpu(), r[:, 0], rtol=1e-5, atol=1e-6)
    diff = (y.cpu().float() - ref.float()).abs()
    assert (diff > 0).float().mean() < 0.01 and diff.max() <= 0.0625 * ref.float().abs().max()   # rare 1-ulp flips only


@pytest.mark.parametrize("M,d", [(7, 128), (1336, 1024), (33, 256)])
def test_layernorm(ops, M, d):
    torch.manual_seed(d + 1)
    x = (torch.randn(M, d) * 2 + 0.3).bfloat16(); w = (1 + 0.1 * torch.randn(d)).bfloat16(); b = (0.1 * torch.randn(d)).bfloat16()
    y = ops.layernorm(x.cuda(), w.cuda(), b.cuda(), 1e-12).cpu().float()
    ref = torch.nn.functional.layer_norm(x.float(), (d,), w.float(), b.float(), 1e-12)
    torch.testing.assert_close(y, ref, rtol=1e-2, atol=1e-2)


def _hf_rope(x, pos, theta, D):
    inv = 1.0 / (theta ** (torch.arange(0, D, 2).float() / D))
    fr = pos.float()[:, None] * inv[None]
    emb = torch.cat([fr, fr], -1)
    return emb.cos(), emb.sin()


def _rot_half(x):
    x1, x2 = x[..., : x.shape[-1] // 2], x[..., x.shape[-1] // 2:]
    return torch.cat([-x2, x1], -1)


def test_qk_rope_qwen(ops):
    torch.manual_seed(9)
    M, nq, nk, D = 50, 4, 2, 128
    qkv = torch.randn(M, (nq + 2 * nk) * D).bfloat16()
    qw = (1 + 0.1 * torch.randn(D)).bfloat16(); kw = (1 + 0.1 * torch.randn(D)).bfloat16()
    pos = torch.randint(0, 3000, (M,), dtype=torch.int32)
    out = ops.qk_rope_(qkv.clone().cuda(), nq, nk, D, pos.cuda(), 1e6, q_norm_w=qw.cuda(), k_norm_w=kw.cuda(), eps=1e-6).cpu()
    cos, sin = _hf_rope(None, pos, 1e6, D); cos, sin = cos.bfloat16(), sin.bfloat16()
    x = qkv[:, : (nq + nk) * D].view(M, nq + nk, D)
    w = torch.cat([qw[None].expand(nq, D), kw[None].expand(nk, D)])[None]
    xf = x.float()
    xn = (w.float() * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6)).bfloat16().float()).bfloat16()
    ref = (xn * cos[:, None]) + (_rot_half(xn) * sin[:, None])               # bf16 arithmetic as HF does it
    torch.testing.assert_close(out[:, : (nq + nk) * D].view(M, nq + nk, D).float(), ref.float(), rtol=2e-2, atol=3e-2)
    assert torch.equal(out[:, (nq + nk) * D:], qkv[:, (nq + nk) * D:])       # V untouched


def test_qk_rope_esm(ops):
    torch.manual_seed(10)
    M, nh, D = 40, 4, 64
    qkv = torch.randn(M, 3 * nh * D).bfloat16()
    pos = torch.arange(M, dtype=torch.int32)
    out = ops.qk_rope_(qkv.clone().cuda(), nh, nh, D, pos.cuda(), 1e4, q_scale=D ** -0.5, mode=1).cpu()
    cos, sin = _hf_rope(None, pos, 1e4, D)
    x = qkv[:, : 2 * nh * D].view(M, 2 * nh, D).clone()
    x[:, :nh] = x[:, :nh] * D ** -0.5                                          # bf16 multiply, esm/modeling_esm.py:341
    ref = (x.float() * cos[:, None] + _rot_half(x.float()) * sin[:, None]).bfloat16()
    torch.testing.assert_close(out[:, : 2 * nh * D].view(M, 2 * nh, D).float(), ref.float(), rtol=1e-2, atol=1e-2)


def test_gather_scatter(ops):
    torch.manual_seed(11)
    table = torch.randn(100, 256).bfloat16().cuda()
    ids = torch.randint(0, 100, (3, 17)).cuda()
    keep = (torch.rand(3, 17) > 0.3).int().cuda()
    out = ops.embed_gather(ids, table, keep=keep)
    ref = table[ids.reshape(-1)] * keep.reshape(-1, 1).to(table.dtype)
    assert torch.equal(out, ref)
    rm = torch.tensor([5, -1, 0, 9], dtype=torch.int32).cuda()
    dst = torch.zeros(10, 256, dtype=torch.bfloat16, device="cuda")
    ops.scatter_rows_(dst, table[:4], rm)
    assert torch.equal(dst[5], table[0]) and torch.equal(dst[0], table[2]) and torch.equal(dst[9], table[3]) and dst[1].abs().sum() == 0
    idx = torch.tensor([3, 3, 99], dtype=torch.int32).cuda()
    assert torch.equal(ops.gather_rows(table, idx), table[idx.long()])


# ---------------------------------------------------------------- attention
def _ref_attn(q, k, v, B, L, nq, nkv, D, ks, ke, scale, causal):
    qf = q.float().view(B, L, nq, D).transpose(1, 2); kf = k.float().view(B, L, nkv, D).transpose(1, 2)
    vf = v.float().view(B, L, nkv, D).transpose(1, 2)
    rep = nq // nkv
    kf = kf.repeat_interleave(rep, 1); vf = vf.repeat_interleave(rep, 1)
    s = qf @ kf.transpose(-1, -2) * scale
    j = torch.arange(L, device=q.device)
    ok = (j[None, None, None, :] >= ks[:, None, None, None]) & (j[None, None, None, :] < ke[:, None, None, None])
    if causal:
        ok = ok & (j[None, None, None, :] <= j[None, None, :, None])
    s = s.masked_fill(~ok, float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.softmax(s, -1).nan_to_num(0.0)
    o = (p @ vf).transpose(1, 2).reshape(B * L, nq * D)
    return o, lse


@pytest.mark.parametrize("B,L,nq,nkv,D,causal", [(2, 200, 4, 2, 128, True), (3, 77, 8, 2, 128, True), (2, 168, 4, 4, 64, False),
                                                 (1, 1337, 32, 8, 128, True), (4, 668, 16, 16, 64, False)])
def test_attn_fwd(ops, B, L, nq, nkv, D, causal):
    torch.manual_seed(L)
    W = (nq + 2 * nkv) * D
    qkv = torch.randn(B * L, W).bfloat16().cuda()
    q, k, v = qkv[:, : nq * D], qkv[:, nq * D: (nq + nkv) * D], qkv[:, (nq + nkv) * D:]
    ks = torch.randint(0, L // 3, (B,), dtype=torch.int32).cuda(); ke = torch.randint(2 * L // 3, L + 1, (B,), dtype=torch.int32).cuda()
    ks[0] = 0; ke[0] = L
    o, lse = ops.attn_fwd(q, k, v, B, L, nq, nkv, D, kv_start=ks, kv_end=ke, causal=causal, want_lse=True)
    ro, rlse = _ref_attn(q, k, v, B, L, nq, nkv, D, ks.long(), ke.long(), D ** -0.5, causal)
    torch.testing.assert_close(o.float(), ro, rtol=2e-2, atol=2e-2)
    fin = torch.isfinite(rlse)
    torch.testing.assert_close(lse[fin], rlse[fin], rtol=1e-3, atol=2e-3)
    assert torch.all(torch.isinf(lse[~fin]))
    assert o.float()[(~fin).transpose(1, 2).reshape(B * L, nq).repeat_interleave(D, 1)].abs().max().item() == 0 if (~fin).any() else True
