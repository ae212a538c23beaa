"""GPU parity tests for the backward kernels and the end-to-end LoRA / projector gradients."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from bioreason_b200 import ops
    return ops


def _rel(a, b):
    return (a.float() - b.float()).norm().item() / (b.float().norm().item() + 1e-12)


def test_rmsnorm_bwd(ops):
    torch.manual_seed(0)
    for M, d in [(100, 256), (777, 2560), (64, 2048)]:
        x = (torch.randn(M, d) * 2).bfloat16().cuda(); w = (1 + 0.1 * torch.randn(d)).bfloat16().cuda()
        dy = torch.randn(M, d).bfloat16().cuda(); dres = torch.randn(M, d).bfloat16().cuda()
        xr = x.float().requires_grad_(True)
        y = w.float() * (xr * torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + 1e-6))
        y.backward(dy.float())
        _, rstd = ops.rmsnorm(x, w, 1e-6, want_rstd=True)
        dx = ops.rmsnorm_bwd(x, w, rstd, dy, dres=dres)
        assert _rel(dx, xr.grad + dres.float()) < 6e-3
        assert _rel(ops.rmsnorm_bwd(x, w, rstd, dy), xr.grad) < 6e-3


def test_swiglu_bwd(ops):
    torch.manual_seed(1)
    M, F = 300, 1536
    gu = torch.randn(M, 2 * F).bfloat16().cuda(); dact = torch.randn(M, F).bfloat16().cuda()
    g4 = gu.float().view(M, F // 8, 2, 8)
    g = g4[:, :, 0].reshape(M, F).clone().requires_grad_(True); u = g4[:, :, 1].reshape(M, F).clone().requires_grad_(True)
    (torch.nn.functional.silu(g) * u).backward(dact.float())
    dgu = ops.swiglu_bwd(gu, dact).float().view(M, F // 8, 2, 8)
    assert _rel(dgu[:, :, 0].reshape(M, F), g.grad) < 6e-3 and _rel(dgu[:, :, 1].reshape(M, F), u.grad) < 6e-3


def test_qk_rope_bwd(ops):
    torch.manual_seed(2)
    M, nq, nk, D = 70, 4, 2, 128
    W = (nq + 2 * nk) * D
    pre = torch.randn(M, W).bfloat16().cuda()
    qw = (1 + 0.1 * torch.randn(D)).bfloat16().cuda(); kw = (1 + 0.1 * torch.randn(D)).bfloat16().cuda()
    pos = torch.randint(0, 2500, (M,), dtype=torch.int32).cuda()
    dy = torch.randn(M, W).bfloat16().cuda()
    x = pre[:, :(nq + nk) * D].float().view(M, nq + nk, D).clone().requires_grad_(True)
    w = torch.cat([qw[None].expand(nq, D), kw[None].expand(nk, D)]).float()[None]
    xn = w * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6))
    inv = 1.0 / (1e6 ** (torch.arange(0, D, 2, device="cuda").float() / D))
    fr = pos.float()[:, None] * inv[None]
    cos, sin = torch.cat([fr, fr], -1).cos()[:, None], torch.cat([fr, fr], -1).sin()[:, None]
    rot = torch.cat([-xn[..., D // 2:], xn[..., :D // 2]], -1)
    y = xn * cos + rot * sin
    y.backward(dy[:, :(nq + nk) * D].float().view(M, nq + nk, D))
    d = dy.clone()
    ops.qk_rope_bwd_(d, pre, nq, nk, D, qw, kw, pos, 1e6, 1e-6)
    assert _rel(d[:, :(nq + nk) * D].view(M, nq + nk, D), x.grad) < 1.5e-2
    assert torch.equal(d[:, (nq + nk) * D:], dy[:, (nq + nk) * D:])


@pytest.mark.parametrize("B,L,nq,nkv", [(2, 200, 4, 2), (1, 333, 8, 2), (2, 1100, 8, 8), (3, 64, 2, 1)])
def test_attn_bwd(ops, B, L, nq, nkv):
    torch.manual_seed(L)
    D = 128
    W = (nq + 2 * nkv) * D
    qkv = (torch.randn(B * L, W) * 0.7).bfloat16().cuda()
    ks = torch.randint(0, L // 4, (B,), dtype=torch.int32).cuda(); ke = torch.randint(3 * L // 4, L + 1, (B,), dtype=torch.int32).cuda()
    ks[0] = 0; ke[0] = L
    q, k, v = qkv[:, :nq * D], qkv[:, nq * D:(nq + nkv) * D], qkv[:, (nq + nkv) * D:]
    o, lse = ops.attn_fwd(q, k, v, B, L, nq, nkv, D, kv_start=ks, kv_end=ke, causal=True, want_lse=True)
    do = torch.randn(B * L, nq * D).bfloat16().cuda()
    dqkv = torch.zeros(B * L, W, dtype=torch.bfloat16, device="cuda")
    ops.attn_bwd(q, k, v, o, do, lse, dqkv[:, :nq * D], dqkv[:, nq * D:(nq + nkv) * D], dqkv[:, (nq + nkv) * D:], B, L, nq, nkv, D,
                 kv_start=ks, kv_end=ke)
    # torch autograd reference (fp32 on the same device)
    x = qkv.float().clone().requires_grad_(True)
    qf = x[:, :nq * D].view(B, L, nq, D).transpose(1, 2)
    kf = x[:, nq * D:(nq + nkv) * D].view(B, L, nkv, D).transpose(1, 2).repeat_interleave(nq // nkv, 1)
    vf = x[:, (nq + nkv) * D:].view(B, L, nkv, D).transpose(1, 2).repeat_interleave(nq // nkv, 1)
    j = torch.arange(L, device="cuda")
    ok = (j[None, None, None, :] >= ks[:, None, None, None]) & (j[None, None, None, :] < ke[:, None, None, None]) & (j[None, None, None, :] <= j[None, None, :, None])
    s = (qf @ kf.transpose(-1, -2)) * D ** -0.5
    p = torch.softmax(s.masked_fill(~ok, float("-inf")), -1).nan_to_num(0.0)
    out = (p @ vf).transpose(1, 2).reshape(B * L, nq * D)
    out.backward(do.float())
    for name, sl in (("dq", slice(0, nq * D)), ("dk", slice(nq * D, (nq + nkv) * D)), ("dv", slice((nq + nkv) * D, W))):
        r = _rel(dqkv[:, sl], x.grad[:, sl])
        assert r < 2e-2, f"{name} rel err {r}"


def test_lora_grad_tn_transpose_colsum(ops):
    """The wgmma TN GEMM behind the LoRA gradients (both operands MN-major, split-K without atomics): all three epilogue modes,
    accumulation into the destination, strided views, bit-reproducibility; plus the transpose and column-sum helpers."""
    torch.manual_seed(3)
    M, P = 1000, 512
    big = torch.randn(M, P).bfloat16().cuda()
    for Rr in (32, 64, 16, 96):
        small = torch.randn(M, Rr).bfloat16().cuda()
        ref = big.float().T @ small.float()
        out = torch.zeros(P, Rr, device="cuda")
        ops.lora_grad_tn(big, small, [(out, 0, P, 0, Rr)])
        assert _rel(out, ref) < 1e-3
        ops.lora_grad_tn(big, small, [(out, 0, P, 0, Rr)])                        # accumulates
        assert _rel(out, 2 * ref) < 1e-3
        outT = torch.zeros(Rr, P, device="cuda")
        ops.lora_grad_tn(big, small, [(outT, 0, P, 0, Rr)], mode=1)
        assert _rel(outT, ref.T) < 1e-3
        again = torch.zeros(Rr, P, device="cuda")
        ops.lora_grad_tn(big, small, [(again, 0, P, 0, Rr)], mode=1)
        assert torch.equal(again, outT), "split-K reduction must be bit-reproducible"
    # block-diagonal segments of a fused product (the q | k | v layout) on strided column views, long M (split-K across many CTAs)
    M2 = 5000
    big2 = torch.randn(M2, 384).bfloat16().cuda(); t = torch.randn(M2, 96).bfloat16().cuda()
    dq, dk, dv = torch.zeros(256, 32, device="cuda"), torch.zeros(64, 32, device="cuda"), torch.zeros(64, 32, device="cuda")
    ops.lora_grad_tn(big2, t, [(dq, 0, 256, 0, 32), (dk, 256, 320, 32, 32), (dv, 320, 384, 64, 32)])
    full = big2.float().T @ t.float()
    assert _rel(dq, full[:256, :32]) < 1e-3 and _rel(dk, full[256:320, 32:64]) < 1e-3 and _rel(dv, full[320:, 64:]) < 1e-3
    ov = torch.zeros(256, 32, device="cuda")
    ops.lora_grad_tn(big2[:, 128:384], t[:, 32:64], [(ov, 0, 256, 0, 32)])
    assert _rel(ov, big2[:, 128:384].float().T @ t[:, 32:64].float()) < 1e-3
    # gate/up-blocked rows (blocks of 16 = 8 gate | 8 up)
    gu = torch.randn(M, 2 * 256).bfloat16().cuda(); t2 = torch.randn(M, 64).bfloat16().cuda()
    g4 = gu.float().view(M, 32, 2, 8)
    og, ou = torch.zeros(256, 32, device="cuda"), torch.zeros(256, 32, device="cuda")
    ops.lora_grad_tn(gu, t2, [(og, 0, 512, 0, 32), (ou, 0, 512, 32, 32)], mode=2)
    assert _rel(og, g4[:, :, 0].reshape(M, 256).T @ t2[:, :32].float()) < 1e-3
    assert _rel(ou, g4[:, :, 1].reshape(M, 256).T @ t2[:, 32:].float()) < 1e-3
    x = torch.randn(77, 130).bfloat16().cuda()
    xt = ops.transpose(x)
    assert xt.shape == (130, 80) and torch.equal(xt[:, :77], x.T) and xt[:, 77:].abs().sum() == 0
    cs = torch.zeros(P, device="cuda")
    ops.colsum_accumulate_(cs, big)
    assert _rel(cs, big.float().sum(0)) < 1e-3
    cs2 = torch.zeros(P, device="cuda")
    ops.colsum_accumulate_(cs2, big)
    assert torch.equal(cs, cs2)


@pytest.mark.parametrize("cfg_name,B,n_seq,dna_len,text_len,C", [("tiny", 2, 1, [12, 9], [20, 14], 6), ("small", 3, 2, 40, [50, 66, 41], 9)])
def test_policy_gradients_vs_oracle(cfg_name, B, n_seq, dna_len, text_len, C):
    """d(sum w * logp)/d(LoRA A, B, projector) through the whole decoder vs torch autograd on the fp32 oracle."""
    from bioreason_b200.configs import text_config, dna_config
    from bioreason_b200.models import DNALLMModel
    from bioreason_b200 import training
    from oracle.models import build_oracle, synth_batch
    from oracle import lora as olora, grpo as og
    tc, dc = text_config(cfg_name), dna_config(cfg_name)
    oracle = build_oracle(tc, dc, seed=11)
    batch = synth_batch(tc, dc, batch=B, n_seq=n_seq, dna_len=dna_len, text_len=text_len, seed=4)
    comp = torch.randint(0, tc.eos_token_id, (B, C), generator=torch.Generator().manual_seed(9))
    ids = torch.cat([batch["input_ids"], comp], 1)
    mask = torch.cat([batch["attention_mask"], torch.ones(B, C, dtype=torch.long)], 1)
    mask[0, -2:] = 0                                                       # a post-EOS tail on one row
    wgt = torch.randn(B, C, generator=torch.Generator().manual_seed(10))
    r, alpha = 16, 32.0
    m = DNALLMModel.from_oracle(oracle)
    lora = m.enable_lora(r=r, alpha=alpha, seed=3)
    with torch.no_grad():                                                  # non-zero B so every gradient path is live
        g = torch.Generator().manual_seed(5)
        for p in lora.params[1::2]:
            p.copy_((torch.randn(p.shape, generator=g) * 0.02).to(p.device))
    m.sync_adapters(rollout=False)
    # oracle with identical adapters
    olora.inject(oracle.text_model, r, alpha)
    sd = {k: v.detach().float().cpu() for k, v in m.text_model.state_dict().items() if "lora_" in k}
    missing, unexpected = oracle.text_model.load_state_dict(sd, strict=False)
    assert not unexpected
    for p in oracle.dna_projection.parameters():
        p.requires_grad_(True)
    mm = dict(dna_tokenized=batch["dna_tokenized"], batch_idx_map=batch["batch_idx_map"])
    lp_o = og.per_token_logps(oracle, ids, mask, **mm)[:, -C:]
    (lp_o * wgt).sum().backward()
    # CUDA path
    m.zero_grad_buffers()
    lp, ctx = training.policy_forward(m, ids, mask, batch["dna_tokenized"], batch["batch_idx_map"], C)
    assert (lp.cpu() - lp_o.detach()).abs().max().item() < 0.03
    training.policy_backward(m, ctx, wgt.cuda())
    m.attach_grads()
    onames = dict(oracle.text_model.named_parameters())
    worst = 0.0
    for name, p in m.text_model.named_parameters():
        if "lora_" not in name:
            continue
        go = onames[name].grad
        rel = _rel(p.grad.cpu(), go)
        worst = max(worst, rel)
        assert rel < 0.08, f"{name}: rel err {rel:.4f} (|g| {go.norm():.3e})"
    rw = _rel(m.dna_projection.weight.grad.cpu(), oracle.dna_projection.weight.grad)
    rb = _rel(m.dna_projection.bias.grad.cpu(), oracle.dna_projection.bias.grad)
    print(f"{cfg_name}: worst LoRA grad rel err {worst:.4f}; projector dW {rw:.4f} db {rb:.4f}")
    assert rw < 0.05 and rb < 0.05
    # autograd bridge gives the same gradients
    for p in m.trainable_parameters():
        p.grad = None
    m.zero_grad_buffers()
    lp2 = training.policy_logps_autograd(m, ids, mask, batch["dna_tokenized"], batch["batch_idx_map"], C)
    (lp2 * wgt.cuda()).sum().backward()
    assert _rel(m.dna_projection.weight.grad.cpu(), oracle.dna_projection.weight.grad) < 0.05
    p0 = lora.params[0]
    assert _rel(p0.grad.cpu(), onames[[n for n, q in m.text_model.named_parameters() if q is p0][0]].grad) < 0.08


def test_sft_step_vs_oracle():
    """Config (b) shape of work: CE loss over assistant-span labels + backward through LoRA and the projector vs torch autograd."""
    from bioreason_b200.configs import text_config, dna_config
    from bioreason_b200.models import DNALLMModel
    from oracle.models import build_oracle, synth_batch
    from oracle import lora as olora
    tc, dc = text_config("small"), dna_config("small")
    oracle = build_oracle(tc, dc, seed=13)
    batch = synth_batch(tc, dc, batch=3, n_seq=2, dna_len=[30, 22, 30], text_len=[64, 50, 71], seed=6)
    labels = batch["input_ids"].clone()
    labels[batch["attention_mask"] == 0] = -100
    labels[:, : labels.shape[1] - 24] = -100                               # only the last 24 tokens ("assistant span") are scored
    m = DNALLMModel.from_oracle(oracle)
    lora = m.enable_lora(r=16, alpha=32.0, seed=1)
    with torch.no_grad():
        g = torch.Generator().manual_seed(2)
        for p in lora.params[1::2]:
            p.copy_((torch.randn(p.shape, generator=g) * 0.02).to(p.device))
    m.sync_adapters(rollout=False)
    olora.inject(oracle.text_model, 16, 32.0)
    sd = {k: v.detach().float().cpu() for k, v in m.text_model.state_dict().items() if "lora_" in k}
    assert not oracle.text_model.load_state_dict(sd, strict=False).unexpected_keys
    for p in oracle.dna_projection.parameters():
        p.requires_grad_(True)
    out = oracle(**batch, labels=labels)
    out.loss.backward()
    m.zero_grad_buffers()
    loss = m.sft_step(**batch, labels=labels)
    assert abs(loss.item() - out.loss.item()) < 5e-3, (loss.item(), out.loss.item())
    # forward-only .loss of the drop-in forward() agrees too
    assert abs(m(**batch, labels=labels).loss.item() - out.loss.item()) < 5e-3
    m.attach_grads()
    onames = dict(oracle.text_model.named_parameters())
    worst = max(_rel(p.grad.cpu(), onames[n].grad) for n, p in m.text_model.named_parameters() if "lora_" in n)
    rw = _rel(m.dna_projection.weight.grad.cpu(), oracle.dna_projection.weight.grad)
    print(f"sft: loss {loss.item():.4f} vs {out.loss.item():.4f}; worst LoRA grad rel err {worst:.4f}; projector dW {rw:.4f}")
    assert worst < 0.08 and rw < 0.05
