"""LoRA dropout on the H100: the device mask against the NumPy rule, the three masked kernels against fp32 torch on the same masks,
the policy / SFT gradients against autograd on the masked fp32 oracle, determinism, and the untouched default path."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from lora_dropout_ref import OracleMasks, keep_mask, mask_oracle, threshold

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from bioreason_b200 import ops
    return ops


def _rel(a, b):
    return (a.float() - b.float()).norm().item() / (b.float().norm().item() + 1e-12)


def _desc(ops, seed=77, pass_id=3, p=0.05, row_offset=0, layer=2, proj=0, r=32):
    from bioreason_b200.engine import LoraDropout
    return ops.lora_dropout_desc(LoraDropout(seed=seed, pass_id=pass_id, threshold=threshold(p), row_offset=row_offset), layer, proj, r)


def _mask(ops, d, M, K):
    return ops.lora_dropout_mask(d, M, K, "cuda").bool()


@pytest.mark.parametrize("M,K,row_offset,layer,proj,seed", [(37, 200, 0, 0, 0, 1), (130, 2560, 1000, 5, 6, 2 ** 40 + 9),
                                                             (5, 9728, 123457, 35, 4, 42)])
def test_device_mask_matches_numpy(ops, M, K, row_offset, layer, proj, seed):
    d = _desc(ops, seed=seed, pass_id=11, p=0.05, row_offset=row_offset, layer=layer, proj=proj)
    got = _mask(ops, d, M, K).cpu().numpy()
    want = keep_mask(seed, 11, layer, proj, np.arange(row_offset, row_offset + M), K, threshold(0.05))
    assert np.array_equal(got, want)


# (M, K = adapter input width, r, n_proj): tiny / small widths and the Qwen3-4B ones (d 2560, Hq*D 4096, F 9728)
DOWN = [(300, 256, 16, 3), (129, 512, 32, 2), (1000, 2560, 32, 3), (777, 4096, 32, 1), (640, 9728, 16, 1), (513, 2560, 16, 2),
        (200, 2560, 64, 1), (333, 2560, 64, 3)]


@pytest.mark.parametrize("M,K,r,n_proj", DOWN)
def test_masked_down_projection(ops, M, K, r, n_proj):
    torch.manual_seed(M + K)
    x = torch.randn(M, K, device="cuda").bfloat16()
    a = (torch.randn(n_proj * r, K, device="cuda") / K ** 0.5).bfloat16()
    scale, T = 2.0, threshold(0.05)
    inv = 65536 / (65536 - T)
    d = _desc(ops, row_offset=4096, layer=1, proj=4 if n_proj == 2 else 0, r=r)
    t = ops.lora_down_dropout(x, a, scale, d)
    ref = torch.cat([(x.float() * _mask(ops, _desc(ops, row_offset=4096, layer=1, proj=d.proj + j, r=r), M, K).float()) @ a[j * r:(j + 1) * r].float().T
                     for j in range(n_proj)], 1) * (scale * inv)
    assert _rel(t, ref) < 1e-2
    assert torch.equal(t, ops.lora_down_dropout(x, a, scale, d))


# (M, N = dx width, Kd = dy width, r, n_proj, first projection)
DX = [(300, 256, 512, 16, 3, 0), (200, 512, 1024, 32, 2, 4), (1000, 2560, 6144, 32, 3, 0), (700, 4096, 2560, 32, 1, 3),
      (513, 9728, 2560, 16, 1, 6), (600, 2560, 19456, 16, 2, 4), (400, 2560, 6144, 64, 3, 0), (300, 2560, 19456, 64, 2, 4)]


@pytest.mark.parametrize("M,N,Kd,r,n_proj,proj", DX)
def test_masked_dx_segment(ops, M, N, Kd, r, n_proj, proj):
    torch.manual_seed(N + Kd)
    dy = torch.randn(M, Kd, device="cuda").bfloat16()
    w = (torch.randn(N, Kd, device="cuda") / Kd ** 0.5).bfloat16()           # w_T [N, Kd]: dx = dy @ w_T.T
    u = torch.randn(M, n_proj * r, device="cuda").bfloat16()
    aT = (torch.randn(N, n_proj * r, device="cuda") * 0.1).bfloat16()
    T = threshold(0.05)
    inv = 65536 / (65536 - T)
    d = _desc(ops, row_offset=77, layer=3, proj=proj, r=r)
    dx = ops.gemm(dy, w, a2=u, b2=aT, dropout=d)
    ref = dy.float() @ w.float().T
    for j in range(n_proj):
        m = _mask(ops, _desc(ops, row_offset=77, layer=3, proj=proj + j, r=r), M, N).float()
        ref += m * inv * (u[:, j * r:(j + 1) * r].float() @ aT[:, j * r:(j + 1) * r].float().T)
    assert _rel(dx, ref) < 1e-2
    plain = ops.gemm(dy, w, a2=u, b2=aT)
    assert not torch.equal(dx, plain)
    assert torch.equal(dx, ops.gemm(dy, w, a2=u, b2=aT, dropout=d))


@pytest.mark.parametrize("M,P,r,proj", [(1000, 512, 16, 0), (300, 256, 32, 5), (5000, 2560, 32, 1), (3000, 4096, 32, 3), (2000, 9728, 16, 6)])
def test_masked_tn_gradient(ops, M, P, r, proj):
    torch.manual_seed(M + P)
    x = torch.randn(M, P, device="cuda").bfloat16()
    u = torch.randn(M, r, device="cuda").bfloat16()
    T = threshold(0.05)
    inv = 65536 / (65536 - T)
    d = _desc(ops, row_offset=333, layer=7, proj=proj, r=r)
    m = _mask(ops, d, M, P).float()
    ref = inv * (u.float().T @ (x.float() * m))                                # dA [r, P]
    out = torch.zeros(r, P, device="cuda")
    ops.lora_grad_tn(x, u, [(out, 0, P, 0, r)], mode=1, dropout=d)
    assert _rel(out, ref) < 1e-3
    again = torch.zeros(r, P, device="cuda")
    ops.lora_grad_tn(x, u, [(again, 0, P, 0, r)], mode=1, dropout=d)
    assert torch.equal(out, again)


def _policy_setup(cfg_name, B, n_seq, dna_len, text_len, C, r=16, alpha=32.0, seed=11):
    from bioreason_b200.configs import text_config, dna_config
    from bioreason_b200.models import DNALLMModel
    from oracle.models import build_oracle, synth_batch
    from oracle import lora as olora
    tc, dc = text_config(cfg_name), dna_config(cfg_name)
    oracle = build_oracle(tc, dc, seed=seed)
    batch = synth_batch(tc, dc, batch=B, n_seq=n_seq, dna_len=dna_len, text_len=text_len, seed=4)
    comp = torch.randint(0, tc.eos_token_id, (B, C), generator=torch.Generator().manual_seed(9))
    ids = torch.cat([batch["input_ids"], comp], 1)
    mask = torch.cat([batch["attention_mask"], torch.ones(B, C, dtype=torch.long)], 1)
    m = DNALLMModel.from_oracle(oracle)
    lora = m.enable_lora(r=r, alpha=alpha, seed=3)
    with torch.no_grad():
        g = torch.Generator().manual_seed(5)
        for p in lora.params[1::2]:
            p.copy_((torch.randn(p.shape, generator=g) * 0.02).to(p.device))
    m.sync_adapters(rollout=False)
    olora.inject(oracle.text_model, r, alpha)
    sd = {k: v.detach().float().cpu() for k, v in m.text_model.state_dict().items() if "lora_" in k}
    assert not oracle.text_model.load_state_dict(sd, strict=False).unexpected_keys
    for p in oracle.dna_projection.parameters():
        p.requires_grad_(True)
    return m, oracle, batch, ids, mask


@pytest.mark.parametrize("cfg_name,B,n_seq,dna_len,text_len,C", [("tiny", 2, 1, [12, 9], [20, 14], 6), ("small", 3, 2, 40, [50, 66, 41], 9)])
def test_policy_gradients_with_dropout_vs_oracle(cfg_name, B, n_seq, dna_len, text_len, C):
    from bioreason_b200 import training
    from oracle import grpo as og
    m, oracle, batch, ids, mask = _policy_setup(cfg_name, B, n_seq, dna_len, text_len, C)
    mask[0, -2:] = 0
    wgt = torch.randn(B, C, generator=torch.Generator().manual_seed(10))
    p, seed = 0.05, 1234
    m.set_lora_dropout(p, seed=seed)
    pid = m.new_lora_dropout_pass()
    mask_oracle(oracle.text_model, OracleMasks(seed, pid, threshold(p)))
    mm = dict(dna_tokenized=batch["dna_tokenized"], batch_idx_map=batch["batch_idx_map"])
    lp_o = og.per_token_logps(oracle, ids, mask, **mm)[:, -C:]
    (lp_o * wgt).sum().backward()
    m.zero_grad_buffers()
    lp, ctx = training.policy_forward(m, ids, mask, batch["dna_tokenized"], batch["batch_idx_map"], C, dropout=True, dropout_pass=pid)
    assert (lp.cpu() - lp_o.detach()).abs().max().item() < 0.03
    training.policy_backward(m, ctx, wgt.cuda())
    m.attach_grads()
    onames = dict(oracle.text_model.named_parameters())
    worst = max(_rel(q.grad.cpu(), onames[n].grad) for n, q in m.text_model.named_parameters() if "lora_" in n)
    rw = _rel(m.dna_projection.weight.grad.cpu(), oracle.dna_projection.weight.grad)
    print(f"{cfg_name} p={p}: worst LoRA grad rel err {worst:.4f}; projector dW {rw:.4f}")
    assert worst < 0.08 and rw < 0.05
    # the undropped forward differs (the masks are live), and the reference-policy pass ignores the dropout
    lp0, _ = training.policy_forward(m, ids, mask, batch["dna_tokenized"], batch["batch_idx_map"], C, save=False)
    assert not torch.equal(lp0, lp)
    r1, _ = training.policy_forward(m, ids, mask, batch["dna_tokenized"], batch["batch_idx_map"], C, save=False, lora=None)
    r2, _ = training.policy_forward(m, ids, mask, batch["dna_tokenized"], batch["batch_idx_map"], C, save=False, lora=None, dropout=True)
    assert torch.equal(r1, r2)


def test_sft_step_with_dropout_vs_oracle():
    m, oracle, batch, ids, mask = _policy_setup("small", 3, 2, [30, 22, 30], [64, 50, 71], 0, seed=13)
    labels = batch["input_ids"].clone()
    labels[batch["attention_mask"] == 0] = -100
    labels[:, : labels.shape[1] - 24] = -100
    p, seed = 0.05, 99
    m.set_lora_dropout(p, seed=seed)
    pid = m._lora.dropout_pass                                              # the pass sft_step will draw
    mask_oracle(oracle.text_model, OracleMasks(seed, pid, threshold(p)))
    out = oracle(**batch, labels=labels)
    out.loss.backward()
    m.zero_grad_buffers()
    loss = m.sft_step(**batch, labels=labels)
    assert m._lora.dropout_pass == pid + 1
    assert abs(loss.item() - out.loss.item()) < 5e-3, (loss.item(), out.loss.item())
    m.attach_grads()
    onames = dict(oracle.text_model.named_parameters())
    worst = max(_rel(q.grad.cpu(), onames[n].grad) for n, q in m.text_model.named_parameters() if "lora_" in n)
    rw = _rel(m.dna_projection.weight.grad.cpu(), oracle.dna_projection.weight.grad)
    print(f"sft p={p}: worst LoRA grad rel err {worst:.4f}; projector dW {rw:.4f}")
    assert worst < 0.08 and rw < 0.05
    # forward-only SFT loss draws no pass and applies no dropout
    m.sft_step(**batch, labels=labels, backward=False)
    assert m._lora.dropout_pass == pid + 1


def test_dropout_determinism_and_chunking():
    from bioreason_b200 import training
    B, C = 3, 9
    m, oracle, batch, ids, mask = _policy_setup("small", B, 2, 40, [50, 66, 41], C)
    m.set_lora_dropout(0.05, seed=5)
    wgt = torch.randn(B, C, generator=torch.Generator().manual_seed(1)).cuda()
    dna, idx = batch["dna_tokenized"], batch["batch_idx_map"]

    def run(pid, chunks):
        from bioreason_b200.trainer.grpo_trainer import _slice_mm
        m.zero_grad_buffers()
        lps = []
        mm = dict(dna_tokenized={k: v.cuda() for k, v in dna.items()}, batch_idx_map=idx)
        for lo, hi in chunks:
            mc = _slice_mm(mm, lo, hi)
            lp, ctx = training.policy_forward(m, ids[lo:hi], mask[lo:hi], mc["dna_tokenized"], mc["batch_idx_map"], C, dropout=True,
                                              dropout_pass=pid, row_offset=lo)
            training.policy_backward(m, ctx, wgt[lo:hi])
            lps.append(lp)
        return torch.cat(lps), m._lora.flat_grad.clone(), m._proj_grad_w.clone()

    whole = [(0, B)]
    a = run(0, whole)
    b = run(0, whole)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    c = run(1, whole)
    assert not torch.equal(a[0], c[0]) and not torch.equal(a[1], c[1])
    rows = run(0, [(i, i + 1) for i in range(B)])
    assert torch.equal(rows[0], a[0])
    assert _rel(rows[1], a[1]) < 1e-4 and _rel(rows[2], a[2]) < 1e-4


def _token_reward(completion_ids, **kw):
    return (completion_ids % 7 == 0).float().sum(1) - 0.1 * (completion_ids % 5 == 0).float().sum(1)


def _trainer(apply, seed=21, mu=1, p=None):
    from bioreason_b200.configs import text_config, dna_config
    from bioreason_b200.models import DNALLMModel
    from bioreason_b200.trainer import DNALLMGRPOConfig, DNALLMGRPOTrainer
    from oracle.models import build_oracle, synth_batch
    tc, dc = text_config("tiny"), dna_config("tiny")
    m = DNALLMModel.from_oracle(build_oracle(tc, dc, seed=seed))
    if p is not None:
        m.lora_dropout = p                                                   # what compat.peft.get_peft_model records
    batch = synth_batch(tc, dc, batch=4, n_seq=2, dna_len=10, text_len=18, seed=14, same_prompt=True)
    cfg = DNALLMGRPOConfig(num_generations=4, max_completion_length=6, per_device_train_batch_size=4, learning_rate=1e-2, lora_r=16,
                           lora_alpha=32.0, apply_lora_dropout=apply, num_iterations=mu)
    return m, DNALLMGRPOTrainer(m, [_token_reward], cfg), batch


def _step(m, tr, batch):
    u = torch.rand(6, 4, generator=torch.Generator().manual_seed(0))
    inp = tr._generate_and_score_completions(batch, m, uniforms=u)
    m.zero_grad_buffers()
    tr._step = 0
    loss = tr.compute_loss(m, inp)
    return inp, loss, m._lora.flat_grad.clone(), m._proj_grad_w.clone()


def test_default_path_unchanged_and_rollout_dropout_free():
    m0, t0, b0 = _trainer(False)
    m1, t1, b1 = _trainer(False)
    m1.set_lora_dropout(0.0)
    assert m0._lora.dropout is None and m1._lora.dropout is None
    with torch.no_grad():                                                   # live adapters so a dropped path would show
        for ma, mb in ((m0, m1),):
            g = torch.Generator().manual_seed(2)
            for pa, pb in zip(ma._lora.params[1::2], mb._lora.params[1::2]):
                v = torch.randn(pa.shape, generator=g) * 0.05
                pa.copy_(v.to(pa.device)); pb.copy_(v.to(pb.device))
    for mm_ in (m0, m1):
        mm_.sync_adapters(rollout=True)
    i0, l0, g0, p0 = _step(m0, t0, b0)
    i1, l1, g1, p1 = _step(m1, t1, b1)
    assert torch.equal(i0["completion_ids"], i1["completion_ids"]) and torch.equal(l0, l1) and torch.equal(g0, g1) and torch.equal(p0, p1)
    # turning dropout on changes the loss gradients but neither the seeded rollout nor the reference log-probs
    m1.set_lora_dropout(0.05, seed=3)
    i2, l2, g2, _ = _step(m1, t1, b1)
    assert torch.equal(i0["completion_ids"], i2["completion_ids"])
    assert torch.equal(i0["ref_per_token_logps"], i2["ref_per_token_logps"])
    assert not torch.equal(g0, g2)


def test_grpo_two_steps_with_dropout():
    m, tr, batch = _trainer(True, mu=2, p=0.1)
    assert m._lora.dropout is not None and m._lora.dropout[0] == 0.1 and m._lora.dropout[2] == 42   # peft's rate, seed + rank
    p0 = [q.detach().clone() for q in m.trainable_parameters()]
    passes = m._lora.dropout_pass
    l1 = tr.training_step(batch)
    l2 = tr.training_step(batch)
    assert torch.isfinite(l1) and torch.isfinite(l2)
    assert m._lora.dropout_pass > passes
    moved = sum(int(not torch.equal(a, b.detach())) for a, b in zip(p0, m.trainable_parameters()))
    assert moved > len(p0) // 2


def test_sass_of_the_dropout_kernels():
    from bioreason_b200 import build
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    for name in ("lora_dropout_tc5.o", "lora_grad_tc5.o", "gemm_tc5.o"):
        sass = subprocess.run([cuobjdump, "-sass", os.path.join(build.OUT_DIR, name)], capture_output=True, text=True).stdout
        assert "HGMMA" in sass and "UTMALDG" in sass and "HMMA." not in sass, name
        if name != "gemm_tc5.o":                                            # masked operands go in as the register-A form
            assert re.search(r"HGMMA\.64x\d+x16\.F32\.BF16 R\d+, R\d+, gdesc", sass), name


def test_config_c_geometry_gradients_with_dropout():
    """Config (c) geometry at Qwen3-4B widths, depth 2, r = 32 (qkv spans two BK blocks of the masked dX segment): L = 2364, G = 8,
    2-row chunks whose row offsets run to 14 184, against autograd on the fp32 oracle carrying the NumPy masks of the whole pass."""
    from bioreason_b200 import training
    from oracle.models import synth_batch
    from test_gpu_bench_shapes import _build_pair, _cfgs, _cuda_batch, _grad_report, _oracle_logps
    tc, dc = _cfgs("qwen3-4b")
    oracle, m, lora = _build_pair(tc, dc, seed=31)
    assert lora.r == 32
    G, C = 8, 512
    batch = synth_batch(tc, dc, batch=G, n_seq=2, dna_len=668, text_len=512, seed=8, same_prompt=True)
    comp = torch.randint(0, tc.eos_token_id, (G, C), generator=torch.Generator().manual_seed(9))
    ids = torch.cat([batch["input_ids"], comp], 1).cuda()
    L = ids.shape[1]
    cmask = torch.ones(G, C, dtype=torch.long); cmask[1, -37:] = 0; cmask[5, -200:] = 0
    mask = torch.cat([batch["attention_mask"], cmask], 1).cuda()
    wgt = (torch.randn(G, C, generator=torch.Generator().manual_seed(10)) * cmask).cuda()
    cb = _cuda_batch(batch)
    mm = dict(dna_tokenized=cb["dna_tokenized"], batch_idx_map=cb["batch_idx_map"])
    p, seed = 0.05, 2024
    m.set_lora_dropout(p, seed=seed)
    pid = m.new_lora_dropout_pass()
    masks = OracleMasks(seed, pid, threshold(p))
    mask_oracle(oracle.text_model, masks)
    lp_o = []
    for r in range(G):                                                     # the oracle one row at a time: its rows are r * L + t
        masks.row0 = r * L
        lp_r = _oracle_logps(oracle, ids[r:r + 1], mask[r:r + 1], dict(dna_tokenized={k: v[2 * r:2 * r + 2] for k, v in mm["dna_tokenized"].items()},
                                                                       batch_idx_map=[0, 0]), C)
        (lp_r * wgt[r:r + 1]).sum().backward()
        lp_o.append(lp_r.detach())
    lp_o = torch.cat(lp_o)
    m.zero_grad_buffers()
    lps = []
    for lo in range(0, G, 2):
        hi = lo + 2
        idx = [i for i, b in enumerate(mm["batch_idx_map"]) if lo <= b < hi]
        dna = {k: v[idx] for k, v in mm["dna_tokenized"].items()}
        lp_c, ctx = training.policy_forward(m, ids[lo:hi], mask[lo:hi], dna, [mm["batch_idx_map"][i] - lo for i in idx], C, dropout=True,
                                            dropout_pass=pid, row_offset=lo)
        training.policy_backward(m, ctx, wgt[lo:hi])
        del ctx
        lps.append(lp_c)
    lp = torch.cat(lps)
    att = cmask.bool().cuda()
    err = (lp - lp_o)[att].abs()
    worst, wname, rw, rb = _grad_report(m, oracle)
    print(f"(c) p={p} r=32: logps max|err| {err.max():.4f} mean {err.mean():.5f}; worst LoRA grad rel err {worst:.4f} ({wname}); "
          f"projector dW {rw:.4f} db {rb:.4f}")
    assert err.mean().item() < 0.02
    assert worst < 0.03 and rw < 0.03 and rb < 0.03
