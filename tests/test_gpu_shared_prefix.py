"""Shared-prefix layout on the GPU: the attention kernels against the dense ones on the equivalent batch, policy log-probs and
gradients with group_size against the dense path (and the fp32 oracle), and the GRPO trainer with share_prompt_prefix on and off."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return (a.float() - b.float()).norm().item() / (b.float().norm().item() + 1e-12)


# ---------------------------------------------------------------------------------------------------------------- kernels
# (U, G, Lp, Ls, nq, nkv, kv_start per group, kv_end per row (None = row end))
KCASES = [
    (1, 8, 1792, 572, 4, 1, [0], [2364, 2364 - 37, 1853, 2364, 1900, 2364, 2364, 2000]),     # config (c) geometry, GQA 4:1, EOS rows
    (2, 2, 64, 150, 4, 2, [30, 70], [214, 101, 101, 180]),        # GQA 2:1; start inside the prefix / inside the tail; end just past P
    (2, 3, 0, 130, 8, 2, [0, 17], None),                           # no prefix: the suffix kernels alone
    (2, 1, 128, 100, 4, 2, [5, 0], [228, 140]),                    # G = 1: prefix dK/dV equal the dense kernel's
    (1, 4, 192, 67, 2, 1, [200], [259, 259, 250, 210]),            # left padding longer than the prefix
]


def _shared_inputs(U, G, Lp, Ls, nq, nkv, seed):
    torch.manual_seed(seed)
    D = 128
    W = (nq + 2 * nkv) * D
    R, L = U * G, Lp + Ls
    pre = (torch.randn(U * Lp, W) * 0.7).bfloat16().cuda()
    suf = (torch.randn(R * Ls, W) * 0.7).bfloat16().cuda()
    buf = torch.cat([pre, suf])
    dense = torch.cat([torch.cat([pre.view(U, Lp, W)[r // G], suf.view(R, Ls, W)[r]]) for r in range(R)])      # [R*L, W]
    return buf, dense, D, W, R, L


@pytest.mark.parametrize("U,G,Lp,Ls,nq,nkv,ks,ke", KCASES)
def test_attn_shared_matches_dense(U, G, Lp, Ls, nq, nkv, ks, ke):
    from bioreason_b200 import ops
    buf, dense, D, W, R, L = _shared_inputs(U, G, Lp, Ls, nq, nkv, seed=Lp + Ls + G)
    kv_start = torch.tensor(ks, dtype=torch.int32, device="cuda")
    kv_end = torch.tensor(ke if ke is not None else [L] * R, dtype=torch.int32, device="cuda")
    ks_d = kv_start.repeat_interleave(G)
    qo, ko, vo = 0, nq * D, (nq + nkv) * D
    views = lambda x: (x[:, qo:ko], x[:, ko:vo], x[:, vo:])
    # ---- forward: bit-identical to the dense kernel
    o_d, lse_d = ops.attn_fwd(*views(dense), R, L, nq, nkv, D, kv_start=ks_d, kv_end=kv_end, causal=True, want_lse=True)
    o_s, (lse_p, lse_s) = ops.attn_fwd_shared(*views(buf), U, G, Lp, Ls, nq, nkv, D, kv_start, kv_end, want_lse=True)
    o_d3 = o_d.view(R, L, nq * D)
    assert torch.equal(o_s[:U * Lp].view(U, Lp, nq * D), o_d3[::G, :Lp])
    assert torch.equal(o_s[U * Lp:].view(R, Ls, nq * D), o_d3[:, Lp:])
    assert torch.equal(lse_p, lse_d[::G, :, :Lp]) and torch.equal(lse_s, lse_d[:, :, Lp:])
    # ---- backward.  Prefix dO lives once per group: the dense equivalent gives it to row g = 0 and zero to the other rows' prefixes
    torch.manual_seed(1)
    do_buf = torch.randn(U * Lp + R * Ls, nq * D).bfloat16().cuda()
    do_d = torch.zeros(R, L, nq * D, dtype=torch.bfloat16, device="cuda")
    do_d[::G, :Lp] = do_buf[:U * Lp].view(U, Lp, nq * D)
    do_d[:, Lp:] = do_buf[U * Lp:].view(R, Ls, nq * D)
    do_d = do_d.view(R * L, nq * D)
    g_d = torch.zeros(R * L, W, dtype=torch.bfloat16, device="cuda")
    ops.attn_bwd(*views(dense), o_d, do_d, lse_d, *views(g_d), R, L, nq, nkv, D, kv_start=ks_d, kv_end=kv_end)

    def shared_bwd():
        g = torch.zeros_like(buf)
        ops.attn_bwd_shared(*views(buf), o_s, do_buf, (lse_p, lse_s), *views(g), U, G, Lp, Ls, nq, nkv, D, kv_start, kv_end)
        return g
    g_s = shared_bwd()
    g_d3 = g_d.view(R, L, W)
    assert torch.equal(g_s[:U * Lp, qo:ko].view(U, Lp, nq * D), g_d3[::G, :Lp, qo:ko]), "prefix dQ"
    assert torch.equal(g_s[U * Lp:].view(R, Ls, W), g_d3[:, Lp:]), "suffix dQ / dK / dV"
    if G == 1:
        assert torch.equal(g_s[:U * Lp].view(U, Lp, W), g_d3[:, :Lp]), "G = 1 prefix dK / dV"
    assert torch.equal(shared_bwd(), g_s), "not bit-reproducible"
    # ---- fp32 autograd on the shared semantics: prefix rows are one leaf per group, seen by all G rows
    x = buf.float().clone().requires_grad_(True)
    xd = torch.cat([torch.cat([x[:U * Lp].view(U, Lp, W)[r // G], x[U * Lp:].view(R, Ls, W)[r]]) for r in range(R)]).view(R, L, W)
    qf = xd[..., qo:ko].view(R, L, nq, D).transpose(1, 2)
    kf = xd[..., ko:vo].view(R, L, nkv, D).transpose(1, 2).repeat_interleave(nq // nkv, 1)
    vf = xd[..., vo:].view(R, L, nkv, D).transpose(1, 2).repeat_interleave(nq // nkv, 1)
    j = torch.arange(L, device="cuda")
    ok = ((j[None, None, None, :] >= ks_d[:, None, None, None]) & (j[None, None, None, :] < kv_end[:, None, None, None])
          & (j[None, None, None, :] <= j[None, None, :, None]))
    p = torch.softmax(((qf @ kf.transpose(-1, -2)) * D ** -0.5).masked_fill(~ok, float("-inf")), -1).nan_to_num(0.0)
    out = (p @ vf).transpose(1, 2).reshape(R * L, nq * D)
    out.backward(do_d.float())
    for name, sl in (("dq", slice(qo, ko)), ("dk", slice(ko, vo)), ("dv", slice(vo, W))):
        r = _rel(g_s[:, sl], x.grad[:, sl])
        assert r < 2e-2, f"{name} rel err {r}"
        if Lp:
            rp = _rel(g_s[:U * Lp, sl], x.grad[:U * Lp, sl])
            assert rp < 2e-2, f"prefix {name} rel err {rp}"


# ---------------------------------------------------------------------------------------------------------------- model
def _cfgs(text, depth=2):
    from bioreason_b200.configs import text_config, dna_config
    tc, dc = text_config(text), dna_config("nt-v2-500m" if text != "tiny" else "tiny")
    tc.num_hidden_layers = depth
    if hasattr(tc, "layer_types"):
        tc.layer_types = tc.layer_types[:depth]
    dc.num_hidden_layers = depth
    return tc, dc


def _grpo_batch(tc, dc, G, U, C, *, n_seq, dna_len, text_len, seed, pad_to=None, eos_rows=()):
    """U prompts x G rows [prompt | completion] (prompt rows of a group identical) with per-row EOS truncation."""
    from oracle.models import synth_batch
    parts = [synth_batch(tc, dc, batch=G, n_seq=n_seq, dna_len=dna_len, text_len=text_len[u] if isinstance(text_len, list) else text_len,
                         seed=seed + u, same_prompt=True, pad_to=pad_to) for u in range(U)]
    P = max(p["input_ids"].shape[1] for p in parts)
    ids, am, dna_i, dna_m, bim = [], [], [], [], []
    for u, p in enumerate(parts):
        w = p["input_ids"].shape[1]
        ids.append(torch.cat([torch.full((G, P - w), tc.pad_token_id), p["input_ids"]], 1))
        am.append(torch.cat([torch.zeros(G, P - w, dtype=torch.long), p["attention_mask"]], 1))
        dna_i.append(p["dna_tokenized"]["input_ids"]); dna_m.append(p["dna_tokenized"]["attention_mask"])
        bim += [b + u * G for b in p["batch_idx_map"]]
    R = U * G
    comp = torch.randint(0, tc.eos_token_id, (R, C), generator=torch.Generator().manual_seed(seed + 99))
    cmask = torch.ones(R, C, dtype=torch.long)
    for r, n in eos_rows:
        cmask[r, n:] = 0
    input_ids = torch.cat([torch.cat(ids), comp], 1).cuda()
    mask = torch.cat([torch.cat(am), cmask], 1).cuda()
    mm = dict(dna_tokenized=dict(input_ids=torch.cat(dna_i).cuda(), attention_mask=torch.cat(dna_m).cuda()), batch_idx_map=bim)
    return input_ids, mask, mm, P, cmask.cuda()


def _run(m, ids, mask, mm, C, wgt, G, lora="policy"):
    from bioreason_b200 import training
    m.zero_grad_buffers()
    lp, ctx = training.policy_forward(m, ids, mask, mm["dna_tokenized"], mm["batch_idx_map"], C, lora=lora, group_size=G)
    if lora == "policy":
        training.policy_backward(m, ctx, wgt)
    del ctx
    return lp, m._lora.flat_grad.clone(), m._proj_grad_w.clone(), m._proj_grad_b.clone()


def _model(tc, dc, seed):
    from bioreason_b200.models import DNALLMModel
    from oracle.models import build_oracle
    m = DNALLMModel.from_oracle(build_oracle(tc, dc, seed=seed))
    lora = m.enable_lora(r=16, alpha=32.0, seed=3)
    with torch.no_grad():
        for p in lora.params[1::2]:
            p.normal_(0, 0.01)
    m.sync_adapters(rollout=False)
    return m


@pytest.mark.parametrize("name,kw", [
    ("tiny_dna_in_tail", dict(U=2, G=4, C=40, n_seq=1, dna_len=40, text_len=80, seed=3, eos_rows=[(1, 3), (6, 1)])),
    ("tiny_padded", dict(U=2, G=2, C=33, n_seq=2, dna_len=12, text_len=[30, 90], seed=4, pad_to=150, eos_rows=[(0, 10)])),
])
def test_policy_logps_and_grads_tiny(name, kw):
    """group_size: log-probs bit-identical to the dense path (policy and reference weights); gradients within 1 % of the dense path
    (the prefix sums change the fp32 order); the backward is bit-reproducible."""
    tc, dc = _cfgs("tiny")
    kw = dict(kw)
    G, U, C = kw.pop("G"), kw.pop("U"), kw.pop("C")
    ids, mask, mm, P, cmask = _grpo_batch(tc, dc, G, U, C, **kw)
    assert 64 * ((P - 1) // 64) > 0
    dna_slots = (ids[0, :P] == tc.dna_token_ids[1]).nonzero().flatten()
    if name == "tiny_dna_in_tail":
        Lp = 64 * ((P - 1) // 64)
        assert (dna_slots < Lp).any() and (dna_slots >= Lp).any()          # DNA features on both sides of the prefix boundary
    m = _model(tc, dc, seed=7)
    wgt = (torch.randn(U * G, C, generator=torch.Generator().manual_seed(5)).cuda() * cmask)
    lp_d, gd, pwd, pbd = _run(m, ids, mask, mm, C, wgt, None)
    lp_s, gs, pws, pbs = _run(m, ids, mask, mm, C, wgt, G)
    assert torch.equal(lp_s, lp_d)
    ref_d = _run(m, ids, mask, mm, C, wgt, None, lora=None)[0]
    ref_s = _run(m, ids, mask, mm, C, wgt, G, lora=None)[0]
    assert torch.equal(ref_s, ref_d)
    print(f"{name}: shared vs dense LoRA grad rel {_rel(gs, gd):.2e}, projector dW {_rel(pws, pwd):.2e} db {_rel(pbs, pbd):.2e}")
    assert _rel(gs, gd) < 1e-2 and _rel(pws, pwd) < 1e-2 and _rel(pbs, pbd) < 1e-2
    lp_s2, gs2, pws2, _ = _run(m, ids, mask, mm, C, wgt, G)
    assert torch.equal(lp_s2, lp_s) and torch.equal(gs2, gs) and torch.equal(pws2, pws)


def test_policy_config_c_geometry():
    """Config (c) geometry (1 prompt x G = 8, P = 1852, C = 512, L = 2364), Qwen3-4B widths, depth 2: log-probs bit-identical to the dense
    path for the policy and the reference weights; LoRA / projector gradients within 3 % of the fp32 oracle."""
    import sys, os
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_gpu_bench_shapes import _build_pair, _cuda_batch, _grad_report, _oracle_logps
    from oracle.models import synth_batch
    from bioreason_b200 import training
    tc, dc = _cfgs("qwen3-4b")
    oracle, m, lora = _build_pair(tc, dc, seed=31)
    G, C = 8, 512
    batch = synth_batch(tc, dc, batch=G, n_seq=2, dna_len=668, text_len=512, seed=8, same_prompt=True)
    comp = torch.randint(0, tc.eos_token_id, (G, C), generator=torch.Generator().manual_seed(9))
    ids = torch.cat([batch["input_ids"], comp], 1).cuda()
    cmask = torch.ones(G, C, dtype=torch.long); cmask[1, -37:] = 0; cmask[5, -200:] = 0
    mask = torch.cat([batch["attention_mask"], cmask], 1).cuda()
    wgt = (torch.randn(G, C, generator=torch.Generator().manual_seed(10)) * cmask).cuda()
    cb = _cuda_batch(batch)
    mm = dict(dna_tokenized=cb["dna_tokenized"], batch_idx_map=cb["batch_idx_map"])

    def dense_chunked():
        lps = []
        for lo in range(0, G, 2):
            idx = [i for i, b in enumerate(mm["batch_idx_map"]) if lo <= b < lo + 2]
            dna = {k: v[idx] for k, v in mm["dna_tokenized"].items()}
            lp_c, ctx = training.policy_forward(m, ids[lo:lo + 2], mask[lo:lo + 2], dna, [mm["batch_idx_map"][i] - lo for i in idx], C)
            training.policy_backward(m, ctx, wgt[lo:lo + 2])
            del ctx
            lps.append(lp_c)
        return torch.cat(lps)

    def shared():
        lp, ctx = training.policy_forward(m, ids, mask, mm["dna_tokenized"], mm["batch_idx_map"], C, group_size=G)
        training.policy_backward(m, ctx, wgt)
        del ctx
        return lp

    m.zero_grad_buffers()
    lp_d = dense_chunked()
    gd, pwd = lora.flat_grad.clone(), m._proj_grad_w.clone()
    m.zero_grad_buffers()
    lp_s = shared()
    assert torch.equal(lp_s, lp_d)
    with torch.no_grad():
        r_d = training.policy_forward(m, ids, mask, mm["dna_tokenized"], mm["batch_idx_map"], C, save=False, lora=None)[0]
        r_s = training.policy_forward(m, ids, mask, mm["dna_tokenized"], mm["batch_idx_map"], C, save=False, lora=None, group_size=G)[0]
    assert torch.equal(r_s, r_d)
    print(f"(c) shared vs dense: LoRA grad rel {_rel(lora.flat_grad, gd):.2e}, projector dW {_rel(m._proj_grad_w, pwd):.2e}")
    g1, pw1 = lora.flat_grad.clone(), m._proj_grad_w.clone()
    # fp32 oracle, row by row
    for r in range(G):
        lp_r = _oracle_logps(oracle, ids[r:r + 1], mask[r:r + 1], dict(dna_tokenized={k: v[2 * r:2 * r + 2] for k, v in mm["dna_tokenized"].items()},
                                                                       batch_idx_map=[0, 0]), C)
        (lp_r * wgt[r:r + 1]).sum().backward()
    worst, wname, rw, rb = _grad_report(m, oracle)
    print(f"(c) shared grads vs fp32 oracle: worst LoRA rel err {worst:.4f} ({wname}); projector dW {rw:.4f} db {rb:.4f}")
    assert worst < 0.03 and rw < 0.03 and rb < 0.03
    m.zero_grad_buffers()
    assert torch.equal(shared(), lp_s)
    assert torch.equal(lora.flat_grad, g1) and torch.equal(m._proj_grad_w, pw1), "shared backward is not run-to-run reproducible"


def test_dropout_refused():
    from bioreason_b200 import training
    from bioreason_b200.trainer import DNALLMGRPOConfig, DNALLMGRPOTrainer
    tc, dc = _cfgs("tiny")
    ids, mask, mm, P, _ = _grpo_batch(tc, dc, 2, 1, 8, n_seq=1, dna_len=10, text_len=80, seed=1)
    m = _model(tc, dc, seed=2)
    m.set_lora_dropout(0.1, seed=1)
    with pytest.raises(ValueError, match="dropout"):
        training.policy_forward(m, ids, mask, mm["dna_tokenized"], mm["batch_idx_map"], 8, dropout=True, group_size=2)
    m.set_lora_dropout(0.0, seed=1)
    cfg = DNALLMGRPOConfig(num_generations=2, per_device_train_batch_size=2, share_prompt_prefix=True, apply_lora_dropout=True)
    with pytest.raises(ValueError, match="apply_lora_dropout"):
        DNALLMGRPOTrainer(m, [lambda completion_ids, **k: completion_ids.float().sum(1)], cfg)


# ---------------------------------------------------------------------------------------------------------------- trainer
def _reward(completion_ids, **kw):
    return (completion_ids % 7 == 0).float().sum(1)


@pytest.mark.parametrize("case", ["mu2_beta0", "ragged_e", "half_groups"])
def test_training_step_flag_on_off(case):
    """One training_step with fixed uniforms and rewards, share_prompt_prefix on and off with equal chunking: same loss and metrics,
    gradients within the bar."""
    from bioreason_b200.trainer import DNALLMGRPOConfig, DNALLMGRPOTrainer
    tc, dc = _cfgs("tiny")
    if case == "mu2_beta0":
        G, U, C, kw, extra = 4, 2, 24, dict(n_seq=1, dna_len=30, text_len=90, seed=11), dict(num_iterations=2, beta=0.0)
        rows, mr = G * U, 4
    elif case == "ragged_e":
        G, U, C, kw, extra = 2, 3, 20, dict(n_seq=2, dna_len=20, text_len=[40, 120, 75], seed=12), dict()
        rows, mr = G * U, 2
    else:                                                                  # one rank's 2 rows of a G = 4 group
        G, U, C, kw, extra = 2, 1, 24, dict(n_seq=1, dna_len=16, text_len=100, seed=13), dict()
        rows, mr = 2, 2
    ids, mask, mm, P, _ = _grpo_batch(tc, dc, G, U, C, **kw)
    base = _model(tc, dc, seed=9)
    u = torch.rand(C, rows, generator=torch.Generator().manual_seed(0))
    results = {}
    for flag in (False, True):
        m = copy.deepcopy(base)
        cfg = DNALLMGRPOConfig(num_generations=G if case != "half_groups" else 2, max_completion_length=C, per_device_train_batch_size=rows,
                               learning_rate=1e-3, lora_r=16, lora_alpha=32.0, micro_rows=mr, share_prompt_prefix=flag, **extra)
        tr = DNALLMGRPOTrainer(m, [_reward], cfg)
        batch = dict(input_ids=ids[:, :P].cpu(), attention_mask=mask[:, :P].cpu(), dna_tokenized={k: v.cpu() for k, v in mm["dna_tokenized"].items()},
                     batch_idx_map=mm["batch_idx_map"])
        inp = tr._generate_and_score_completions(batch, m, uniforms=u.cuda())
        if flag:
            assert inp["local_group_size"] == G
        m.zero_grad_buffers()
        tr._step = 0
        loss = tr.compute_loss(m, inp)
        results[flag] = dict(loss=loss.item(), old=inp["old_per_token_logps"], ref=inp["ref_per_token_logps"],
                             grad=m._lora.flat_grad.clone(), pw=m._proj_grad_w.clone(), met={k: [float(x) for x in v] for k, v in tr._metrics.items()})
    a, b = results[False], results[True]
    assert a["loss"] == b["loss"]
    assert a["met"] == b["met"]
    for k in ("old", "ref"):
        assert (a[k] is None and b[k] is None) or torch.equal(a[k], b[k])
    print(f"{case}: flag on vs off LoRA grad rel {_rel(b['grad'], a['grad']):.2e}, projector dW {_rel(b['pw'], a['pw']):.2e}")
    assert _rel(b["grad"], a["grad"]) < 1e-2 and _rel(b["pw"], a["pw"]) < 1e-2


def test_micro_rows_must_hold_whole_groups():
    from bioreason_b200.trainer import DNALLMGRPOConfig, DNALLMGRPOTrainer
    tc, dc = _cfgs("tiny")
    G, C = 4, 8
    ids, mask, mm, P, _ = _grpo_batch(tc, dc, G, 1, C, n_seq=1, dna_len=10, text_len=80, seed=1)
    m = _model(tc, dc, seed=2)
    cfg = DNALLMGRPOConfig(num_generations=G, max_completion_length=C, per_device_train_batch_size=G, micro_rows=3, share_prompt_prefix=True)
    tr = DNALLMGRPOTrainer(m, [_reward], cfg)
    batch = dict(input_ids=ids[:, :P].cpu(), attention_mask=mask[:, :P].cpu(), dna_tokenized={k: v.cpu() for k, v in mm["dna_tokenized"].items()},
                 batch_idx_map=mm["batch_idx_map"])
    inp = tr._generate_and_score_completions(batch, m, uniforms=torch.rand(C, G, generator=torch.Generator().manual_seed(0)).cuda())
    with pytest.raises(ValueError, match="micro_rows"):
        tr.compute_loss(m, inp)
