"""The GRPO objectives of later TRL releases on CPU: the float64 restatement in grpo_objective_ref.py against the oracle's loss and its
one-bug variants; the config fields and TrlParser; and DNALLMGRPOTrainer.compute_loss with the CUDA ops replaced by the restatement
(row chunks, gradient accumulation, num_iterations > 1, the defaults' calls, and the dapo normaliser under gloo at world 2)."""
import collections
import contextlib
import math
import os
import socket
import types

import pytest
import torch

from grpo_objective_ref import VARIANTS, advantages, entropy_keep, objective_with_grad, token_terms, truncated_mask
from oracle import grpo as og

B, P, C, MAXLEN = 8, 5, 12, 16
RTOL = 2e-5                                                  # the GPU kernel's bar


# ------------------------------------------------------------------ 1. the restatement
@pytest.mark.parametrize("case,beta,lo,hi,use_old", [("mu1", 0.04, 0.2, 0.2, False), ("mu2", 0.04, 0.2, 0.2, True),
                                                     ("mu2_nokl", 0.0, 0.2, 0.2, True), ("mu2_asym", 0.1, 0.1, 0.3, True)])
def test_defaults_are_the_oracle_loss(golden, case, beta, lo, hi, use_old):
    G = golden["G"]
    old = G["old"].double() if use_old else None
    ref = G["ref"].double() if beta > 0 else None
    got = objective_with_grad(G["lp"], old, ref, G["adv"].double(), G["mask"], beta, lo, hi)
    x = G["lp"].double().clone().requires_grad_(True)
    want, kl, clip = og.grpo_loss(x, old, ref, G["adv"].double(), G["mask"], beta, lo, hi)
    want.backward()
    torch.testing.assert_close(got["loss"], want.detach(), rtol=1e-14, atol=0)
    torch.testing.assert_close(got["dlp"], x.grad, rtol=1e-13, atol=1e-18)
    assert abs(got["clip"].item() - clip.item()) < 1e-7                  # the oracle takes the ratio in fp32
    if beta > 0:
        assert abs(got["kl"].item() - kl.item()) < 1e-12
    assert abs(got["loss"].item() - G[case]["loss"].item()) <= 2e-6 * abs(G[case]["loss"].item())   # the reference run's fp32 value


def _case(seed=3, mu=2, beta=0.04, width=C, rows=B):
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(rows, width, generator=g, dtype=torch.float64) * 3
    old = lp + torch.randn(rows, width, generator=g, dtype=torch.float64) * 0.3 if mu > 1 else None
    ref = lp + torch.randn(rows, width, generator=g, dtype=torch.float64) * 0.2 if beta > 0 else None
    samp = lp + torch.randn(rows, width, generator=g, dtype=torch.float64) * 0.8
    adv = torch.randn(rows, generator=g, dtype=torch.float64)
    cmask = (torch.arange(width)[None, :] < torch.randint(2, width + 1, (rows, 1), generator=g)).int()
    return lp, old, ref, samp, adv, cmask


def _differs(a, b):
    """Farther apart than the GPU kernel's tolerance, in the loss or in some gradient element."""
    la, lb = a["loss"].item(), b["loss"].item()
    return abs(la - lb) > RTOL * max(1.0, abs(lb)) or not torch.allclose(a["dlp"], b["dlp"], rtol=RTOL, atol=1e-8)


@pytest.mark.parametrize("variant", VARIANTS)
def test_one_bug_variants_are_caught(variant):
    lp, old, ref, samp, adv, cmask = _case()
    kw = dict(loss_type="grpo")
    if variant.startswith("seq_"):
        kw.update(level="sequence")
    elif variant == "dr_grpo_trimmed_width":
        kw.update(loss_type="dr_grpo", max_completion_length=MAXLEN)
    elif variant == "dapo_without_world":
        kw.update(loss_type="dapo", num_items=int(cmask.sum()) * 2, world=2)
    elif variant == "delta_on_c2":
        kw.update(delta=1.1)
    elif variant in ("batch_std_biased", "none_still_divides"):
        r = torch.randn(B, 2, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
        scale = "batch" if variant == "batch_std_biased" else "none"
        good, bad = advantages(r, 4, scale)[0], advantages(r, 4, scale, variant=variant)[0]
        assert not torch.allclose(good, bad, rtol=RTOL, atol=1e-6)
        return
    elif variant == "threshold_without_truncation":
        ids = torch.randint(3, 50, (B, C), generator=torch.Generator().manual_seed(2))
        ids[::2, 5] = 1                                        # EOS in the even rows; the odd rows are truncated
        tmask, _ = truncated_mask(ids, 1)
        pre = (torch.arange(C)[None, :] < truncated_mask(ids, 1)[1][:, None]).int()
        ent = torch.rand(B, C, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
        ent[1::2] += 1.0                                       # truncated rows hold the high entropies
        keep_good = entropy_keep(ent, tmask, 0.3, pre)
        keep_bad = entropy_keep(ent, tmask, 0.3, pre, variant=variant)
        good = objective_with_grad(lp, old, ref, adv, tmask, 0.04, 0.2, 0.28, keep=keep_good)
        bad = objective_with_grad(lp, old, ref, adv, tmask, 0.04, 0.2, 0.28, keep=keep_bad)
        assert _differs(bad, good)
        return
    good = objective_with_grad(lp, old, ref, adv, cmask, 0.04, 0.2, 0.28, **kw)
    bad = objective_with_grad(lp, old, ref, adv, cmask, 0.04, 0.2, 0.28, variant=variant, **kw)
    assert _differs(bad, good)


def test_advantage_modes_and_truncated_mask():
    r = torch.tensor([[1.0], [1.0], [1.0], [1.0], [0.0], [1.0], [2.0], [3.0]], dtype=torch.float64)
    adv, sd, zero = advantages(r, 4, "group")
    torch.testing.assert_close(adv, og.group_advantages(r, 4), rtol=1e-15, atol=0)
    assert zero.tolist() == [True] * 4 + [False] * 4
    adv_b, sd_b, zero_b = advantages(r, 4, "batch")
    assert torch.allclose(sd_b, r.sum(1).std().expand(8)) and not zero_b.any()
    adv_n, _, _ = advantages(r, 4, "none")
    assert adv_n.tolist() == [0, 0, 0, 0, -1.5, -0.5, 0.5, 1.5]
    ids = torch.tensor([[5, 1, 7, 1], [5, 6, 7, 8], [1, 2, 2, 2]])
    m, n = truncated_mask(ids, 1)
    assert m.tolist() == [[1, 1, 0, 0], [0, 0, 0, 0], [1, 0, 0, 0]] and n.tolist() == [2, 4, 1]
    torch.testing.assert_close(m[[0, 2]], og.completion_mask_from_eos(ids, 1)[[0, 2]])


def test_sequence_level_equals_token_level_at_mu1():
    """mu = 1: every ratio is 1 at both levels, and with w = k = 1 the gradients agree."""
    lp, _, ref, _, adv, cmask = _case(mu=1)
    for lt in ("grpo", "bnpo", "dr_grpo", "dapo"):
        kw = dict(loss_type=lt, max_completion_length=MAXLEN, num_items=40, world=1)
        a = objective_with_grad(lp, None, ref, adv, cmask, 0.04, 0.2, 0.28, **kw)
        b = objective_with_grad(lp, None, ref, adv, cmask, 0.04, 0.2, 0.28, level="sequence", **kw)
        torch.testing.assert_close(a["loss"], b["loss"], rtol=1e-14, atol=0)
        torch.testing.assert_close(a["dlp"], b["dlp"], rtol=1e-12, atol=1e-18)


# ------------------------------------------------------------------ 2. config
def test_config_fields_and_validation():
    from bioreason_b200.trainer import DNALLMGRPOConfig
    c = DNALLMGRPOConfig()
    assert (c.loss_type, c.importance_sampling_level, c.delta, c.scale_rewards, c.mask_truncated_completions) == ("grpo", "token", None, "group", False)
    for v, want in ((True, "group"), (False, "none"), ("true", "group"), ("False", "none"), ("batch", "batch"), ("none", "none")):
        assert DNALLMGRPOConfig(scale_rewards=v).scale_rewards == want
    assert DNALLMGRPOConfig(delta=4.0).delta == 4.0 and DNALLMGRPOConfig(delta=2).delta == 2
    bad = [dict(loss_type="dpo"), dict(importance_sampling_level="seq"), dict(scale_rewards="rows"), dict(delta=0.0), dict(delta=-1.0),
           dict(delta=math.inf), dict(delta=float("nan")), dict(delta="4"), dict(mask_truncated_completions=True, suppress_eos=True)]
    for kw in bad:
        with pytest.raises(ValueError):
            DNALLMGRPOConfig(**kw)


def test_trl_parser_reads_the_new_fields():
    from compat.trl import TrlParser
    from bioreason_b200.trainer import DNALLMGRPOConfig
    (c,) = TrlParser([DNALLMGRPOConfig]).parse_args_and_config(["--loss_type", "dr_grpo", "--scale_rewards", "batch", "--delta", "4",
                                                                 "--importance_sampling_level", "sequence", "--mask_truncated_completions"])
    assert (c.loss_type, c.scale_rewards, c.delta, c.importance_sampling_level, c.mask_truncated_completions) == \
        ("dr_grpo", "batch", 4.0, "sequence", True)
    (c,) = TrlParser([DNALLMGRPOConfig]).parse_args_and_config(["--scale_rewards", "false"])
    assert c.scale_rewards == "none"
    (c,) = TrlParser([DNALLMGRPOConfig]).parse_args_and_config(["--scale_rewards", "True"])
    assert c.scale_rewards == "group"


# ------------------------------------------------------------------ 3. trainer control flow, ops replaced
def _fake_trainer(micro_rows, mu=1, ga=1, beta=0.04, **fields):
    from bioreason_b200.trainer.grpo_trainer import DNALLMGRPOTrainer, TrainerState
    t = object.__new__(DNALLMGRPOTrainer)
    t.args = types.SimpleNamespace(micro_rows=micro_rows, gradient_accumulation_steps=ga, **fields)
    t.beta, t.num_iterations, t.epsilon_low, t.epsilon_high = beta, mu, 0.2, 0.28
    t.max_completion_length = MAXLEN
    t.state = TrainerState()
    t.global_step, t._step = 0, 0
    t._buffered_inputs = [None] * ga
    t._metrics = collections.defaultdict(list)
    t.timings = collections.defaultdict(float)
    t._ev = []
    t._mark = lambda phase: contextlib.nullcontext()
    return t


def _inputs(lp, old, ref, samp, adv, cmask, n_items=None):
    rows = lp.shape[0]
    prompt_ids = torch.zeros(rows, P, dtype=torch.long)
    prompt_ids[:, 0] = torch.arange(rows)                              # row id smuggled in the first prompt token
    d = dict(prompt_ids=prompt_ids, prompt_mask=torch.ones(rows, P, dtype=torch.long), completion_ids=torch.zeros_like(cmask).long(),
             completion_mask=cmask, old_per_token_logps=old, ref_per_token_logps=ref, advantages=adv, sampling_per_token_logps=samp,
             multimodal_inputs=dict(dna_tokenized=None, batch_idx_map=[]))
    if n_items is not None:
        d["num_items_in_batch"] = n_items
    return d


def fake_objective_raw(lp, old_lp, ref_lp, adv, mask, beta, lo, hi, *, norm_rows=0, norm=None, sequence_level=False, delta=None,
                       rollout_lp=None, is_cap=2.0, entropy=None, tau=None, want_grad=True, log=None):
    """ops.grpo_objective_raw restated in float64 (sums over the call's rows, like the kernel)."""
    x = lp.double().clone().requires_grad_(True)
    keep = None if entropy is None else entropy >= tau
    T = token_terms(x, old_lp, ref_lp, adv, mask, beta, lo, hi, level="sequence" if sequence_level else "token", delta=delta,
                    rollout=rollout_lp, cap=is_cap, keep=keep)
    m = T["m"]
    if norm_rows:
        loss = ((T["per"] * m).sum(1) / T["nrm"]).sum() / norm_rows
    else:
        loss = (T["per"] * m).sum() / norm.double()[0]
    loss.backward()
    if log is not None:
        log.append(dict(rows=lp.shape[0], norm_rows=norm_rows, norm=None if norm is None else float(norm[0])))
    a, c1, l1, l2 = T["a"], T["c1"], T["l1"], T["l2"]
    low = ((c1 < 1 - lo) & (a < 0)).double()
    high = ((c1 > 1 + hi) & (a > 0)).double()
    kl = torch.zeros(()) if T["kl"] is None else torch.where(T["cnt"] > 0, (T["kl"] * m).sum(1) / T["nrm"], torch.zeros_like(T["cnt"])).sum()
    s = lambda v: (v * m).sum().detach()
    out7 = torch.stack([loss.detach(), kl.detach().double(), s((l1 < l2).double()), s(low), s(high), s(low + high), m.sum()])
    is_sums = None if rollout_lp is None else T["is_stats"] * T["tot"]
    ent_sum = None if entropy is None else (entropy * m).sum().reshape(1)
    return out7, is_sums, ent_sum, x.grad if want_grad else None


def _patch(monkeypatch, lp_full, got_grad, log=None):
    from bioreason_b200 import ops, training

    def fake_policy_forward(model, ids, mask, dna, idx_map, keep_last, save=True, **kw):
        rows = ids[:, 0].tolist()
        return lp_full[rows].clone(), types.SimpleNamespace(rows=rows)

    def fake_backward(model, ctx, dlp, on_layer_done=None):
        got_grad[ctx.rows] += dlp

    def no_old_loss(*a, **k):
        raise AssertionError("an existing loss entry point was called on the new objective path")

    monkeypatch.setattr(training, "policy_forward", fake_policy_forward)
    monkeypatch.setattr(training, "policy_backward", fake_backward)
    monkeypatch.setattr(ops, "grpo_objective_raw", lambda *a, **k: fake_objective_raw(*a, log=log, **k))
    for name in ("grpo_loss_raw", "grpo_loss_is_raw", "grpo_loss_ent_raw"):
        monkeypatch.setattr(ops, name, no_old_loss)


OBJECTIVES = [dict(loss_type="grpo", importance_sampling_level="sequence"), dict(loss_type="grpo", delta=1.1),
              dict(loss_type="bnpo"), dict(loss_type="dr_grpo"), dict(loss_type="dapo", importance_sampling_level="sequence"),
              dict(loss_type="dapo", delta=1.25)]


def _want(lp, old, ref, samp, adv, cmask, fields, tis, n_items=None):
    return objective_with_grad(lp, old, ref, adv, cmask, 0.04, 0.2, 0.28, loss_type=fields["loss_type"],
                               level=fields.get("importance_sampling_level", "token"), delta=fields.get("delta"),
                               rollout=samp if tis else None, cap=2.0, max_completion_length=MAXLEN,
                               num_items=int(cmask.sum()) if n_items is None else n_items, world=1)


@pytest.mark.parametrize("tis", [False, True])
@pytest.mark.parametrize("micro_rows", [B, 3, 1])                      # 1, 3 and 8 row chunks
@pytest.mark.parametrize("fields", OBJECTIVES, ids=lambda f: "-".join(str(v) for v in f.values()))
def test_chunked_objective_matches_full_batch(monkeypatch, fields, micro_rows, tis):
    from bioreason_b200.trainer import grpo_trainer as gt
    lp, old, ref, samp, adv, cmask = _case()
    cmask[2] = 0                                                       # an empty row
    got_grad, log = torch.zeros(B, C, dtype=torch.float64), []
    _patch(monkeypatch, lp, got_grad, log)
    t = _fake_trainer(micro_rows, mu=2, rollout_is_correction=tis, rollout_is_cap=2.0, **fields)
    loss = gt.DNALLMGRPOTrainer.compute_loss(t, None, _inputs(lp, old, ref, samp, adv, cmask))
    want = _want(lp, old, ref, samp, adv, cmask, fields, tis)
    assert abs(loss.item() - want["loss"].item()) < 1e-6
    torch.testing.assert_close(got_grad, want["dlp"], rtol=1e-12, atol=1e-15)
    assert len(log) == math.ceil(B / micro_rows)
    if fields["loss_type"] == "grpo":
        assert all(e["norm_rows"] == B for e in log)                   # the whole local batch, not the chunk
    for k in ("clip", "low", "high", "region"):                        # token means, exact across chunks
        name = "clip_ratio" if k == "clip" else f"clip_ratio/{k}_mean"
        assert abs(float(t._metrics[name][0]) - want[k].item()) < 1e-6, name
    assert abs(float(t._metrics["kl"][0]) - want["kl"].item()) < 1e-6
    if tis:
        for i, name in enumerate(("ratio_mean", "capped_frac", "logp_diff", "kl")):
            assert abs(float(t._metrics[f"rollout_is/{name}"][0]) - want["is_stats"][i].item()) < 1e-6


def test_delta_and_sequence_metrics_are_live(monkeypatch):
    """The case above really has clipped tokens on both sides, and delta binds."""
    lp, old, ref, samp, adv, cmask = _case()
    w = _want(lp, old, ref, samp, adv, cmask, dict(loss_type="grpo"), False)
    d = _want(lp, old, ref, samp, adv, cmask, dict(loss_type="grpo", delta=1.1), False)
    assert w["low"] > 0 and w["high"] > 0 and not torch.allclose(w["dlp"], d["dlp"])


def test_gradient_accumulation_scaling(monkeypatch):
    """ga = 2: the returned loss is the micro-step's loss; the gradient is scaled by 1/ga."""
    from bioreason_b200.trainer import grpo_trainer as gt
    lp, old, ref, samp, adv, cmask = _case()
    got_grad = torch.zeros(B, C, dtype=torch.float64)
    _patch(monkeypatch, lp, got_grad)
    fields = dict(loss_type="dapo", importance_sampling_level="sequence")
    t = _fake_trainer(3, mu=2, ga=2, **fields)
    loss = gt.DNALLMGRPOTrainer.compute_loss(t, None, _inputs(lp, old, ref, samp, adv, cmask))
    want = _want(lp, old, ref, samp, adv, cmask, fields, False)
    assert abs(loss.item() - want["loss"].item()) < 1e-6
    torch.testing.assert_close(got_grad, want["dlp"] / 2, rtol=1e-12, atol=1e-15)


def test_num_items_in_batch_is_buffered_for_mu2(monkeypatch):
    """dapo: the normaliser travels with the buffered inputs, so the second pass over the batch uses it (here a value unlike the
    local mask count, as another rank's tokens would make it); inputs without it get the local count."""
    from bioreason_b200.trainer import grpo_trainer as gt
    lp, old, ref, samp, adv, cmask = _case()
    got_grad, log = torch.zeros(B, C, dtype=torch.float64), []
    _patch(monkeypatch, lp, got_grad, log)
    fields = dict(loss_type="dapo")
    t = _fake_trainer(None, mu=2, **fields)
    n_items = torch.tensor([3.0 * float(cmask.sum())])
    loss1 = gt.DNALLMGRPOTrainer.compute_loss(t, None, _inputs(lp, old, ref, samp, adv, cmask, n_items=n_items))
    t.global_step = 1
    loss2 = gt.DNALLMGRPOTrainer.compute_loss(t, None, {})
    want = _want(lp, old, ref, samp, adv, cmask, fields, False, n_items=int(n_items))
    assert [e["norm"] for e in log] == [float(n_items)] * 2
    assert abs(loss1.item() - want["loss"].item()) < 1e-6 and loss2.item() == loss1.item()
    log.clear()
    t2 = _fake_trainer(None, mu=1, **fields)
    gt.DNALLMGRPOTrainer.compute_loss(t2, None, _inputs(lp, old, ref, samp, adv, cmask))
    assert [e["norm"] for e in log] == [float(cmask.sum())]


@pytest.mark.parametrize("tis", [None, False, True])
def test_defaults_call_todays_ops(monkeypatch, tis):
    """The new fields at their defaults (or absent, as in args that predate them): the existing loss entry point, never the new one."""
    from bioreason_b200 import ops, training
    from bioreason_b200.trainer import grpo_trainer as gt
    lp, old, ref, samp, adv, cmask = _case()
    calls = []

    def fake_loss_raw(lp_, old_lp, ref_lp, adv_, mask_, beta_, lo, hi, want_grad=True):
        calls.append("plain")
        x = lp_.clone().requires_grad_(True)
        loss, kl, clip = og.grpo_loss(x, old_lp, ref_lp, adv_, mask_, beta_, lo, hi)
        loss.backward()
        return torch.stack([loss.detach(), kl.detach(), clip.detach()]), x.grad

    def fake_loss_is_raw(*a, **k):
        calls.append("is")
        return torch.zeros(3, dtype=torch.float64), torch.zeros(4, dtype=torch.float64), torch.zeros_like(a[0])

    def no_new(*a, **k):
        raise AssertionError("grpo_objective_raw called at the defaults")

    monkeypatch.setattr(training, "policy_forward", lambda model, ids, *a, **k: (lp[ids[:, 0].tolist()].clone(), None))
    monkeypatch.setattr(ops, "grpo_loss_raw", fake_loss_raw)
    monkeypatch.setattr(ops, "grpo_loss_is_raw", fake_loss_is_raw)
    monkeypatch.setattr(ops, "grpo_objective_raw", no_new)
    fields = {} if tis is None else dict(rollout_is_correction=tis, loss_type="grpo", importance_sampling_level="token", delta=None,
                                         scale_rewards="group", mask_truncated_completions=False)
    t = _fake_trainer(3, mu=2, **fields)
    gt.DNALLMGRPOTrainer.compute_loss(t, None, _inputs(lp, old, ref, samp, adv, cmask), backward=False)
    assert calls == (["is"] * 3 if tis else ["plain"] * 3)
    assert not any(k.startswith("clip_ratio/") for k in t._metrics)


# ------------------------------------------------------------------ 4. dapo under DP (gloo, world 2)
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _dp_case(rank):
    # rank 0: long completions, rank 1: short ones -> uneven valid counts
    lp, old, ref, samp, adv, cmask = _case(seed=60 + rank, beta=0.0)
    keep = (10, 3)[rank]
    cmask = (torch.arange(C)[None, :] < torch.randint(1, keep + 1, (B, 1), generator=torch.Generator().manual_seed(rank))).int()
    return lp, old, adv, cmask


def _dp_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from bioreason_b200 import ops, training
        from bioreason_b200.trainer.grpo_trainer import DNALLMGRPOTrainer
        lp, old, adv, cmask = _dp_case(rank)
        got = torch.zeros(B, C, dtype=torch.float64)

        def fwd(model, ids, mask, dna, idx_map, keep_last, save=True, **kw):
            rows = ids[:, 0].tolist()
            return lp[rows].clone(), types.SimpleNamespace(rows=rows)

        def bwd(model, ctx, dlp, on_layer_done=None):
            got[ctx.rows] += dlp

        training.policy_forward, training.policy_backward = fwd, bwd
        ops.grpo_objective_raw = fake_objective_raw
        t = _fake_trainer(3, mu=2, beta=0.0, loss_type="dapo")
        DNALLMGRPOTrainer.compute_loss(t, None, _inputs(lp, old, None, None, adv, cmask))
        # the gradient all-reduce averages the ranks' parameter gradients: per row of the global batch, that is dlp / world
        ret[rank] = got / world
    finally:
        dist.destroy_process_group()


def test_dapo_normaliser_is_the_global_token_mean():
    import torch.multiprocessing as mp
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_dp_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    cases = [_dp_case(r) for r in range(2)]
    lp = torch.cat([c[0] for c in cases])
    old = torch.cat([c[1] for c in cases])
    adv = torch.cat([c[2] for c in cases])
    cmask = torch.cat([c[3] for c in cases])
    assert int(cases[0][3].sum()) != int(cases[1][3].sum())
    want = objective_with_grad(lp, old, None, adv, cmask, 0.0, 0.2, 0.28, loss_type="bnpo")       # the global token mean
    torch.testing.assert_close(torch.cat([ret[0], ret[1]]), want["dlp"], rtol=1e-12, atol=1e-15)
