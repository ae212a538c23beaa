"""CPU checks of the entropy feature: the float64 entropy reference and its bound against one-bug variants, the torch.quantile
restatement of the threshold against the installed torch, the config fields, and the trainer's control flow with the CUDA ops replaced
by the float64 restatements in entropy_ref.py (the token mask does not depend on the row chunking; under DP the threshold is the
global one)."""
import collections
import contextlib
import math
import os
import socket
import types

import numpy as np
import pytest
import torch

from entropy_ref import ENTROPY_VARIANTS, RHOS, _tile_entropy, entropy_ref, grpo_loss_ent_with_grad, quantile_ref, threshold_cases
from gemm_ref import lmhead_targets, make_lmhead_inputs, make_lmhead_weight, worst_ratio


def _inputs(V, K, M, family, seed):
    w = make_lmhead_weight(V, K, seed=seed)
    h, _, same_sign = make_lmhead_inputs(family, w, M, lmhead_targets(M, V, seed=seed), seed=seed + 1)
    return h, w, same_sign


@pytest.mark.parametrize("V,K", [(1000, 64), (12289, 96)])
def test_tile_combine_is_within_the_bound(V, K):
    """The kernel's tile-partial algebra (S, U, H = log S - U / S), done in float64, lies far inside the bound of the exact H."""
    for family in ("random", "peaked", "tail_max"):
        h, w, ss = _inputs(V, K, 24, family, 5)
        ref = entropy_ref(h, w, same_sign=ss)
        z = (h.double() @ w.double().T)
        ht = _tile_entropy(z)
        assert worst_ratio(ht, ref["H"], ref["b_H"]) < 0.01
        assert (ht >= 0).all()                                         # log S >= 0 and -U / S >= 0 term by term


@pytest.mark.parametrize("variant", ENTROPY_VARIANTS)
def test_one_bug_variants_exceed_the_bound(variant):
    V, K = 1000, 64
    worst = 0.0
    for family in ("random", "tail_max"):
        h, w, ss = _inputs(V, K, 32, family, 11)
        ref = entropy_ref(h, w, same_sign=ss)
        bad = entropy_ref(h, w, same_sign=ss, variant=variant)
        worst = max(worst, worst_ratio(bad["H"], ref["H"], ref["b_H"]))
    assert worst >= 10.0, (variant, worst)


@pytest.mark.parametrize("rho", RHOS)
def test_quantile_restatement_equals_torch(rho):
    for name, x, m in threshold_cases():
        want = quantile_ref(x, m, 1.0 - rho)
        valid = x[m != 0].float()
        if valid.numel() == 0:
            assert want == np.float32(math.inf), name
            continue
        got = torch.quantile(valid, 1.0 - rho)
        assert np.float32(got.item()).tobytes() == want.tobytes(), (name, rho, got.item(), want)


def test_config_fields():
    from bioreason_b200.trainer import DNALLMGRPOConfig
    c = DNALLMGRPOConfig()
    assert c.top_entropy_quantile == 1.0 and c.log_entropy is False
    for ok in (0.0, 0.2, 1.0):
        assert DNALLMGRPOConfig(top_entropy_quantile=ok).top_entropy_quantile == ok
    for bad in (-0.1, 1.5, float("nan"), math.inf):
        with pytest.raises(ValueError, match="top_entropy_quantile"):
            DNALLMGRPOConfig(top_entropy_quantile=bad)


# ---------------------------------------------------------------------------------------------------------------- trainer logic
B, P, C = 8, 5, 12


def _fake_trainer(micro_rows, rho, log_entropy=False, beta=0.04, tis=False):
    from bioreason_b200.trainer.grpo_trainer import DNALLMGRPOTrainer, TrainerState
    t = object.__new__(DNALLMGRPOTrainer)
    t.args = types.SimpleNamespace(micro_rows=micro_rows, gradient_accumulation_steps=1, top_entropy_quantile=rho,
                                   log_entropy=log_entropy, rollout_is_correction=tis, rollout_is_cap=2.0)
    t.beta, t.num_iterations, t.epsilon_low, t.epsilon_high = beta, 1, 0.2, 0.28
    t.state = TrainerState()
    t.global_step, t._step = 0, 0
    t._buffered_inputs = [None]
    t._metrics = collections.defaultdict(list)
    t.timings = collections.defaultdict(float)
    t._ev = []
    t._mark = lambda phase: contextlib.nullcontext()
    return t


def _case(seed=3, width=C, rows=B, shift=0.0):
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(rows, width, generator=g, dtype=torch.float64) * 3
    ref = lp + torch.randn(rows, width, generator=g, dtype=torch.float64) * 0.2
    ent = (torch.rand(rows, width, generator=g) * 4 + shift).float()
    adv = torch.randn(rows, generator=g, dtype=torch.float64)
    cmask = (torch.arange(width)[None, :] < torch.randint(2, width + 1, (rows, 1), generator=g)).int()
    return lp, ref, ent, adv, cmask


def _batch(ref, adv, cmask, rows=B):
    prompt_ids = torch.zeros(rows, P, dtype=torch.long)
    prompt_ids[:, 0] = torch.arange(rows)                            # row id smuggled in the first prompt token
    return dict(prompt_ids=prompt_ids, prompt_mask=torch.ones(rows, P, dtype=torch.long),
                completion_ids=torch.zeros(rows, cmask.shape[1], dtype=torch.long), completion_mask=cmask, old_per_token_logps=None,
                ref_per_token_logps=ref, advantages=adv, multimodal_inputs=dict(dna_tokenized=None, batch_idx_map=[]))


def _patch(monkeypatch, lp_full, ent_full, log):
    from bioreason_b200 import ops, training

    def fake_policy_forward(model, ids, mask, dna, idx_map, keep_last, save=True, lora="policy", targets=None, want_entropy=False, **kw):
        rows = ids[:, 0].tolist()
        log["fwd"].append((save, tuple(rows), kw.get("row_offset")))
        out = (lp_full[rows].clone(), types.SimpleNamespace(rows=rows))
        return out + (ent_full[rows].clone(),) if want_entropy else out

    def fake_threshold(vals, valid, level):
        log["thr_n"].append(int((valid != 0).sum()))
        return torch.tensor([float(quantile_ref(vals, valid, level))])

    def fake_loss_ent(lp, old, ref, rollout, adv, mask, ent, tau, beta, lo, hi, is_cap=2.0, want_grad=True):
        log["tau"].append(float(tau[0]))
        loss, kl, clip, ent_sum, grad = grpo_loss_ent_with_grad(lp, old, ref, rollout, adv, mask, ent, tau[0], beta, lo, hi, is_cap)
        return torch.stack([loss, kl if kl is not None else torch.zeros((), dtype=loss.dtype), clip]), None, ent_sum.reshape(1), grad

    def fake_backward(model, ctx, dlp, on_layer_done=None):
        log["grad"][ctx.rows] += dlp

    monkeypatch.setattr(training, "policy_forward", fake_policy_forward)
    monkeypatch.setattr(training, "policy_backward", fake_backward)
    monkeypatch.setattr(ops, "entropy_threshold", fake_threshold)
    monkeypatch.setattr(ops, "grpo_loss_ent_raw", fake_loss_ent)
    monkeypatch.setattr(ops, "grpo_loss_raw", lambda *a, **k: (_ for _ in ()).throw(AssertionError("plain loss with entropy on")))


def _run(monkeypatch, micro_rows, rho, log_entropy=False):
    from bioreason_b200.trainer import grpo_trainer as gt
    lp, ref, ent, adv, cmask = _case()
    log = dict(fwd=[], thr_n=[], tau=[], grad=torch.zeros(B, C, dtype=torch.float64))
    _patch(monkeypatch, lp, ent, log)
    t = _fake_trainer(micro_rows, rho, log_entropy)
    loss = gt.DNALLMGRPOTrainer.compute_loss(t, None, _batch(ref, adv, cmask))
    return loss, log, t, (lp, ref, ent, adv, cmask)


@pytest.mark.parametrize("rho", [0.2, 0.5])
def test_mask_does_not_depend_on_micro_rows(monkeypatch, rho):
    runs = {mr: _run(monkeypatch, mr, rho) for mr in (None, 1, 3)}
    loss0, log0, t0, (lp, ref, ent, adv, cmask) = runs[None]
    tau = float(quantile_ref(ent, cmask, 1.0 - rho))
    want, _, _, ent_sum, grad = grpo_loss_ent_with_grad(lp, None, ref, None, adv, cmask, ent, tau, 0.04, 0.2, 0.28)
    kept = ((ent >= tau) & (cmask != 0)).sum().item()
    assert 0 < kept < cmask.sum().item()
    for mr, (loss, log, t, _) in runs.items():
        assert set(log["tau"]) == {tau}, (mr, log["tau"])              # one threshold per call, the same for every chunking
        assert log["thr_n"] == [int(cmask.sum())]                       # over every valid token of the batch, once
        assert abs(loss.item() - want.item()) < 1e-6
        torch.testing.assert_close(log["grad"], grad, rtol=1e-12, atol=1e-15)
        pre = [f for f in log["fwd"] if not f[0]]
        if mr is None:
            assert not pre                                             # one chunk: the loss pass's own entropies
        else:
            assert [r for _, r, _ in pre] == [r for s, r, _ in log["fwd"] if s]     # pre-pass: the loss pass's row chunks
        assert float(t._metrics["entropy/threshold"][0]) == np.float32(tau)
        assert abs(float(t._metrics["entropy"][0]) - (ent_sum / cmask.sum()).item()) < 1e-5


def test_log_entropy_alone_keeps_every_token(monkeypatch):
    loss, log, t, (lp, ref, ent, adv, cmask) = _run(monkeypatch, 3, 1.0, log_entropy=True)
    assert set(log["tau"]) == {-math.inf} and not log["thr_n"]
    assert not [f for f in log["fwd"] if not f[0]]                     # no pre-pass
    assert "entropy" in t._metrics and "entropy/threshold" not in t._metrics


def test_defaults_call_the_plain_loss(monkeypatch):
    """Both fields at their defaults: no entropy is requested and the existing loss call is the one made."""
    from bioreason_b200 import ops, training
    from bioreason_b200.trainer import grpo_trainer as gt
    lp, ref, ent, adv, cmask = _case()
    calls = []
    monkeypatch.setattr(training, "policy_forward", lambda model, ids, *a, **k: (calls.append(k) or (lp[ids[:, 0].tolist()].clone(), None)))
    monkeypatch.setattr(ops, "grpo_loss_raw", lambda lp_, *a, **k: (torch.zeros(3), None))
    monkeypatch.setattr(ops, "grpo_loss_ent_raw", lambda *a, **k: (_ for _ in ()).throw(AssertionError("entropy loss with the fields off")))
    t = _fake_trainer(3, 1.0)
    gt.DNALLMGRPOTrainer.compute_loss(t, None, _batch(ref, adv, cmask), backward=False)
    assert all("want_entropy" not in k for k in calls) and not any(k.startswith("entropy") for k in t._metrics)


# ------------------------------------------------------------------------------------------------------------ DP (gloo, world 2)
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _dp_worker(rank, world, port, rho, ret):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from bioreason_b200 import ops
        from bioreason_b200.trainer.grpo_trainer import DNALLMGRPOTrainer
        ops.entropy_threshold = lambda vals, valid, level: torch.tensor([float(quantile_ref(vals, valid, level))])
        # rank 0 holds low entropies on 12 columns, rank 1 high ones on 7: the local quantiles differ from the global one
        _, _, ent, _, cmask = _case(seed=40 + rank, width=(12, 7)[rank], shift=(0.0, 3.0)[rank])
        t = object.__new__(DNALLMGRPOTrainer)
        tau = DNALLMGRPOTrainer._entropy_threshold(t, ent, cmask, rho)
        ret[rank] = (float(tau[0]), ent, cmask)
    finally:
        dist.destroy_process_group()


def test_dp_threshold_is_global():
    import torch.multiprocessing as mp
    rho = 0.2
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_dp_worker, args=(2, _free_port(), rho, ret), nprocs=2, join=True)
    (tau0, e0, m0), (tau1, e1, m1) = ret[0], ret[1]
    glob = float(quantile_ref(torch.cat([e0.reshape(-1), e1.reshape(-1)]), torch.cat([m0.reshape(-1), m1.reshape(-1)]), 1 - rho))
    local = [float(quantile_ref(e, m, 1 - rho)) for e, m in ((e0, m0), (e1, m1))]
    assert tau0 == tau1 == glob
    assert glob not in local
