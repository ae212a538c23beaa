"""Host logic of the truncated importance-sampling (TIS) correction in DNALLMGRPOTrainer.compute_loss, on CPU: the CUDA ops are
replaced by the float64 restatement in rollout_is_ref.py (and the oracle's loss for the flag-off path); only the trainer's own control
flow runs -- the rollout log-probs reach the loss sliced per row chunk, chunked runs equal the full batch, mu > 1 reuses the buffered
log-probs, and with the flag off the existing loss call is the one made."""
import collections
import math
import types

import pytest
import torch

from oracle import grpo as og
from rollout_is_ref import grpo_loss_is, grpo_loss_is_with_grad

B, P, C = 8, 5, 12


def _fake_trainer(beta, mu, micro_rows, *, tis=None, cap=2.0):
    from bioreason_b200.trainer.grpo_trainer import DNALLMGRPOTrainer, TrainerState
    t = object.__new__(DNALLMGRPOTrainer)
    args = dict(micro_rows=micro_rows, gradient_accumulation_steps=1)
    if tis is not None:
        args.update(rollout_is_correction=tis, rollout_is_cap=cap)
    t.args = types.SimpleNamespace(**args)
    t.beta, t.num_iterations, t.epsilon_low, t.epsilon_high = beta, mu, 0.2, 0.28
    t.state = TrainerState()
    t.global_step, t._step = 0, 0
    t._buffered_inputs = [None]
    t._metrics = collections.defaultdict(list)
    t.timings = collections.defaultdict(float)
    t._ev = []
    t._mark = lambda phase: __import__("contextlib").nullcontext()
    return t


def _case(beta, mu, seed=3):
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(B, C, generator=g, dtype=torch.float64) * 3
    old = lp + torch.randn(B, C, generator=g, dtype=torch.float64) * 0.3 if mu > 1 else None
    ref = lp + torch.randn(B, C, generator=g, dtype=torch.float64) * 0.2 if beta > 0 else None
    samp = lp + torch.randn(B, C, generator=g, dtype=torch.float64) * 0.8          # weights on both sides of the cap
    adv = torch.randn(B, generator=g, dtype=torch.float64)
    cmask = (torch.arange(C)[None, :] < torch.randint(2, C + 1, (B, 1), generator=g)).int()
    return lp, old, ref, samp, adv, cmask


def _inputs(old, ref, samp, adv, cmask):
    prompt_ids = torch.zeros(B, P, dtype=torch.long)
    prompt_ids[:, 0] = torch.arange(B)                                  # row id smuggled in the first prompt token
    d = dict(prompt_ids=prompt_ids, prompt_mask=torch.ones(B, P, dtype=torch.long), completion_ids=torch.zeros(B, C, dtype=torch.long),
             completion_mask=cmask, old_per_token_logps=old, ref_per_token_logps=ref, advantages=adv,
             multimodal_inputs=dict(dna_tokenized=None, batch_idx_map=[]))
    if samp is not None:
        d["sampling_per_token_logps"] = samp
    return d


def _patch(monkeypatch, lp_full, seen, got_grad):
    from bioreason_b200 import ops, training

    def fake_policy_forward(model, ids, mask, dna, idx_map, keep_last, save=True, lora="policy", targets=None, **kw):
        rows = ids[:, 0].tolist()
        return lp_full[rows].clone(), types.SimpleNamespace(rows=rows)

    def fake_loss_is_raw(lp, old_lp, ref_lp, rollout_lp, adv_, mask_, beta_, lo, hi, is_cap, want_grad=True):
        seen.append(rollout_lp.clone())
        loss, kl, clip, stats, grad = grpo_loss_is_with_grad(lp, old_lp, ref_lp, rollout_lp, adv_, mask_, beta_, lo, hi, is_cap)
        return torch.stack([loss, kl if kl is not None else torch.zeros((), dtype=loss.dtype), clip]), stats, grad

    def no_plain_loss(*a, **k):
        raise AssertionError("grpo_loss_raw called with the correction on")

    def fake_backward(model, ctx, dlp, on_layer_done=None):
        got_grad[ctx.rows] += dlp

    monkeypatch.setattr(training, "policy_forward", fake_policy_forward)
    monkeypatch.setattr(training, "policy_backward", fake_backward)
    monkeypatch.setattr(ops, "grpo_loss_is_raw", fake_loss_is_raw)
    monkeypatch.setattr(ops, "grpo_loss_raw", no_plain_loss)


@pytest.mark.parametrize("micro_rows", [None, 1, 3])
@pytest.mark.parametrize("beta,mu", [(0.04, 1), (0.04, 2), (0.0, 2)])
def test_chunked_is_loss_matches_full_batch(monkeypatch, micro_rows, beta, mu):
    from bioreason_b200.trainer import grpo_trainer as gt
    lp, old, ref, samp, adv, cmask = _case(beta, mu)
    seen, got_grad = [], torch.zeros(B, C, dtype=torch.float64)
    _patch(monkeypatch, lp, seen, got_grad)
    t = _fake_trainer(beta, mu, micro_rows, tis=True, cap=2.0)
    loss = gt.DNALLMGRPOTrainer.compute_loss(t, None, _inputs(old, ref, samp, adv, cmask))
    want, kl, clip, stats, grad = grpo_loss_is_with_grad(lp, old, ref, samp, adv, cmask, beta, 0.2, 0.28, 2.0)
    assert abs(loss.item() - want.item()) < 1e-6                         # the trainer accumulates the chunk losses in fp32
    torch.testing.assert_close(got_grad, grad, rtol=1e-12, atol=1e-15)
    # the rollout log-probs reach the loss sliced per row chunk, in order
    mr = micro_rows or B
    assert len(seen) == math.ceil(B / mr)
    assert torch.equal(torch.cat(seen), samp)
    assert {"rollout_is/ratio_mean", "rollout_is/capped_frac", "rollout_is/logp_diff", "rollout_is/kl", "clip_ratio"} <= set(t._metrics)
    if micro_rows is None:                                               # token means: exact for one chunk
        for i, name in enumerate(("ratio_mean", "capped_frac", "logp_diff", "kl")):
            assert abs(float(t._metrics[f"rollout_is/{name}"][0]) - stats[i].item()) < 1e-6
    assert 0 < float(t._metrics["rollout_is/capped_frac"][0]) < 1
    if mu > 1:
        # the second iteration reuses the buffered inputs, rollout log-probs included
        seen.clear()
        t.global_step = 1
        got_grad.zero_()
        loss2 = gt.DNALLMGRPOTrainer.compute_loss(t, None, {})
        assert torch.equal(torch.cat(seen), samp) and abs(loss2.item() - want.item()) < 1e-6


def test_missing_rollout_logps_is_refused(monkeypatch):
    from bioreason_b200.trainer import grpo_trainer as gt
    lp, old, ref, samp, adv, cmask = _case(0.04, 1)
    _patch(monkeypatch, lp, [], torch.zeros(B, C, dtype=torch.float64))
    t = _fake_trainer(0.04, 1, None, tis=True)
    with pytest.raises(ValueError, match="sampling_per_token_logps"):
        gt.DNALLMGRPOTrainer.compute_loss(t, None, _inputs(old, ref, None, adv, cmask))


@pytest.mark.parametrize("tis", [None, False])
def test_flag_off_calls_the_plain_loss(monkeypatch, tis):
    """Flag off (or a trainer whose args predate the flag): grpo_loss_raw with its existing signature, rollout log-probs ignored."""
    from bioreason_b200 import ops, training
    from bioreason_b200.trainer import grpo_trainer as gt
    lp, old, ref, samp, adv, cmask = _case(0.04, 2)
    calls = []

    def fake_loss_raw(lp_, old_lp, ref_lp, adv_, mask_, beta_, lo, hi, want_grad=True):
        calls.append(lp_.shape[0])
        x = lp_.clone().requires_grad_(True)
        loss, kl, clip = og.grpo_loss(x, old_lp, ref_lp, adv_, mask_, beta_, lo, hi)
        loss.backward()
        return torch.stack([loss.detach(), kl.detach(), clip.detach()]), x.grad

    def no_is_loss(*a, **k):
        raise AssertionError("grpo_loss_is_raw called with the correction off")

    monkeypatch.setattr(training, "policy_forward", lambda model, ids, *a, **k: (lp[ids[:, 0].tolist()].clone(), None))
    monkeypatch.setattr(ops, "grpo_loss_raw", fake_loss_raw)
    monkeypatch.setattr(ops, "grpo_loss_is_raw", no_is_loss)
    t = _fake_trainer(0.04, 2, 3, tis=tis)
    loss = gt.DNALLMGRPOTrainer.compute_loss(t, None, _inputs(old, ref, samp, adv, cmask), backward=False)
    want, _, _ = og.grpo_loss(lp, old, ref, adv, cmask, 0.04, 0.2, 0.28)
    assert calls == [3, 3, 2] and abs(loss.item() - want.item()) < 1e-6
    assert not any(k.startswith("rollout_is/") for k in t._metrics)


@pytest.mark.parametrize("beta,mu", [(0.04, 1), (0.04, 2), (0.0, 2)])
def test_restatement_reduces_to_the_oracle_loss(beta, mu):
    """cap = inf and rollout log-probs equal to o: every weight is 1, so the TIS loss is the reference's loss and gradient."""
    lp, old, ref, _, adv, cmask = _case(beta, mu, seed=7)
    b = lp if old is None else old
    x = lp.clone().requires_grad_(True)
    loss, kl, clip, stats = grpo_loss_is(x, old, ref, b, adv, cmask, beta, 0.2, 0.28, math.inf)
    loss.backward()
    y = lp.clone().requires_grad_(True)
    want, kl_w, clip_w = og.grpo_loss(y, old, ref, adv, cmask, beta, 0.2, 0.28)
    want.backward()
    assert torch.equal(loss, want) and torch.equal(x.grad, y.grad)
    assert abs(clip.item() - clip_w.item()) < 1e-7                       # the oracle's clip ratio is a float32 ratio
    if beta > 0:
        assert torch.equal(kl, kl_w)
    assert stats.tolist() == [1.0, 0.0, 0.0, 0.0]


def test_config_validates_the_cap():
    from bioreason_b200.trainer import DNALLMGRPOConfig
    c = DNALLMGRPOConfig()
    assert c.rollout_is_correction is False and c.rollout_is_cap == 2.0
    assert DNALLMGRPOConfig(rollout_is_correction=True, rollout_is_cap=math.inf).rollout_is_cap == math.inf
    assert DNALLMGRPOConfig(rollout_is_cap=0.5).rollout_is_cap == 0.5
    for bad in (0.0, -1.0, float("nan"), -math.inf):
        with pytest.raises(ValueError, match="rollout_is_cap"):
            DNALLMGRPOConfig(rollout_is_correction=True, rollout_is_cap=bad)
