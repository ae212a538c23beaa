"""Float64 restatement of the GRPO loss with truncated importance sampling (TIS) against the rollout's own log-probs.

The reference trainer computes the clipped-ratio loss on samples it assumes came from the policy it scores with
(grpo_trainer.py:786-812, restated in oracle/grpo.py).  When the rollout samples from another set of weights (merged decode weights,
FP8 weights), each token's policy-gradient term is weighted by

    w = min(exp(o - b), cap),   o = old log-prob (the policy's own log-prob, detached, when mu == 1),  b = rollout log-prob

and w carries no gradient; the beta * k3 KL term stays unweighted.  With cap = inf and b = o this is oracle.grpo.grpo_loss.
"""
from __future__ import annotations

import torch


def grpo_loss_is(lp, old, ref, rollout, adv, mask, beta=0.04, eps_low=0.2, eps_high=0.2, cap=2.0):
    """Returns (loss, mean_kl, clip_ratio, stats[4]); differentiable w.r.t. lp.  Rows with an empty mask add 0 to the row mean
    (the kernels' convention).  stats = masked token means of (w, [exp(o - b) > cap], o - b, exp(o - b) - 1 - (o - b))."""
    m = mask.to(lp.dtype)
    o = lp.detach() if old is None else old
    d = o - rollout
    r = torch.exp(d)
    w = torch.clamp(r, max=cap)
    coef_1 = torch.exp(lp - o)
    coef_2 = torch.clamp(coef_1, 1 - eps_low, 1 + eps_high)
    l1 = coef_1 * adv.unsqueeze(1)
    l2 = coef_2 * adv.unsqueeze(1)
    per_token = -torch.min(l1, l2) * w
    cnt = m.sum(1)
    safe = torch.where(cnt > 0, cnt, torch.ones_like(cnt))
    mean_kl = None
    if beta > 0:
        dk = ref - lp
        kl = torch.exp(dk) - dk - 1
        per_token = per_token + beta * kl
        mean_kl = torch.where(cnt > 0, (kl * m).sum(1) / safe, torch.zeros_like(cnt)).mean()
    loss = torch.where(cnt > 0, (per_token * m).sum(1) / safe, torch.zeros_like(cnt)).mean()
    tot = m.sum()
    clip_ratio = ((l1 < l2).to(lp.dtype) * m).sum() / tot
    stats = torch.stack([(w * m).sum(), ((r > cap).to(lp.dtype) * m).sum(), (d * m).sum(), ((r - 1 - d) * m).sum()]) / tot
    return loss, mean_kl, clip_ratio, stats.detach()


def grpo_loss_is_with_grad(lp, old, ref, rollout, adv, mask, beta, eps_low, eps_high, cap):
    """(loss, mean_kl, clip_ratio, stats, dloss/dlp), all float64."""
    f = lambda t: None if t is None else t.double()
    x = lp.double().clone().requires_grad_(True)
    loss, kl, clip, stats = grpo_loss_is(x, f(old), f(ref), f(rollout), adv.double(), mask, beta, eps_low, eps_high, cap)
    loss.backward()
    return loss.detach(), (kl.detach() if kl is not None else None), clip, stats, x.grad
