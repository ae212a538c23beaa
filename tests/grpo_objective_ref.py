"""Float64 restatement of the GRPO objectives of later TRL releases (DESIGN.md §3), as torch autograd of the formulas.

Notation: m = the completion mask (after mask_truncated_completions), |o_b| = sum_t m_bt, o = the old log-prob (lp detached when
mu == 1), A_b the row's advantage, w the truncated importance weight min(exp(o - rollout_lp), cap) (1 without TIS), k the entropy
keep-mask (1 without entropy selection).

    token level     s_bt = lp_bt - o_bt
    sequence level  s_b  = sum_t m_bt (lp_bt - o_bt) / max(|o_b|, 1)            (GSPO; every token of the row uses it)
    c1 = exp(s), c2 = clamp(c1, 1 - eps_low, 1 + eps_high), then c1 <- clamp(c1, max=delta) when delta is set
    l_bt = -min(c1 A_b, c2 A_b) w_bt k_bt + beta k3_bt

    grpo     sum_b (sum_t m l / max(|o_b|, 1)) / B
    bnpo     sum m l / max(sum m, 1)
    dr_grpo  sum m l / (B max_completion_length)
    dapo     sum m l / (N / world),  N = max(completion tokens of all ranks, 1)

torch.min splits the gradient evenly at a tie and torch.clamp passes it at the bound: the kernels follow both rules.  With the
defaults this is oracle.grpo.grpo_loss.  `VARIANTS` are one-bug versions that the tests require to be distinguishable.
"""
from __future__ import annotations

import torch

VARIANTS = ("seq_mean_unmasked", "seq_mean_over_C", "dr_grpo_trimmed_width", "dapo_without_world", "delta_on_c2",
            "batch_std_biased", "none_still_divides", "threshold_without_truncation")


def token_terms(lp, old, ref, adv, mask, beta=0.04, eps_low=0.2, eps_high=0.2, *, level="token", delta=None, rollout=None, cap=2.0,
                keep=None, variant=None):
    """The per-token loss l and what the metrics need (before aggregation)."""
    B, C = lp.shape
    m = mask.to(lp.dtype)
    o = lp.detach() if old is None else old
    cnt = m.sum(1)
    nrm = cnt.clamp(min=1)
    a = adv.to(lp.dtype)[:, None]
    if level == "sequence":
        if variant == "seq_mean_unmasked":
            s = (lp - o).sum(1) / nrm
        elif variant == "seq_mean_over_C":
            s = ((lp - o) * m).sum(1) / C
        else:
            s = ((lp - o) * m).sum(1) / nrm
        s = s[:, None].expand(B, C)
    else:
        s = lp - o
    c1 = torch.exp(s)
    c2 = torch.clamp(c1, 1 - eps_low, 1 + eps_high)
    if delta is not None:
        if variant == "delta_on_c2":
            c2 = torch.clamp(c2, max=delta)
        else:
            c1 = torch.clamp(c1, max=delta)
    l1, l2 = c1 * a, c2 * a
    per = -torch.min(l1, l2)
    w = torch.ones_like(m)
    is_stats = None
    tot = m.sum().clamp(min=1)
    if rollout is not None:
        d = o - rollout
        r = torch.exp(d)
        w = torch.clamp(r, max=cap)
        is_stats = (torch.stack([(w * m).sum(), ((r > cap).to(lp.dtype) * m).sum(), (d * m).sum(), ((r - 1 - d) * m).sum()]) / tot).detach()
    if keep is not None:
        w = w * keep.to(lp.dtype)
    per = per * w
    kl = None
    if beta > 0:
        dk = ref - lp
        kl = torch.exp(dk) - dk - 1
        per = per + beta * kl
    return dict(per=per, m=m, nrm=nrm, cnt=cnt, kl=kl, l1=l1, l2=l2, c1=c1, a=a, tot=tot, is_stats=is_stats)


def objective(lp, old, ref, adv, mask, beta=0.04, eps_low=0.2, eps_high=0.2, *, loss_type="grpo", level="token", delta=None,
              rollout=None, cap=2.0, keep=None, max_completion_length=None, num_items=None, world=1, variant=None):
    """Returns dict(loss, kl, clip, low, high, region, is_stats); loss differentiable w.r.t. lp.  kl is the mean over rows of the
    row-mean k3 (rows with |o_b| = 0 add 0), the clip metrics and is_stats are masked token means over the batch."""
    B, C = lp.shape
    T = token_terms(lp, old, ref, adv, mask, beta, eps_low, eps_high, level=level, delta=delta, rollout=rollout, cap=cap, keep=keep,
                    variant=variant)
    per, m, nrm, cnt, kl, l1, l2, c1, a, tot = (T[k] for k in ("per", "m", "nrm", "cnt", "kl", "l1", "l2", "c1", "a", "tot"))
    kl_mean = None if kl is None else torch.where(cnt > 0, (kl * m).sum(1) / nrm, torch.zeros_like(cnt)).mean().detach()
    if loss_type == "grpo":
        loss = ((per * m).sum(1) / nrm).sum() / B
    elif loss_type == "bnpo":
        loss = (per * m).sum() / m.sum().clamp(min=1)
    elif loss_type == "dr_grpo":
        width = C if variant == "dr_grpo_trimmed_width" else max_completion_length
        loss = (per * m).sum() / (B * width)
    elif loss_type == "dapo":
        n = max(float(num_items), 1.0)
        loss = (per * m).sum() / (n if variant == "dapo_without_world" else n / world)
    else:
        raise ValueError(loss_type)
    low = ((c1 < 1 - eps_low) & (a < 0)).to(lp.dtype)
    high = ((c1 > 1 + eps_high) & (a > 0)).to(lp.dtype)
    f = lambda x: ((x * m).sum() / tot).detach()
    return dict(loss=loss, kl=kl_mean, clip=f((l1 < l2).to(lp.dtype)), low=f(low), high=f(high), region=f(torch.clamp(low + high, max=1)),
                is_stats=T["is_stats"])


def objective_with_grad(lp, *args, **kw):
    """objective() in float64 plus d loss / d lp."""
    f = lambda t: None if t is None else t.double()
    args = [f(t) if isinstance(t, torch.Tensor) else t for t in args]
    kw = {k: f(v) if isinstance(v, torch.Tensor) and k in ("rollout",) else v for k, v in kw.items()}
    x = lp.double().clone().requires_grad_(True)
    out = objective(x, *args, **kw)
    out["loss"].backward()
    out["loss"] = out["loss"].detach()
    out["dlp"] = x.grad
    return out


def advantages(rewards_per_func, G, scale="group", variant=None):
    """TRL's scale_rewards, float64: returns (advantages, std_used per row, zero_std per row).  std_used is the group std in
    "group" and "none" modes (TRL logs it; "none" divides by nothing) and the std of all rows in "batch" mode; all unbiased."""
    r = rewards_per_func.double().sum(1)
    g = r.view(-1, G)
    mean = g.mean(1).repeat_interleave(G)
    if scale == "batch":
        sd = r.std(unbiased=variant != "batch_std_biased").expand_as(r)
    else:
        sd = g.std(1).repeat_interleave(G)
    adv = r - mean
    if scale != "none" or variant == "none_still_divides":
        adv = adv / (sd + 1e-4)
    return adv, sd, sd <= 1e-8


def truncated_mask(completion_ids, eos):
    """(mask, lengths): the EOS-inclusive completion mask with rows that hold no EOS zeroed, and the per-row counts before that."""
    is_eos = completion_ids == eos
    C = completion_ids.shape[1]
    first = torch.where(is_eos.any(1), is_eos.int().argmax(1), torch.full_like(is_eos[:, 0], C, dtype=torch.long))
    pre = (torch.arange(C)[None, :] <= first[:, None]).int()
    return pre * is_eos.any(1, keepdim=True).int(), pre.sum(1).int()


def entropy_keep(entropy, mask, rho, pre_mask=None, variant=None):
    """TRL's top_entropy_quantile keep-mask: entropy >= quantile(entropy over the valid tokens, 1 - rho).  The valid tokens are those
    of the loss mask (after truncation masking); the one-bug variant takes them from the mask before it."""
    valid = (pre_mask if variant == "threshold_without_truncation" else mask).bool()
    tau = torch.quantile(entropy[valid].float(), 1.0 - rho)
    return entropy >= tau
