"""float64 reference of the per-token entropy that the fused lm-head pass writes (br_lmhead_logprob_entropy_fwd), with a per-element
error bound, one-bug variants, and a bit-exact restatement of torch.quantile for the entropy threshold (br_entropy_threshold).
Test infrastructure: torch / numpy only, runs on CPU or GPU.

Entropy.  z = scale h w^T (float64 from the exact bf16 inputs), p = softmax(z), lse = logsumexp(z),
  H = -sum_j p_j log p_j = lse - sum_j p_j z_j.
The kernel forms, per 128-column tile t with maximum m_t, s_t = sum e^(z - m_t) and u_t = sum e^(z - m_t) (z - m_t) from the same
exps, then with M = max m_t, r_t = e^(m_t - M): S = sum s_t r_t, U = sum r_t (u_t + (m_t - M) s_t), H = log S - U / S.

Error model (on gemm_ref.lmhead_ref's model; e = 2^-24, E(x) = 2^-21 + 2^-23 |x| the relative error of __expf, dz_j = |scale| w S_j +
e |z_j| the error of the fp32 logit, A = sum_j p_j (zmax - z_j) = -U / S >= 0, nt = ceil(V / 128)):
  logits     dH/dz_j = -p_j (z_j - lse + H), so an error dz_j in z_j moves H by at most p_j |z_j - lse + H| dz_j.
  exps       each weight e^(z_j - m_t) and r_t carries a relative error <= E(zmax - z_j).  A relative error eps in weight j moves H by
             p_j (1 - (z_j - lse + H)) eps (the weight enters S and U, the offset z_j - m_t does not move), so the exps add
             sum_j p_j (1 + |z_j - lse + H|) 2 E(zmax - z_j).
  sums       S and U are sums of terms of one sign (S of >= 0, U of <= 0): 32 adds in a tile, 2 shuffles, ceil(nt / 32) partials per
             lane in the combine, a 5-step warp sum, plus the roundings of z - m_t, of each product and of m_t - M: at most
             (45 + ceil(nt / 32)) e relative, i.e. that times 1 in log S and times A in U / S.
  division   U / S rounds once: e A.
  log, sub   logf (1 ulp of log S) and the final subtraction (1 ulp of H).
  b_H = SAFETY (sum_j p_j |z_j - lse + H| dz_j + sum_j p_j (1 + |z_j - lse + H|) 2 E(zmax - z_j)
                + (45 + ceil(nt / 32)) e (1 + A) + e A + ulp(log S) + ulp(H))
Both terms of the kernel's H are >= 0 (S >= 1, U <= 0), so H >= 0 exactly as well; the tests check that separately.

Threshold.  torch.quantile(x, q) (linear) sorts the n values, forms r = q * (n - 1) in fp32, takes the order statistics a, b at
floor(r) and ceil(r) and returns lerp(a, b, w), w = r - floor(r): fma(w, b - a, a) for |w| < 0.5, else fma(-(b - a), 1 - w, b)
(fp32, each a single rounding).  quantile_ref restates that on the valid entries, +inf when none is valid.
"""
import math

import numpy as np
import torch

from attn_ref import SAFETY
from gemm_ref import E32, TILE, _f64, acc_weight, exp_err, ulp32

ENTROPY_VARIANTS = ("no_tile_shift", "no_divide", "no_last_tile", "temperature_0.6", "top_k_only")


def _logits64(h, w, scale, vchunk=16384):
    h = _f64(h)
    V = w.shape[0]
    z = torch.empty(h.shape[0], V, dtype=torch.float64, device=h.device)
    S = torch.empty_like(z)
    for v0 in range(0, V, vchunk):
        wc = _f64(w[v0:v0 + vchunk]).to(h.device)
        z[:, v0:v0 + vchunk] = h @ wc.T
        S[:, v0:v0 + vchunk] = h.abs() @ wc.abs().T
    return z * scale, S


def _tile_entropy(z, *, shift=True, divide=True, tiles=None):
    """H from 128-column tile partials as the kernel combines them (float64); `tiles` limits the tiles used."""
    M, V = z.shape
    nt = math.ceil(V / TILE)
    zp = torch.nn.functional.pad(z, (0, nt * TILE - V), value=-math.inf).view(M, nt, TILE)
    if tiles is not None:
        zp = zp[:, :tiles]
    mt = zp.amax(2)
    d = zp - mt[..., None]
    e = torch.exp(d)
    s = e.sum(2)
    u = torch.where(e > 0, e * d, 0.0).sum(2)
    Mx = mt.amax(1, keepdim=True)
    r = torch.exp(mt - Mx)
    S = (s * r).sum(1)
    U = (r * (u + (mt - Mx) * s)).sum(1) if shift else (r * u).sum(1)
    return torch.log(S) - (U / S if divide else U)


def entropy_ref(h, w, scale=1.0, *, same_sign=False, variant=None):
    """float64 H [M] of softmax(scale h w^T) with the bound of the module doc; variant: one of ENTROPY_VARIANTS (its value is returned
    as "H", the bound is the correct reference's).  Returns a dict: H, b_H, lse."""
    M, K = h.shape
    V = w.shape[0]
    z, Sabs = _logits64(h, w, scale)
    dz = abs(scale) * acc_weight(K, same_sign) * Sabs + E32 * z.abs()
    del Sabs
    zmax = z.amax(1, keepdim=True)
    lse = torch.logsumexp(z, 1)
    p = torch.exp(z - lse[:, None])
    H = lse - (p * z).sum(1)
    c = (z - lse[:, None] + H[:, None]).abs()
    A = (p * (zmax - z)).sum(1)
    logS = torch.log(torch.exp(z - zmax).sum(1))
    nt = math.ceil(V / TILE)
    b = ((p * c * dz).sum(1) + (p * (1 + c) * 2 * exp_err(zmax - z)).sum(1) + (45 + math.ceil(nt / 32)) * E32 * (1 + A) + E32 * A
         + ulp32(logS) + ulp32(H))
    out = {"b_H": SAFETY * b, "lse": lse}
    if variant is None:
        out["H"] = H
    elif variant == "no_tile_shift":
        out["H"] = _tile_entropy(z, shift=False)
    elif variant == "no_divide":
        out["H"] = _tile_entropy(z, divide=False)
    elif variant == "no_last_tile":
        out["H"] = _tile_entropy(z, tiles=nt - 1)
    elif variant == "temperature_0.6":
        lp = torch.log_softmax(z / 0.6, 1)
        out["H"] = -(lp.exp() * lp).sum(1)
    elif variant == "top_k_only":
        lp = torch.log_softmax(z.topk(min(20, V), 1).values, 1)
        out["H"] = -(lp.exp() * lp).sum(1)
    else:
        raise ValueError(variant)
    return out


# ------------------------------------------------------------------------------------------------------------------- threshold
def _fma32(x, y, z):
    """fp32 fma(x, y, z), correctly rounded: the product of two fp32 values is exact in float64, the sum is formed with its exact
    error (two-sum) and rounded to odd, which then rounds to fp32 without double rounding."""
    x, y, z = float(x), float(y), float(z)
    p = x * y
    s = p + z
    bb = s - p
    err = (p - (s - bb)) + (z - bb)
    if err != 0 and (np.float64(s).view(np.int64) & 1) == 0:
        s = float(np.nextafter(s, math.inf if err > 0 else -math.inf))
    return np.float32(s)


def quantile_ref(x, mask, level):
    """torch.quantile(x[mask != 0].float(), level) restated in numpy fp32 (module doc); +inf with no valid entry."""
    x = np.asarray(x.detach().cpu() if torch.is_tensor(x) else x, dtype=np.float32).reshape(-1)
    m = np.asarray(mask.detach().cpu() if torch.is_tensor(mask) else mask).reshape(-1) != 0
    v = np.sort(x[m])
    n = v.size
    if n == 0:
        return np.float32(math.inf)
    if np.isnan(v).any():
        return np.float32(math.nan)
    q = np.float32(level)
    r = np.float32(q * np.float32(n - 1))
    lo, hi = int(np.floor(r)), int(np.ceil(r))
    w = np.float32(r - np.float32(lo))
    a, b = v[lo], v[hi]
    d = np.float32(b - a)
    return _fma32(w, d, a) if abs(w) < 0.5 else _fma32(-d, np.float32(1) - w, b)


def threshold_cases(seed=0):
    """(name, values fp32 [n], mask int32 [n]) of the threshold checks: n in {1, 2, 3, 4095, 4096, 4097, 2^20} (random, ~75 % valid, NaN /
    inf / huge garbage in the masked slots), all-equal values, heavy ties (8 distinct values), and an empty mask."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for n in (1, 2, 3, 4095, 4096, 4097, 1 << 20):
        x = torch.rand(n, generator=g) * 8
        m = (torch.rand(n, generator=g) < 0.75).to(torch.int32)
        m[0] = 1
        junk = torch.tensor([math.nan, math.inf, -math.inf, -1e30, 1e30])
        bad = torch.nonzero(m == 0)[:, 0]
        x[bad] = junk[torch.arange(bad.numel()) % junk.numel()]
        out.append((f"random_{n}", x, m))
    n = 5000
    out.append(("all_equal", torch.full((n,), 2.5), torch.ones(n, dtype=torch.int32)))
    ties = (torch.randint(0, 8, (n,), generator=g).float() * 0.75)
    out.append(("heavy_ties", ties, (torch.rand(n, generator=g) < 0.9).to(torch.int32)))
    out.append(("empty_mask", torch.full((n,), math.nan), torch.zeros(n, dtype=torch.int32)))
    return out


RHOS = (0.0, 0.2, 0.5, 0.8, 1 - 2.0 ** -20)            # top_entropy_quantile values; the quantile level is 1 - rho


# ------------------------------------------------------------------------------------------------------------------------ loss
def grpo_loss_ent_with_grad(lp, old, ref, rollout, adv, mask, ent, tau, beta, eps_low, eps_high, cap=2.0):
    """float64 restatement of br_grpo_loss_ent_fwd_bwd, TRL's formula: the clipped policy-gradient term (times the truncated IS weight
    min(exp(o - rollout), cap) when rollout is given) counts only where mask and ent >= tau; the beta k3-KL term and the per-row mean
    over mask are as in the plain loss.  Returns (loss, mean_kl or None, clip_ratio, ent_sum, dloss/dlp)."""
    f = lambda t: None if t is None else t.double()
    x = lp.double().clone().requires_grad_(True)
    m = mask.double()
    keep = ((ent.double() >= float(tau)) & (mask != 0)).double()
    o = x.detach() if old is None else f(old)
    c1 = torch.exp(x - o)
    c2 = torch.clamp(c1, 1 - eps_low, 1 + eps_high)
    l1, l2 = c1 * adv.double()[:, None], c2 * adv.double()[:, None]
    pt = -torch.min(l1, l2)
    if rollout is not None:
        pt = pt * torch.clamp(torch.exp(o - f(rollout)), max=cap)
    pt = pt * keep
    cnt = m.sum(1)
    safe = torch.where(cnt > 0, cnt, torch.ones_like(cnt))
    mean_kl = None
    if beta > 0:
        d = f(ref) - x
        kl = torch.exp(d) - d - 1
        pt = pt + beta * kl
        mean_kl = torch.where(cnt > 0, (kl * m).sum(1) / safe, torch.zeros_like(cnt)).mean().detach()
    loss = torch.where(cnt > 0, (pt * m).sum(1) / safe, torch.zeros_like(cnt)).mean()
    loss.backward()
    clip = ((l1 < l2).double() * m).sum() / m.sum().clamp(min=1)
    return loss.detach(), mean_kl, clip.detach(), (ent.double() * m).sum(), x.grad
