"""float64 reference of the rollout's token draw (sampler.cu: temperature -> top-k -> top-p -> inverse CDF with a supplied uniform),
with a per-draw error margin, seeded logit families that reach each branch of the two-stage sampler, and one-bug variants.  Test
infrastructure: numpy / torch on the CPU; oracle/ is not involved.

Contract (sampler.cu's header, ops.sample_next, oracle/generate.py).  z is the fp32 logits row, T and p the fp32 values the C ABI
receives, u the fp32 uniform of (step, row).  top_k is clamped to V.  Top-k keeps every finite value >= the k-th (HF's tie rule); past
MAXC = 1024 such values the kernel keeps every value above the k-th plus the lowest-id ties (the one departure from HF, deterministic).
The kept tokens are ordered by descending value, then ascending id; top-p drops from the end of that order while the cumulative
probability (at T) is <= 1 - p and always keeps the first.  Among equal values the higher ids are dropped first: HF sorts with
torch.sort(stable=False), which leaves that order unspecified, so the reference adopts the kernel's.  The draw walks the kept tokens in
ascending id and returns the first whose running sum of e_j = exp((z_j - z_max) / T) exceeds u * sum(kept e_j).  Top-k is selected on
the exact fp32 logits; HF selects on z / T rounded to fp32, which can merge two neighbouring logits into a tie -- a known and accepted
difference from HF run in fp32 (the float64 reference agrees with the kernel).

Error model.  Stage 2's thread 0 (or the single-stage CTA's) does the arithmetic in fp32; e = 2^-24, E(x) = 2^-21 + 2^-23 |x|
(gemm_ref.exp_err, __expf), F = 2^-126 (ex2.approx.ftz flushes a subnormal result to 0).  j runs over the c top-k-kept tokens in the
order above, a_j = (z_j - z_0) / T <= 0 exactly, W = sum_j e_j.
  exp arg   da_j = 2e (|z_j| + |z_0|) / T + e |a_j|      inv_t = 1/T rounded (e), z inv_t and z_0 inv_t rounded (or one fused
                                                         rounding), the difference rounded
  weight    |w_j - e_j| <= e_j r_j + F,  r_j = da_j + E(a_j)      (first order in da_j; SAFETY covers the second)
  tot       dB = sum_j (e_j r_j + F) + (c - 1) e W        sequential fp32 sum of c positive terms
  top-p     d_topp(j) = A_j / W + P_j dB / W + (c - j) e P_j + e (1 - p)     P_j = sum_{i >= j} e_i / W (the cumulative probability the
            loop compares), A_j = sum_{i >= j} (e_i r_i + F); the divisions w_i / tot (e each), the c - j - 1 adds of cum, 1 - p in fp32
  ktot      dK = sum_kept (e_j r_j + F) + (keep - 1) e K  K = sum_kept e_j
  target    dt = u dK + e u K                             u ktot rounded
  acc       dS_i = sum_{i' <= i} (e r + F) + i e S_i      S_i: the exact running sum after the i-th kept id (ascending id)
A draw is at risk when m_cdf <= SAFETY (dt + dS) at the boundary S_{i-1} or S_i of the chosen interval (no boundary below the first
id, none above the last: the kernel returns the last id it visited), or when m_topp = |P_j - (1 - p)| <= SAFETY d_topp(j) at the
last dropped or the first kept position of the cut.  An at-risk draw may be the reference token or the token on the other side of
the boundary at risk (for the cut: the draw with one token more or fewer kept).
"""
import math

import numpy as np
import torch

from attn_ref import SAFETY
from gemm_ref import exp_err

E32 = 2.0 ** -24
FTZ = 2.0 ** -126
MAXC = 1024
CHUNK = 4096
CAND_CAP = 64

# variant -> the family on which it must be seen to differ from the reference
EXPOSED_BY = {"strict_topk": "tie_overflow_chunk", "topp_before_topk": "randn3", "topp_at_T1": "randn3",
              "topp_off_by_one": "randn3", "no_renorm": "randn3", "cdf_prob_order": "randn3", "uniforms_row_major": "randn3",
              "cap64_per_chunk": "tie_overflow_chunk", "first1024": "tie_overflow_1024"}
VARIANTS = tuple(EXPOSED_BY)
RANDOM_FAMILIES = ("randn1", "randn3", "randn10", "randn30")
FAMILIES = RANDOM_FAMILIES + ("peaked", "flat_top", "chunk_local", "fewer_finite_than_k", "tie_overflow_chunk", "tie_overflow_1024",
                              "uniform_grid")


def f32(x):
    return float(np.float32(x))


def _E(a):
    return exp_err(torch.from_numpy(np.asarray(a, dtype=np.float64))).numpy()


# ------------------------------------------------------------------------------------------------------------------- families
def make_logits(family, R, V, seed):
    """Seeded fp32 logits [R, V] (CPU).  The branch each family is meant to reach:
      randn{1,3,10}  stage 1 / stage 2 fast histograms (spread well inside 64 units)
      randn30        spread beyond the 64-unit histogram: the exact radix selects of both stages
      peaked         one token per row holds > 0.99 of the mass at every T <= 1.5: top-p keeps one token
      flat_top       30 near-equal top values (jitter 1e-3): the top-p cut falls inside the run
      chunk_local    the whole top 64 in one chunk (the tail chunk on even rows, chunk 0 on odd rows)
      fewer_finite_than_k  rows of 1 to 12 finite logits, the rest -inf (stage 1's all -inf chunks, the k-th value is -inf)
      tie_overflow_chunk   10 distinct values above 100 exact ties of the k-th, all inside one chunk, the rest -5: stage 1 cannot
                     emit every tie (CAND_CAP = 64) and must send stage 2 to the row
      tie_overflow_1024    19 distinct top values (one per chunk), then 1200 ties of the 20th spread evenly over >= 20 chunks (at
                     most 61 values >= the k-th per chunk), the rest below: more than MAXC values >= the k-th, no chunk overflows
      uniform_grid   one randn*3 row repeated on every row (the draws use the (i + 1/2) / N grid of uniforms)"""
    g = torch.Generator().manual_seed(seed)
    if family.startswith("randn"):
        return torch.randn(R, V, generator=g) * float(family[5:])
    z = torch.randn(R, V, generator=g) * 2
    if family == "peaked":
        j = torch.randint(0, V, (R,), generator=g)
        z[torch.arange(R), j] = z.max(1).values + 24.0
    elif family == "flat_top":
        for r in range(R):
            j = torch.randperm(V, generator=g)[:min(30, V)]
            z[r, j] = 8.0 + 1e-3 * torch.randn(len(j), generator=g)
    elif family == "chunk_local":
        n_chunks = (V + CHUNK - 1) // CHUNK
        for r in range(R):
            c = n_chunks - 1 if r % 2 == 0 else 0
            lo, hi = c * CHUNK, min(V, (c + 1) * CHUNK)
            j = lo + torch.randperm(hi - lo, generator=g)[:64]
            z[r, j] += 12.0
    elif family == "fewer_finite_than_k":
        z = torch.full((R, V), -math.inf)
        for r in range(R):
            n = 1 + r % 12
            j = torch.randperm(V, generator=g)[:n]
            z[r, j] = torch.randn(len(j), generator=g) * 3
    elif family == "tie_overflow_chunk":
        z = torch.full((R, V), -5.0)
        n_chunks = (V + CHUNK - 1) // CHUNK
        for r in range(R):
            c = int(torch.randint(0, n_chunks, (1,), generator=g))
            lo, hi = c * CHUNK, min(V, (c + 1) * CHUNK)
            j = lo + torch.randperm(hi - lo, generator=g)[:110]
            z[r, j[:10]] = 1.0 + 0.01 * torch.arange(10).float()
            z[r, j[10:]] = 0.0
    elif family == "tie_overflow_1024":
        assert V >= 20 * CHUNK, "tie_overflow_1024 spreads its ties over at least 20 chunks"
        n_chunks = V // CHUNK
        z = torch.randn(R, V, generator=g) - 10.0
        for r in range(R):
            ties = []
            for c in range(n_chunks):
                n_c = 1200 // n_chunks + (c < 1200 % n_chunks)
                ties.append(c * CHUNK + 1 + torch.randperm(CHUNK - 1, generator=g)[:n_c])
            z[r, torch.cat(ties)] = 0.0
            z[r, torch.arange(19) * CHUNK] = 1.0 + 0.1 * torch.arange(19).float()   # one distinct top value per chunk, low ids
    elif family == "uniform_grid":
        z = (torch.randn(1, V, generator=g) * 3).expand(R, V).contiguous()
    else:
        raise ValueError(family)
    return z.float()


def grid_uniforms(S, R):
    """u[s, r] = (i + 1/2) / N over the N = S R cells in a scrambled order (fp32): every CDF interval wider than 1/N is hit, and a
    transposed index reads a different value."""
    N = S * R
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(N))
    return ((perm.double() + 0.5) / N).float().view(S, R)


def distinct_uniforms(S, R, seed):
    """Random fp32 uniforms [S, R], all distinct."""
    u = torch.rand(S, R, generator=torch.Generator().manual_seed(seed))
    assert len(torch.unique(u)) == S * R
    return u


# ------------------------------------------------------------------------------------------------------------------- reference
def _kept_topk(z, k, maxc, variant, top_k):
    """Token ids kept by top-k (unordered)."""
    V = len(z)
    ids = np.arange(V)
    fin = z > -math.inf
    if variant == "cap64_per_chunk":                                   # stage 1 emitting at most 64 per chunk, ties by id
        cand = []
        for lo in range(0, V, CHUNK):
            zc = z[lo:lo + CHUNK]
            kc = min(top_k, len(zc))
            kth = np.sort(zc)[::-1][kc - 1]
            above = lo + np.nonzero(zc > kth)[0]
            ties = lo + np.nonzero(zc == kth)[0]
            cand.append(np.concatenate([above, ties[:CAND_CAP - len(above)]]))
        cand = np.concatenate(cand)
        cand = cand[fin[cand]]
        zc = z[cand]
        kth = np.sort(zc)[::-1][min(k, len(zc)) - 1]
        return cand[zc >= kth]
    kth = np.partition(z, V - k)[V - k]                               # the k-th largest (may be -inf)
    if variant == "strict_topk":
        order = np.lexsort((ids, -z))
        sel = order[:k]
        return sel[fin[sel]]
    above = ids[(z > kth) & fin]
    ties = ids[(z == kth) & fin]
    if variant == "first1024":                                         # whichever MAXC reach the counter first: high ids first here
        both = np.sort(np.concatenate([above, ties]))[::-1]
        return both[:MAXC]
    if maxc is not None and len(above) + len(ties) > maxc:
        ties = ties[:maxc - len(above)]
    return np.concatenate([above, ties])


def _topp_keep(p_desc, lim):
    """Kernel's cut on probabilities in (value desc, id asc) order: number kept, and the cumulative probabilities cum[j] (j >= 1)."""
    c = len(p_desc)
    cum = np.zeros(c)
    cum[1:] = np.cumsum(p_desc[:0:-1])[::-1]                           # cum[j] = sum_{i >= j} p_i
    keep = 1 + int(np.count_nonzero(cum[1:] > lim))
    return keep, cum


class Row:
    """The top-k / top-p decision for one logits row, and the draw for any number of uniforms (draw())."""

    def __init__(self, z, T, top_k, top_p, *, maxc=MAXC, variant=None):
        z = np.asarray(z, dtype=np.float32).astype(np.float64)
        T, p = f32(T), f32(top_p)
        V = len(z)
        k = min(top_k, V)
        self.variant = variant
        if variant == "topp_before_topk":
            kept0 = np.nonzero(z > -math.inf)[0]
        else:
            kept0 = _kept_topk(z, k, maxc, variant, top_k)
        order = np.lexsort((kept0, -z[kept0]))
        sel = kept0[order]                                             # value desc, id asc
        zs = z[sel]
        a = (zs - zs[0]) / T
        e = np.exp(a)
        c = len(sel)
        W = e.sum()
        da = 2 * E32 * (np.abs(zs) + abs(zs[0])) / T + E32 * np.abs(a)
        err = e * (da + _E(a)) + FTZ                                   # |w_j - e_j|
        dB = err.sum() + (c - 1) * E32 * W
        keep, self.m_topp, self.d_topp, alt_keep = c, math.inf, 0.0, None
        if p < 1.0:
            lim = 1.0 - p
            pt = np.exp(zs - zs[0]) / np.exp(zs - zs[0]).sum() if variant == "topp_at_T1" else e / W
            keep, cum = _topp_keep(pt, lim)
            A = np.zeros(c)
            A[1:] = np.cumsum(err[:0:-1])[::-1]
            j = np.arange(c)
            dtp = A / W + cum * dB / W + (c - j) * E32 * cum + E32 * lim
            cands = []
            if keep < c:                                               # the last dropped position: cum <= lim
                cands.append(((lim - cum[keep]) / dtp[keep], keep + 1))
            if keep >= 2:                                              # the position that stopped the loop: cum > lim
                cands.append(((cum[keep - 1] - lim) / dtp[keep - 1], keep - 1))
            if cands:
                r, alt = min(cands)
                self.m_topp = r                                        # margin / d_topp at the nearer side of the cut
                alt_keep = alt
            if variant == "topp_off_by_one":
                keep = min(c, keep + 1)
        if variant == "topp_before_topk":                              # then top-k (HF tie rule) on what top-p kept
            zk = zs[:keep]
            kth = zk[min(k, keep) - 1]
            keep = int(np.count_nonzero(zk >= kth))
        self.kept_topk = np.sort(sel)
        self.sel, self.zs, self.e, self.err = sel, zs, e, err
        self.c, self.keep, self.tot = c, keep, W
        self.alt_keep = alt_keep
        self.kept = np.sort(sel[:keep])

    def _draw(self, u, keep):
        u = np.asarray(u, dtype=np.float32).astype(np.float64)
        ids, e, err = self.sel[:keep], self.e[:keep], self.err[:keep]
        if self.variant == "cdf_prob_order":
            o = np.arange(keep)
        else:
            o = np.argsort(ids)
        ids, e, err = ids[o], e[o], err[o]
        K = e.sum()
        S = np.cumsum(e)
        dS = np.cumsum(err) + np.arange(keep) * E32 * S
        dK = err.sum() + (keep - 1) * E32 * K
        target = u * (self.e.sum() if self.variant == "no_renorm" else K)
        dt = u * dK + E32 * u * K
        i = np.minimum(np.searchsorted(S, target, side="right"), keep - 1)
        lo_m = np.where(i > 0, target - np.where(i > 0, S[i - 1], 0.0), math.inf)
        lo_d = dt + np.where(i > 0, dS[i - 1], 0.0)
        hi_m = np.where(i < keep - 1, S[i] - target, math.inf)
        hi_d = dt + dS[i]
        with np.errstate(divide="ignore", invalid="ignore"):
            lo_r = np.where(lo_m == math.inf, math.inf, lo_m / lo_d)
            hi_r = np.where(hi_m == math.inf, math.inf, hi_m / hi_d)
        nb_lo = np.where(i > 0, ids[np.maximum(i - 1, 0)], -1)
        nb_hi = np.where(i < keep - 1, ids[np.minimum(i + 1, keep - 1)], -1)
        return ids[i], lo_r, hi_r, nb_lo, nb_hi

    def draw(self, u):
        """Vectorised over the uniforms u.  Returns a dict: token, ratio (m_cdf / delta_cdf at the nearer boundary of the draw, inf
        when none applies; the cut's ratio is the row's m_topp), at_risk, allowed (int64 [n, 4]: the tokens an at-risk draw may take, -1 padded)."""
        tok, lo_r, hi_r, nb_lo, nb_hi = self._draw(u, self.keep)
        ratio = np.minimum(lo_r, hi_r)
        risk_lo, risk_hi = lo_r <= SAFETY, hi_r <= SAFETY
        risk_p = self.m_topp <= SAFETY
        alt = self._draw(u, self.alt_keep)[0] if risk_p and self.alt_keep is not None else np.full_like(tok, -1)
        allowed = np.stack([tok, np.where(risk_lo, nb_lo, -1), np.where(risk_hi, nb_hi, -1), alt], 1)
        # a cut at risk matters only where one token more or fewer kept changes the draw
        return {"token": tok, "ratio": ratio, "at_risk": risk_lo | risk_hi | (risk_p & (alt != tok)), "allowed": allowed}


def draw_ref(z, T, top_k, top_p, u, *, maxc=MAXC, variant=None):
    """One row z (fp32 logits), any number of uniforms u.  Returns Row.draw(u) plus the kept sets (top-k, after top-p), the exact
    weights e (in the kept order: value desc, id asc) and the top-p margin ratio."""
    row = Row(z, T, top_k, top_p, maxc=maxc, variant=variant)
    out = row.draw(np.atleast_1d(u))
    out.update(kept_topk=row.kept_topk, kept=row.kept, e=row.e, m_topp=row.m_topp, row=row)
    return out


def greedy_ref(z):
    """The largest logit; the smallest id among equal maxima."""
    z = np.asarray(z, dtype=np.float32)
    return int(np.lexsort((np.arange(len(z)), -z.astype(np.float64)))[0])


def uniform_index(step, row, S, R, variant=None):
    """Flat index of the uniform of (step, row) in the [S, R] buffer; uniforms_row_major reads it as [R, S]."""
    return row * S + step if variant == "uniforms_row_major" else step * R + row


# ------------------------------------------------------------------------------------------------------------------- fp32 emulation
def emulate_fp32(z, T, top_k, top_p, u, signs):
    """Thread 0's fp32 arithmetic (fused z inv_t - mx, sequential sums) on the kept set of draw_ref, with each __expf perturbed by
    signs_j * E(a_j) relative (signs in [-1, 1]) and flushed to 0 below 2^-126.  Vectorised over u; returns the tokens."""
    row = Row(z, T, top_k, top_p)
    zs = row.zs.astype(np.float32)
    inv_t = np.float32(1.0) / np.float32(T)
    mx = np.float32(zs[0] * inv_t)
    a = (zs.astype(np.float64) * np.float64(inv_t) - np.float64(mx)).astype(np.float32)   # one rounding (fma)
    w = (np.exp(a.astype(np.float64)) * (1 + signs[:len(a)] * _E(a))).astype(np.float32)
    w = np.where(w < np.float32(FTZ), np.float32(0), w)
    tot = np.add.accumulate(w, dtype=np.float32)[-1]
    c, keep = len(w), len(w)
    if np.float32(top_p) < 1:
        lim = np.float32(1) - np.float32(top_p)
        cum = np.float32(0)
        for j in range(c - 1, 0, -1):
            cum = np.float32(cum + np.float32(w[j] / tot))
            if cum <= lim:
                keep = j
            else:
                break
    ktot = np.add.accumulate(w[:keep], dtype=np.float32)[-1]
    ids = row.sel[:keep]
    o = np.argsort(ids)
    acc = np.add.accumulate(w[:keep][o], dtype=np.float32)
    target = (np.asarray(u, dtype=np.float32) * ktot).astype(np.float32)
    i = np.minimum(np.searchsorted(acc, target, side="right"), keep - 1)
    return ids[o][i]
