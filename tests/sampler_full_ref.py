"""float64 reference of the full-vocabulary sampler (sampler_full.cu, br_sample_next_full), with a per-draw error margin, seeded
families that reach each branch, one-bug variants and an emulation of the kernel's integer arithmetic.  Test infrastructure, CPU only.

Contract (include/bioreason_b200.h).  z' is the fp32 row after the processors (sampler_proc_ref.penalize; z itself without them), T, p
and min_p the fp32 values the C ABI receives, u the fp32 uniform of (step, row).  top_k = 0: every finite value is kept; top_k >= 1 is
clamped to V and every finite value >= the k-th is kept (ties included, no cap).  The kept tokens are ordered by descending value, then
ascending id; top-p keeps the shortest prefix of that order whose probability (at T) reaches p -- the same set as dropping from the end
while the cumulative probability is <= 1 - p, the first always kept, the higher ids of equal values dropped first.  Min-p then drops
e_j = exp((z'_j - z'_max) / T) < min_p (the maximum has e = 1 and stays).  The draw walks the kept tokens in ascending id and returns
the first whose running sum of e exceeds u * sum(kept e).  A row with no finite value draws pad.

Error model.  The kernel's weight is w_j = exp(fp64((z'_j - M) / T)) in fp64 (an fp32 exp's relative error, summed over 10^5 kept
tokens, would be as large as a typical token's weight on a nearly flat row) and its mass is the integer q_j = rint(w_j 2^40).  With
a_j = (z'_j - M) / T, the division's rounding and the fp64 exp's error (a few ulp) give
    |q_j 2^-40 - e_j| <= err_j = e_j 2^-52 (|a_j| + 4) + 2^-41
and everything after is exact integer arithmetic: the masses of the cuts and of the CDF are sums of q, need = ceil(p Q) and
target = floor(u K) are exact.  There is no sequential fp32 sum, so the margins are sums of per-token errors, dominated by the
fixed-point rounding (about 10^5 2^-41 ~ 5e-8 of the maximum's weight).  With A_j = sum_{i < j} err_i and B the kept mass's error sum:
  top-p   at the positions around the cut, |prefix(j) - p W| <= SAFETY (A_j + p B + 2^-40) is at risk (keep one token more or fewer)
  min-p   |e_j - min_p| <= SAFETY (err_j + 2^-24 min_p) at the last kept / first dropped position is at risk
  draw    |S_i - u K| <= SAFETY (sum_{i' <= i} err + u B + 2^-40) at either edge of the chosen interval is at risk
An at-risk draw may be the reference token or one of the tokens on the other side of the boundary at risk.
"""
import math

import numpy as np
import torch

from attn_ref import SAFETY

E32 = 2.0 ** -24
QUNIT = 2.0 ** -40
CHUNK = 4096

# variant -> the family on which it must be seen to differ from the reference
EXPOSED_BY = {"topk_off_as_1024": "flat", "cut_id_order": "randn3", "ties_low_id_dropped": "ties_spread", "cut_at_T1": "randn3",
              "last_chunk_ignored": "last_chunk_mass", "draw_value_order": "randn3", "no_renorm": "randn3"}
VARIANTS = tuple(EXPOSED_BY)
RANDOM_FAMILIES = ("randn1", "randn3", "randn10", "randn30")
FAMILIES = ("flat",) + RANDOM_FAMILIES + ("peaked", "ties_spread", "last_chunk_mass", "neg_inf_chunks", "zero_mass")


def f32(x):
    return float(np.float32(x))


def _err(e, a):
    """Bound on |q 2^-40 - e| of one token (module doc)."""
    return e * 2.0 ** -52 * (np.abs(a) + 4) + QUNIT / 2


# ------------------------------------------------------------------------------------------------------------------- families
def make_logits(family, R, V, seed):
    """Seeded fp32 logits [R, V] (CPU).  The branch each family is meant to reach:
      flat            randn * 0.05: top_p = 0.95 keeps most of the vocabulary
      randn{1,3,10,30}
      peaked          one token per row 24 above the rest: top-p keeps one token
      ties_spread     20 distinct top values, then 3000 exact ties of 0 spread over every chunk, the rest -3: the top-k and top-p cut
                      values are ties whose kept part spans several chunks
      last_chunk_mass the 64 best values in the last (partial) chunk, 12 above the rest
      neg_inf_chunks  every other chunk entirely -inf, and rows (r % 3 == 2) with only 1 .. 12 finite values (fewer than k)
      zero_mass       randn plus 8 tokens 40 above: the rest have e < 2^-41 at T <= 1 and round to zero fixed-point mass"""
    g = torch.Generator().manual_seed(seed)
    if family == "flat":
        return (torch.randn(R, V, generator=g) * 0.05).float()
    if family.startswith("randn"):
        return (torch.randn(R, V, generator=g) * float(family[5:])).float()
    z = torch.randn(R, V, generator=g) * 2
    if family == "peaked":
        j = torch.randint(0, V, (R,), generator=g)
        z[torch.arange(R), j] = z.max(1).values + 24.0
    elif family == "ties_spread":
        z = torch.full((R, V), -3.0)
        for r in range(R):
            j = torch.randperm(V, generator=g)[:min(V, 3020)]
            z[r, j[:20]] = 1.0 + 0.05 * torch.arange(min(20, len(j))).float()[:len(j[:20])]
            z[r, j[20:]] = 0.0
    elif family == "last_chunk_mass":
        lo = ((V - 1) // CHUNK) * CHUNK
        for r in range(R):
            j = lo + torch.randperm(V - lo, generator=g)[:64]
            z[r, j] += 12.0
    elif family == "neg_inf_chunks":
        for c in range(1, (V + CHUNK - 1) // CHUNK, 2):
            z[:, c * CHUNK:(c + 1) * CHUNK] = -math.inf
        for r in range(2, R, 3):
            n = 1 + r % 12
            row = torch.full((V,), -math.inf)
            j = torch.randperm(V, generator=g)[:n]
            row[j] = torch.randn(n, generator=g) * 3
            z[r] = row
    elif family == "zero_mass":
        z = torch.randn(R, V, generator=g)
        for r in range(R):
            z[r, torch.randperm(V, generator=g)[:8]] += 40.0
    else:
        raise ValueError(family)
    return z.float()


# ------------------------------------------------------------------------------------------------------------------- reference
class FullRow:
    """The kept set of one processed row and the draw for any number of uniforms."""

    def __init__(self, zp, T, top_k, top_p, min_p=0.0, *, variant=None):
        z = np.asarray(zp, dtype=np.float32).astype(np.float64)
        V = len(z)
        T, p, mp = f32(T), f32(top_p), f32(min_p)
        self.variant = variant
        ids = np.arange(V)
        fin = z > -math.inf
        if variant == "last_chunk_ignored" and V % CHUNK:
            fin &= ids < (V // CHUNK) * CHUNK
        self.empty = not fin.any()
        if self.empty:
            return
        k = 1024 if (variant == "topk_off_as_1024" and top_k == 0) else top_k
        kept = fin.copy()
        if k > 0 and k < fin.sum():
            kth = np.sort(z[fin])[::-1][k - 1]
            kept &= z >= kth
        kid = ids[kept]
        order = np.lexsort((-kid if variant == "ties_low_id_dropped" else kid, -z[kid]))
        sel = kid[order]
        zs = z[sel]
        a = (zs - zs[0]) / T
        e = np.exp(a)
        err = _err(e, a)
        c = len(sel)
        self.m_cut, self.alt_keep = math.inf, None
        keep = c
        if p < 1.0:
            ec = np.exp(zs - zs[0]) if variant == "cut_at_T1" else e
            if variant == "cut_id_order":
                o = np.argsort(sel)
                ecs, errs = ec[o], err[o]
            else:
                o, ecs, errs = None, ec, err
            W, B = ecs.sum(), errs.sum()
            pre = np.concatenate([[0.0], np.cumsum(ecs)])            # pre[j] = mass of the first j
            A = np.concatenate([[0.0], np.cumsum(errs)])
            need = p * W
            keep = max(1, int(np.searchsorted(pre[1:], need, side="left")) + 1)
            keep = min(keep, c)
            d = A + p * B + QUNIT
            cands = []
            if keep >= 2:                                              # keep - 1 tokens reach less than need
                cands.append((abs(need - pre[keep - 1]) / d[keep - 1], keep - 1))
            if keep < c:                                               # keep tokens reach need
                cands.append((abs(pre[keep] - need) / d[keep], keep + 1))
            if cands:
                self.m_cut, self.alt_keep = min(cands)
            if o is not None:                                          # the cut in id order: the first keep ids of the kept set
                sel_keep = np.sort(sel[o[:keep]])
                sel = np.concatenate([sel_keep, np.setdiff1d(sel, sel_keep)])
                zsort = z[sel]
                e = np.exp((zsort - zs[0]) / T)
                err = _err(e, (zsort - zs[0]) / T)
        self.m_minp = math.inf
        if mp > 0:
            drop = np.nonzero(e[1:keep] < mp)[0]
            cut = 1 + int(drop[0]) if len(drop) else keep
            dm = err + E32 * mp
            cands = []
            if cut < keep:
                cands.append((abs(e[cut] - mp) / dm[cut], cut + 1))
            if cut >= 2:
                cands.append((abs(e[cut - 1] - mp) / dm[cut - 1], cut - 1))
            if cands:
                r, alt = min(cands)
                self.m_minp = r
                if cut < keep or r < self.m_cut:
                    self.m_cut, self.alt_keep = r, alt
            keep = cut
        self.sel, self.e, self.err, self.keep, self.c = sel, e, err, keep, c
        self.W_all = e.sum()
        self.kept = np.sort(sel[:keep])

    def _draw(self, u, keep):
        u = np.asarray(u, dtype=np.float32).astype(np.float64)
        ids, e, err = self.sel[:keep], self.e[:keep], self.err[:keep]
        o = np.arange(keep) if self.variant == "draw_value_order" else np.argsort(ids)
        ids, e, err = ids[o], e[o], err[o]
        K, B = e.sum(), err.sum()
        S, dS = np.cumsum(e), np.cumsum(err)
        target = u * (self.W_all if self.variant == "no_renorm" else K)
        dt = u * B + QUNIT
        i = np.minimum(np.searchsorted(S, target, side="right"), keep - 1)
        lo_m = np.where(i > 0, target - np.where(i > 0, S[np.maximum(i - 1, 0)], 0.0), math.inf)
        lo_d = dt + np.where(i > 0, dS[np.maximum(i - 1, 0)], 0.0)
        hi_m = np.where(i < keep - 1, S[i] - target, math.inf)
        hi_d = dt + dS[i]
        with np.errstate(divide="ignore", invalid="ignore"):
            lo_r = np.where(lo_m == math.inf, math.inf, np.abs(lo_m) / lo_d)
            hi_r = np.where(hi_m == math.inf, math.inf, np.abs(hi_m) / hi_d)
        # a zero-mass token can not be drawn by the kernel: the neighbour across a boundary is the next token with mass
        nb_lo = np.where(i > 0, ids[np.maximum(i - 1, 0)], -1)
        nb_hi = np.where(i < keep - 1, ids[np.minimum(i + 1, keep - 1)], -1)
        return ids[i], lo_r, hi_r, nb_lo, nb_hi

    def draw(self, u, pad=0):
        u = np.atleast_1d(u)
        if self.empty:
            n = len(u)
            return {"token": np.full(n, pad), "at_risk": np.zeros(n, bool), "allowed": np.full((n, 4), pad)}
        tok, lo_r, hi_r, nb_lo, nb_hi = self._draw(u, self.keep)
        risk_lo, risk_hi = lo_r <= SAFETY, hi_r <= SAFETY
        risk_c = self.m_cut <= SAFETY
        alt = self._draw(u, self.alt_keep)[0] if risk_c and self.alt_keep is not None else np.full_like(tok, -1)
        allowed = np.stack([tok, np.where(risk_lo, nb_lo, -1), np.where(risk_hi, nb_hi, -1), alt], 1)
        return {"token": tok, "at_risk": risk_lo | risk_hi | (risk_c & (alt != tok)), "allowed": allowed}


def draw_full_ref(zp, T, top_k, top_p, u, min_p=0.0, *, variant=None, pad=0):
    row = FullRow(zp, T, top_k, top_p, min_p, variant=variant)
    out = row.draw(u, pad=pad)
    out["row"] = row
    return out


# ------------------------------------------------------------------------------------------------------------------- kernel emulation
def emulate_kernel(zp, T, top_k, top_p, u, min_p=0.0, signs=None, pad=0):
    """The kernel's arithmetic: fp64 weights exp((z' - M) / T) (each perturbed by signs_j 2^-52 (|a_j| + 4) relative, signs in
    [-1, 1]: the adversarial end of the error model), integer masses rint(w 2^40), exact integer cuts and target.  Vectorised over u;
    returns the tokens."""
    z = np.asarray(zp, dtype=np.float32)
    V = len(z)
    u = np.atleast_1d(np.asarray(u, dtype=np.float32))
    fin = z > -np.inf
    if not fin.any():
        return np.full(len(u), pad)
    M = z[fin].max()
    with np.errstate(invalid="ignore"):
        a = (z.astype(np.float64) - np.float64(M)) / np.float64(np.float32(T))
    w = np.exp(a)
    if signs is not None:
        w = w * (1 + np.where(fin, signs, 0) * 2.0 ** -52 * (np.abs(np.where(fin, a, 0)) + 4))
    w = np.where(fin, w, 0.0)
    q = np.rint(w * 2.0 ** 40).astype(np.int64).astype(object)
    ids = np.arange(V)
    kept = fin.copy()
    if 0 < top_k < fin.sum():
        kth = np.sort(z[fin])[::-1][top_k - 1]
        kept &= z >= kth
    kid = ids[kept]
    sel = kid[np.lexsort((kid, -z[kid].astype(np.float64)))]
    keep = len(sel)
    if np.float32(top_p) < 1:
        Q = int(sum(q[sel]))
        pf = np.float32(top_p)
        man, ex = math.frexp(float(pf))                               # exact: p = man 2^ex
        num, den = int(man * 2 ** 53), 2 ** (53 - ex)
        need = -((-num * Q) // den)                                   # ceil(p Q)
        acc = 0
        for j, t in enumerate(sel):
            acc += int(q[t])
            if acc >= need:
                keep = j + 1
                break
    if np.float32(min_p) > 0:
        for j in range(1, keep):
            if w[sel[j]] < float(np.float32(min_p)):
                keep = j
                break
    ks = np.sort(sel[:keep])
    S = np.cumsum([int(q[t]) for t in ks], dtype=object)
    K = int(S[-1])
    out = []
    for uu in u:
        man, ex = math.frexp(float(uu))
        target = (int(man * 2 ** 53) * K) // 2 ** (53 - ex)
        target = min(target, K - 1)
        i = next(i for i, s in enumerate(S) if s > target)
        out.append(int(ks[i]))
    return np.asarray(out)
