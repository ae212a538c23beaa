"""Reference of the processed sampler (sampler.cu PROC path: HF's RepetitionPenalty -> MinNewTokens processors, then temperature -> top-k
-> top-p -> MinP -> draw), built on sampler_ref.py, with seeded families and one-bug variants.  Test infrastructure, CPU only.

Contract (include/bioreason_b200.h, br_sample_proc).  z is the raw fp32 row, S the set of tokens the row has emitted (a set: a token
emitted twice is penalised once), theta the fp32 penalty, s the step (tokens generated so far), m = min_new_tokens.
  z'_j = z_j < 0 ? fp32(z_j * theta) : fp32(z_j / theta)   for j in S      (the same two fp32 operations HF's processor does)
  z'_eos = -inf                                            while s < m
Greedy takes the argmax of z' (smallest id among equal maxima).  Sampling runs sampler_ref's draw on z' with one more cut after top-p:
min-p drops every kept j with e_j = exp((z'_j - z'_max) / T) < min_p; the maximum always stays.

Error model.  The penalty and the EOS mask are exact: the kernel does the same fp32 operations, so z' feeds sampler_ref.Row unchanged
and the draw's margins are sampler_ref's.  The min-p cut compares the kernel's w_j (|w_j - e_j| <= e_j r_j + F, sampler_ref's notation)
with min_p (rounded to fp32 by the C ABI; the reference uses that fp32 value, so the comparison itself adds no error); the cut is at risk
when |e_j - min_p| <= SAFETY (e_j r_j + F + e min_p) at the last kept or the first dropped position.  An at-risk cut may keep one token
more or fewer.  The log-prob reads the raw row: logp = z_y - logsumexp(z), the quantity of the *_logp entry points.
"""
import math

import numpy as np

import sampler_ref as sr
from attn_ref import SAFETY

# variant -> the family on which it must be seen to differ from the reference
EXPOSED_BY = {"dup_twice": "history_dups", "penalty_after_T": "penalty_tie", "neg_divided": "negatives_in_set",
              "prompt_in_set": "prompt_overlap", "min_new_le": "eos_argmax", "minp_raw_max": "max_demoted", "minp_T1": "minp_boundary"}
VARIANTS = tuple(EXPOSED_BY)
FAMILIES = ("max_demoted", "negatives_in_set", "penalty_tie", "tie_overflow_chunk", "chunk_in_set", "eos_argmax", "minp_only_max",
            "minp_boundary", "history_dups", "prompt_overlap", "randn3")


def penalize(z, ids, theta, *, eos=-1, blocked=False, variant=None, T=1.0):
    """Processed fp32 row z' (numpy float32).  ids: the emitted tokens in order (duplicates allowed: the set counts each once)."""
    z = np.asarray(z, dtype=np.float32).copy()
    th = np.float32(theta)
    ids = np.asarray(ids, dtype=np.int64)
    if variant == "dup_twice":
        uniq, cnt = np.unique(ids, return_counts=True)
        for j, c in zip(uniq, cnt):
            for _ in range(c):
                z[j] = z[j] * th if z[j] < 0 else z[j] / th
    else:
        uniq = np.unique(ids)
        if len(uniq):
            v = z[uniq]
            if variant == "neg_divided":
                z[uniq] = v / th
            elif variant == "penalty_after_T":                         # penalised on z / T, then scaled back to the logit scale
                t = np.float32(T)
                vt = (v / t).astype(np.float32)
                vt = np.where(vt < 0, vt * th, vt / th).astype(np.float32)
                z[uniq] = (vt * t).astype(np.float32)
            else:
                z[uniq] = np.where(v < 0, v * th, v / th).astype(np.float32)
    if blocked and eos >= 0:
        z[eos] = -np.inf
    return z


def eos_blocked(step, m, variant=None):
    return step <= m if variant == "min_new_le" else step < m


class ProcRow(sr.Row):
    """sampler_ref.Row on the processed row, plus the min-p cut.  z_raw: only for minp_raw_max (min-p against the unpenalised max)."""

    def __init__(self, zp, T, top_k, top_p, min_p=0.0, *, variant=None, z_raw=None):
        super().__init__(zp, T, top_k, top_p, variant=variant if variant in sr.VARIANTS else None)
        self.m_minp = math.inf
        mp = sr.f32(min_p)
        if not mp > 0:
            return
        keep = self.keep
        if variant == "minp_T1":
            e = np.exp(self.zs - self.zs[0])
        elif variant == "minp_raw_max":
            zr = np.asarray(z_raw, dtype=np.float32).astype(np.float64)
            e = np.exp((self.zs - np.max(zr[zr > -math.inf])) / sr.f32(T))
        else:
            e = self.e
        drop = np.nonzero(e[1:keep] < mp)[0]
        cut = 1 + int(drop[0]) if len(drop) else keep
        # the margin of the cut: the last kept (e >= min_p) and the first dropped position
        d = self.err + sr.E32 * mp
        cands = []
        if cut < keep:
            cands.append((abs(self.e[cut] - mp) / d[cut], cut + 1))
        if cut >= 2:
            cands.append((abs(self.e[cut - 1] - mp) / d[cut - 1], cut - 1))
        if cands:
            r, alt = min(cands)
            self.m_minp = r
            # a binding min-p cut (cut < keep) leaves top-p's cut no say; otherwise the nearer of the two cuts decides the alternative
            if cut < keep or r < self.m_topp:
                self.m_topp, self.alt_keep = r, alt
        self.keep = cut
        self.kept = np.sort(self.sel[:cut])


def draw_proc_ref(z, ids, theta, step, m, eos, T, top_k, top_p, min_p, u, *, variant=None):
    """One raw row z, emitted ids, any number of uniforms u -> ProcRow(...).draw(u) plus 'row' and 'zp'."""
    zp = penalize(z, ids, theta, eos=eos, blocked=eos_blocked(step, m, variant), variant=variant, T=T)
    row = ProcRow(zp, T, top_k, top_p, min_p, variant=variant, z_raw=z)
    out = row.draw(np.atleast_1d(u))
    out.update(row=row, zp=zp)
    return out


def greedy_proc_ref(z, ids, theta, step, m, eos, *, variant=None):
    return sr.greedy_ref(penalize(z, ids, theta, eos=eos, blocked=eos_blocked(step, m, variant), variant=variant))


def logp_raw(z, y):
    z = np.asarray(z, dtype=np.float64)
    f = z[z > -math.inf]
    mx = f.max()
    return float(z[y] - (mx + math.log(np.exp(f - mx).sum())))


# ------------------------------------------------------------------------------------------------------------------- families
def make_case(family, V, seed, *, top_k=20, theta=1.3, T=1.0):
    """(z fp32 [V] numpy, emitted ids, eos, prompt ids) of one row.  The branch each family is meant to reach:
      max_demoted        the row's 3 largest logits (positive) are in the set and fall below the k-th after the penalty
      negatives_in_set   every top logit is negative; the set holds the best ones (theta > 1 pushes them down, theta < 1 up)
      penalty_tie        a penalised value lands exactly on the k-th unpenalised value (fp32 z / theta == y): the kept set has a tie,
                         which penalty_after_T's rounding breaks
      tie_overflow_chunk 10 distinct tops, then 100 values in one chunk that the penalty maps onto one tie of the k-th: more than 64
                         ties in one chunk (stage 2 selects on the row)
      chunk_in_set       every id of one 4096-logit chunk (or of the row when V < 4096) is in the set
      eos_argmax         EOS holds the largest logit by 20 (argmax under no processor)
      minp_only_max      one token 12 above the rest: min-p keeps only the maximum
      minp_boundary      top values at exp(-a) ratios around min_p = 0.1 (a spread over 2.0 .. 2.6 at T = 1)
      history_dups       emitted ids repeat (each of the 5 best emitted 3 times); the best stays the argmax only if penalised once
      prompt_overlap     'prompt' ids (not in the set) are the 5 best logits: prompt_in_set penalises them
      randn3             z ~ 3 N(0, 1), 30 random emitted ids"""
    g = np.random.default_rng(seed)
    z = (g.standard_normal(V) * 2).astype(np.float32)
    eos, prompt = int(g.integers(0, V)), np.zeros(0, dtype=np.int64)
    order = lambda: np.argsort(-z, kind="stable")
    th = np.float32(theta)
    if family == "max_demoted":
        top = order()[:3]
        z[top] = np.float32(z.max() + 4.0) + np.arange(3, dtype=np.float32)
        ids = np.concatenate([top, g.integers(0, V, 20)])
    elif family == "negatives_in_set":
        z = (-np.abs(z) - 1.0).astype(np.float32)
        ids = np.concatenate([order()[:10], g.integers(0, V, 10)])
    elif family == "penalty_tie":
        # y is the k-th value; x (in the set) penalises exactly onto y, so both are kept.  Penalised after temperature T, x rounds
        # below y and drops out of the top-k.
        t = np.float32(T)
        for _ in range(100000):
            y = np.float32(g.uniform(1.0, 4.0)); x = np.float32(y * th)
            if np.float32(x / th) == y and (t == 1 or np.float32(np.float32(np.float32(x / t) / th) * t) < y):   # (T = 1: no variant)
                break
        else:
            raise RuntimeError("no penalty_tie value")
        o = order()
        z = np.minimum(z, np.float32(0.5)).astype(np.float32)
        k = min(top_k, V - 1)
        z[o[:k - 1]] = y + np.float32(0.05) * np.arange(1, k, dtype=np.float32)   # weights near y's: draws land on x
        z[o[k - 1]] = y
        x_idx = o[-1]
        z[x_idx] = x
        ids = np.array([x_idx])
    elif family == "tie_overflow_chunk":
        z = np.full(V, -5.0, dtype=np.float32)
        c = int(g.integers(0, max(1, V // sr.CHUNK)))                 # a full chunk (the whole row when V < 4096)
        lo, hi = c * sr.CHUNK, min(V, (c + 1) * sr.CHUNK)
        j = lo + g.permutation(hi - lo)[:110]
        z[j[:10]] = 1.0 + 0.01 * np.arange(10, dtype=np.float32)
        for _ in range(100000):                                        # v / theta rounds back to exactly t
            t = np.float32(g.uniform(0.4, 0.6)); v = np.float32(t * th)
            if np.float32(v / th) == t:
                break
        z[j[10:]] = v
        ids = j[10:]
    elif family == "chunk_in_set":
        c = int(g.integers(0, max(1, V // sr.CHUNK)))
        lo, hi = c * sr.CHUNK, min(V, (c + 1) * sr.CHUNK)
        z[lo:hi] += 6.0
        ids = np.arange(lo, hi)
    elif family == "eos_argmax":
        z[eos] = z.max() + 20.0
        ids = g.integers(0, V, 10)
        ids = ids[ids != eos]
    elif family == "minp_only_max":
        z[int(g.integers(0, V))] = z.max() + 12.0
        ids = g.integers(0, V, 10)
    elif family == "minp_boundary":
        o = order()
        top = o[:12]
        z[top[0]] = 10.0
        z[top[1:]] = (10.0 - g.uniform(2.0, 2.6, 11)).astype(np.float32)
        ids = g.integers(0, V, 10)
        ids = ids[~np.isin(ids, top)]
    elif family == "history_dups":
        o = order()
        best = o[:5]
        z[best[0]] = np.float32(abs(z[o[5]]) * float(th) ** 1.5)          # above the rest after one penalty, below after three
        ids = np.concatenate([np.repeat(best, 3), g.integers(0, V, 10)])
        g.shuffle(ids)
    elif family == "prompt_overlap":
        prompt = order()[:5]
        ids = g.integers(0, V, 10)
        ids = ids[~np.isin(ids, prompt)]
    elif family == "randn3":
        z = (g.standard_normal(V) * 3).astype(np.float32)
        ids = g.integers(0, V, 30)
    else:
        raise ValueError(family)
    return z.astype(np.float32), np.asarray(ids, dtype=np.int64), eos, np.asarray(prompt, dtype=np.int64)


def bitmap(id_sets, V):
    """int32 [R, ceil(V / 32)] bitmap of each row's id set (numpy)."""
    W = (V + 31) // 32
    out = np.zeros((len(id_sets), W), dtype=np.uint32)
    for r, ids in enumerate(id_sets):
        for j in np.unique(np.asarray(ids, dtype=np.int64)):
            out[r, j >> 5] |= np.uint32(1) << np.uint32(j & 31)
    return out.view(np.int32)


def ids_of_bitmap(bm, V):
    """Sorted id list of each row of an int32 bitmap."""
    u = np.asarray(bm).view(np.uint32)
    bits = ((u[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(u.shape[0], -1)[:, :V]
    return [np.nonzero(b)[0] for b in bits]


# ------------------------------------------------------------------------------------------------------------------- generation loop
def manual_processed_generate(oracle, batch, *, max_new_tokens, do_sample=False, temperature=1.0, top_k=50, top_p=1.0, min_p=None,
                              repetition_penalty=1.0, min_new_tokens=0, uniforms=None, eos_token_id=None, pad_token_id=0,
                              return_margins=False, variant=None):
    """oracle/generate.py's loop with HF's processor classes in HF's order (RepetitionPenalty -> MinNewTokensLength, then when sampling
    Temperature -> TopK -> TopP -> MinP) and the draw from the supplied uniforms.  As with HF generate(inputs_embeds=...), the
    processors' input_ids hold only the generated tokens.  variant='prompt_in_set' puts the prompt's text ids in the set as well.
    margins: per step, greedy: the fp32 top-2 gap of the processed logits; sampled: the distance of the draw's target from the edges of
    the chosen token's CDF interval, as a fraction of the kept mass."""
    import torch
    from transformers.generation.logits_process import (MinNewTokensLengthLogitsProcessor, MinPLogitsWarper,
                                                        RepetitionPenaltyLogitsProcessor, TemperatureLogitsWarper, TopKLogitsWarper,
                                                        TopPLogitsWarper)
    with torch.no_grad():
        embeds = oracle._merged_embeds(batch["input_ids"], batch.get("dna_tokenized"), batch.get("batch_idx_map"))
        dev = embeds.device
        mask = batch["attention_mask"].clone().to(dev)
        B = embeds.shape[0]
        procs = []
        if repetition_penalty != 1.0:
            procs.append(RepetitionPenaltyLogitsProcessor(repetition_penalty))
        if min_new_tokens > 0 and eos_token_id is not None:
            procs.append(MinNewTokensLengthLogitsProcessor(0, min_new_tokens, eos_token_id))
        if do_sample:
            if temperature != 1.0:
                procs.append(TemperatureLogitsWarper(temperature))
            if top_k:
                procs.append(TopKLogitsWarper(top_k=top_k, min_tokens_to_keep=1))
            if top_p < 1.0:
                procs.append(TopPLogitsWarper(top_p=top_p, min_tokens_to_keep=1))
            if min_p is not None and min_p > 0:
                procs.append(MinPLogitsWarper(min_p=min_p))
        seen = batch["input_ids"].to(dev) if variant == "prompt_in_set" else torch.zeros(B, 0, dtype=torch.long, device=dev)
        unfinished = torch.ones(B, dtype=torch.long, device=dev)
        emb_table = oracle.text_model.get_input_embeddings()
        out, margins = [], []
        for step in range(max_new_tokens):
            pos = (mask.long().cumsum(-1) - 1).masked_fill(mask == 0, 1)
            logits = oracle.text_model(inputs_embeds=embeds, attention_mask=mask, position_ids=pos).logits[:, -1, :].float()
            scores = logits
            for p in procs:
                scores = p(seen, scores)
            if do_sample:
                probs = torch.softmax(scores, dim=-1)
                cdf = probs.cumsum(-1)
                u = uniforms[step].to(device=dev, dtype=cdf.dtype)[:, None] * cdf[:, -1:]
                nxt = (cdf > u).int().argmax(-1)
                # distance of the target from the chosen token's CDF interval edges (a fraction of the total mass)
                hi = cdf.gather(1, nxt[:, None])[:, 0]
                lo = torch.where(nxt > 0, cdf.gather(1, (nxt - 1).clamp(min=0)[:, None])[:, 0], torch.zeros_like(hi))
                margins.append(torch.minimum(hi - u[:, 0], u[:, 0] - lo) / cdf[:, -1])
            else:
                nxt = scores.argmax(-1)
                top2 = scores.topk(2, dim=-1).values
                margins.append(top2[:, 0] - top2[:, 1])
            if eos_token_id is not None:
                nxt = nxt * unfinished + pad_token_id * (1 - unfinished)
                unfinished = unfinished & (nxt != eos_token_id).long()
            out.append(nxt)
            seen = torch.cat([seen, nxt[:, None]], dim=1)
            embeds = torch.cat([embeds, emb_table(nxt)[:, None, :]], dim=1)
            mask = torch.cat([mask, torch.ones(B, 1, dtype=mask.dtype, device=dev)], dim=1)
            if eos_token_id is not None and unfinished.max() == 0:
                break
        ids = torch.stack(out, dim=1)
        return (ids, torch.stack(margins, dim=1)) if return_margins else ids
