"""float64 reference of the pooled score head (br_seqcls_score), with the kernel's rounding points, a per-element bound and one-bug
variants, plus HF's own pooling rule run on a stub trunk.  Test infrastructure: torch only, runs on CPU or GPU.

Contract, per row b (HF GenericForSequenceClassification on Qwen3, transformers 5.5 modeling_layers.py):
  t    = the rightmost column whose id != pad (over all L columns, the attention mask is not read); 0 when every column is pad;
         L - 1 when there is no pad id
  v_i  = x_i rstd, x = h[b, t], rstd = 1 / sqrt(sum x^2 / d + eps)
  xn_i = bf16(v_i),  y_i = bf16(w_i xn_i)                                            (Qwen3RMSNorm's two roundings)
  out  = bf16(sum_i y_i S_ji)                                                        (bf16 Linear output), stored as fp32

Error model (e = 2^-24).  The kernel sums the squares in fp32 along a chain of n1 = 8 ceil(d / 8 / 256) + 5 + 8 adds of positive
terms (per-thread chunks of 8, a 5-step warp sum, 8 warp partials), then divides by d, adds eps and takes rsqrtf (<= 2 ulp): rstd
carries a relative error <= (n1 / 2 + 8) e, and the fp32 product x_i rstd one more e.  So the fp32 value the kernel rounds to bf16 lies
within v_i (1 +- eta), eta = SAFETY (n1 / 2 + 9) e, and, bf16 rounding being monotone, xn_i within [bf16(v_i (1 - eta)),
bf16(v_i (1 + eta))].  w_i xn_i is exact in fp32, so y_i lies between the roundings of the two ends.  The score's fp32 FMA chain has
n2 = 8 ceil(d / 8 / 256) + 5 + 8 steps: |sum - sum_ref| <= Delta = sum_i |S_ji| |y_i - y_ref_i|max + SAFETY n2 e sum_i |y_i S_ji|.
The output lies in [bf16(s - Delta), bf16(s + Delta)]; the per-element bound is the larger distance of those ends from bf16(s).
Most elements therefore have a bound of 0: the kernel must give the reference's bits unless a rounding boundary is within reach.
"""
import math
import types

import torch

from attn_ref import SAFETY

E = 2.0 ** -24
NT = 256
VARIANTS = ("leftmost_pad", "index_from_mask", "no_norm_round", "no_out_round", "wrong_row")


def bf16r(x: torch.Tensor) -> torch.Tensor:
    """Round float64 to the nearest bf16 value (ties to even) in one step, as __float2bfloat16 does from an fp32 value."""
    x = x.double()
    m, ex = torch.frexp(x)
    s = torch.pow(2.0, (ex - 8).double())
    return torch.where(x == 0, x, torch.round(x / s) * s)


def pooled_index(input_ids: torch.Tensor, pad_id) -> torch.Tensor:
    """The rightmost non-pad column of each row (module doc), int64 [B]."""
    B, L = input_ids.shape
    if pad_id is None:
        return torch.full((B,), L - 1, dtype=torch.long)
    col = torch.arange(L)[None, :].expand(B, L)
    return torch.where(input_ids.cpu() != pad_id, col, -1).amax(1).clamp(min=0)


def hf_pooled_index(input_ids: torch.Tensor, pad_id) -> torch.Tensor:
    """HF's own GenericForSequenceClassification.forward on a stub trunk whose hidden state at column t is t, so the pooled logit is the
    pooled column."""
    from transformers.modeling_layers import GenericForSequenceClassification
    from transformers.modeling_outputs import BaseModelOutputWithPast

    class Stub:
        base_model_prefix = "model"
        config = types.SimpleNamespace(pad_token_id=pad_id, use_return_dict=True, return_dict=True)

        @staticmethod
        def model(input_ids, **kw):
            B, L = input_ids.shape
            return BaseModelOutputWithPast(last_hidden_state=torch.arange(L, dtype=torch.float64)[None, :, None].expand(B, L, 1))

        @staticmethod
        def score(h):
            return h

    out = GenericForSequenceClassification.forward(Stub(), input_ids=input_ids.cpu())
    return out.logits[:, 0].long()


def _chain(d):
    return 8 * math.ceil(d / 8 / NT) + 5 + 8


def seqcls_ref(h, input_ids, pad_id, norm_w, eps, score_w, *, attention_mask=None, variant=None):
    """float64 reference of br_seqcls_score with the module doc's bound.  h [B*L, d] bf16, input_ids [B, L], score_w [n, d].
    variant: one of VARIANTS (the returned index / out are the variant's, the bound the correct reference's); index_from_mask needs
    attention_mask.  Returns a dict: index [B], out [B, n] (float64 holding the bf16 value), bound [B, n]."""
    B, L = input_ids.shape
    d = h.shape[1]
    idx = pooled_index(input_ids, pad_id)
    if variant == "leftmost_pad":
        isp = input_ids.cpu() == pad_id
        first = torch.where(isp, torch.arange(L)[None, :].expand(B, L), L).amin(1)
        idx = (first - 1).clamp(min=0)
    elif variant == "index_from_mask":
        m = attention_mask.cpu() != 0
        idx = torch.where(m, torch.arange(L)[None, :].expand(B, L), -1).amax(1).clamp(min=0)
    rows = idx.clone()
    if variant == "wrong_row":
        rows = torch.where(idx > 0, idx - 1, (idx + 1).clamp(max=L - 1))
    x = h.detach().cpu().double().view(B, L, d)[torch.arange(B), rows]
    w = norm_w.detach().cpu().double()
    S = score_w.detach().cpu().double()
    rstd = 1.0 / torch.sqrt((x * x).sum(1, keepdim=True) / d + eps)
    v = x * rstd
    eta = SAFETY * (_chain(d) / 2 + 9) * E
    xn = bf16r(v) if variant != "no_norm_round" else v
    a, b = bf16r(v * (1 - eta)), bf16r(v * (1 + eta))
    y = bf16r(w * xn)
    ya, yb = bf16r(w * a), bf16r(w * b)
    dy = torch.maximum((ya - y).abs(), (yb - y).abs())
    s = y @ S.T
    delta = dy @ S.abs().T + SAFETY * _chain(d) * E * (y.abs() @ S.abs().T)
    ref = bf16r(s)
    bound = torch.maximum(bf16r(s + delta) - ref, ref - bf16r(s - delta))
    out = s if variant == "no_out_round" else ref
    return {"index": idx, "out": out, "bound": bound}


def cases(d, n_labels, B, L, pad_id, seed=0, families=("random",)):
    """(h bf16 [B*L, d], ids int64 [B, L], mask [B, L], norm_w bf16 [d], score_w bf16 [n, d]) of one shape.  Families of the id rows:
    random ids with pad ids sprinkled in the middle, right padding, left padding and all-pad rows, cycled over the rows.  The mask
    is the padding's (ones over the text), so in-text pad ids sit under mask 1 as an EOS = pad token does in a completion."""
    g = torch.Generator().manual_seed(seed)
    h = (torch.randn(B * L, d, generator=g) * (0.5 + 3 * torch.rand(B * L, 1, generator=g))).to(torch.bfloat16)
    norm_w = (1 + 0.3 * torch.randn(d, generator=g)).to(torch.bfloat16)
    score_w = (torch.randn(n_labels, d, generator=g) * d ** -0.5).to(torch.bfloat16)
    pad = 0 if pad_id is None else pad_id
    ids = torch.randint(1, 50, (B, L), generator=g)
    ids[ids == pad] = pad + 1
    mask = torch.ones(B, L, dtype=torch.long)
    for r in range(B):
        kind = r % 5
        n = int(torch.randint(1, L + 1, (1,), generator=g)) if L > 1 else 1
        if pad_id is None:
            continue
        if kind == 1:                                            # pad ids inside the text (mask 1), then right padding
            ids[r, torch.rand(L, generator=g) < 0.3] = pad
            ids[r, n:] = pad
            mask[r, n:] = 0
        elif kind == 2:                                          # right padding
            ids[r, n:] = pad
            mask[r, n:] = 0
        elif kind == 3:                                          # left padding
            ids[r, :L - n] = pad
            mask[r, :L - n] = 0
        elif kind == 4 and r % 10 == 4:                          # all pad
            ids[r] = pad
            mask[r] = 0
    return h, ids, mask, norm_w, score_w
