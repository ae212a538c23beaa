"""Kernel-level orchestration of the hot path: NT-v2 encoder forward, projector+scatter, Qwen3 decoder forward.

Python here only sequences C-ABI kernel launches on the current CUDA stream (no tensor math in torch on the
product path beyond index bookkeeping on tiny int tensors).  Reference call sites: dna_llm.py:103-179 (encode,
project, regroup), :208-244 (merge + LLM forward).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional

import torch

from . import ops
from .packing import LINEARS, DecoderLayerW, DecoderW, EncoderW, FusedLinear


# ---------------------------------------------------------------------------------------------
# attention-window bookkeeping (the reference's 0/1 masks are always one contiguous run per row)
# ---------------------------------------------------------------------------------------------
def mask_window(attention_mask: torch.Tensor):
    """[B, L] 0/1 mask -> (kv_start[B], kv_end[B]) int32 on the same device, no host sync."""
    m = attention_mask != 0
    L = m.shape[1]
    idx = torch.arange(L, device=m.device)
    start = torch.where(m, idx, L).amin(dim=1)
    end = torch.where(m, idx + 1, 0).amax(dim=1)
    start = torch.minimum(start, end)
    return start.to(torch.int32), end.to(torch.int32)


def forward_positions(B: int, L: int, device) -> torch.Tensor:
    """DNALLMModel.forward passes no position_ids -> HF uses arange over the PADDED row (SURVEY.md §3.1)."""
    return torch.arange(L, device=device, dtype=torch.int32).repeat(B)


def generate_positions(attention_mask: torch.Tensor) -> torch.Tensor:
    """HF generate(): position_ids = cumsum(mask) - 1, pads clamped to 1 (generation/utils.py:719-721)."""
    pos = attention_mask.long().cumsum(-1) - 1
    pos = pos.masked_fill(attention_mask == 0, 1)
    return pos.to(torch.int32).reshape(-1)


# ---------------------------------------------------------------------------------------------
# LoRA adapters in kernel layout (packed from the fp32 master parameters each optimizer step)
# ---------------------------------------------------------------------------------------------
@dataclass
class LoraLinearW:
    """The adapters of one fused linear, laid out as packing.FusedLinear describes."""
    a: torch.Tensor          # [n r, in]    rows = A of each target
    b: torch.Tensor          # [out, n r]   block diagonal
    a_T: torch.Tensor
    b_T: torch.Tensor


@dataclass
class LoraW:
    r: int
    scale: float             # alpha / r, applied in the A-GEMM epilogue
    layers: List[Dict[str, LoraLinearW]]      # per layer, keyed by FusedLinear.name


@dataclass
class LoraDropout:
    """Dropout of one pass through the adapters (the mask rule is next to br_lora_dropout in include/bioreason_b200.h)."""
    seed: int
    pass_id: int             # advanced once per dropout-applying pass; every row chunk of a pass shares it
    threshold: int           # T = round(p * 65536); p_eff = T / 65536
    row_offset: int = 0      # global token row (b * L + t of the whole pass) of this chunk's first row


@dataclass
class LayerSaved:
    """Activations one decoder layer keeps for the hand-written backward."""
    h_in: torch.Tensor = None
    rstd1: torch.Tensor = None
    xn1: torch.Tensor = None
    q: torch.Tensor = None            # post qk-norm + RoPE (views of one [M, (Hq+Hkv)D] buffer)
    k: torch.Tensor = None
    v: torch.Tensor = None            # view of the QKV GEMM output
    qkv_pre: torch.Tensor = None      # the QKV GEMM output itself: pre-norm q/k (for the qk-norm backward) | v
    attn: torch.Tensor = None
    lse: torch.Tensor = None
    h_mid: torch.Tensor = None
    rstd2: torch.Tensor = None
    xn2: torch.Tensor = None
    gu: torch.Tensor = None
    act: torch.Tensor = None
    t: Dict[str, torch.Tensor] = field(default_factory=dict)   # LoRA bottleneck x @ A.T of each fused linear


_ROPE_TABLES = {}


def _rope_table(n_pos: int, D: int, theta: float, device):
    """(cos, sin) pairs of positions [0, n_pos), bf16-rounded like HF's rotary tables; cached per (device, D, theta), grown on demand."""
    key = (str(device), D, float(theta))
    t = _ROPE_TABLES.get(key)
    if t is None or t.shape[0] < n_pos:
        t = _ROPE_TABLES[key] = ops.rope_table(max(n_pos, 4096), D, theta, device)
    return t


def _linear(f: FusedLinear, x, Lw: DecoderLayerW, li: int, lora: Optional[LoraW], dropout: Optional[LoraDropout], S, **kw):
    """y = x @ w.T of fused linear f in layer li (+ (scale * x @ A.T) @ B.T as a second K segment of the same wgmma accumulation).
    dropout: masks the adapter input per projection (ids f.proj0 + i): t = scale / (1 - p_eff) * (x * m_j) @ A_j.T; the base GEMM
    reads x.  S (LayerSaved or None) keeps t for the backward."""
    if lora is None:
        return ops.gemm(x, getattr(Lw, f.name), **kw)
    ad = lora.layers[li][f.name]
    if dropout is None:
        t = ops.gemm(x, ad.a, alpha=lora.scale)
    else:
        t = ops.lora_down_dropout(x, ad.a, lora.scale, ops.lora_dropout_desc(dropout, li, f.proj0, lora.r))
    if S is not None:
        S.t[f.name] = t
    return ops.gemm(x, getattr(Lw, f.name), a2=t, b2=ad.b, **kw)


def decoder_forward(W: DecoderW, h: torch.Tensor, B: int, L: int, positions: torch.Tensor, kv_start, kv_end, *,
                    lora: Optional[LoraW] = None, saved: Optional[List[LayerSaved]] = None,
                    kv_sink: Optional[Callable[[int, torch.Tensor], None]] = None, final_norm: bool = True,
                    dropout: Optional[LoraDropout] = None, layout=None) -> torch.Tensor:
    """Qwen3 decoder stack over dense rows [B, L] (HF qwen3/modeling_qwen3.py:294-336, 378-430).

    h: merged input embeddings [B*L, d] bf16 (not modified).  Returns the final-normed hidden states [B*L, d].
    dropout: LoRA dropout of this pass (only with `lora`); None runs the adapters undropped.
    layout: optional training.SharedPrefixPlan: h, positions and the result are in its shared-prefix token buffer ([layout.N, d]) and
    kv_start / kv_end are its per-group / per-row windows.  Only attention sees the layout (br_attn_fwd_shared); with `saved`, the
    layer's lse is the (prefix, suffix) pair of segment buffers.
    """
    cfg = W.cfg
    Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
    eps = cfg.rms_norm_eps
    theta = cfg.rope_parameters["rope_theta"] if hasattr(cfg, "rope_parameters") else cfg.rope_theta
    QKV, O, GU, DOWN = LINEARS
    q_rows, k_rows, v_rows = QKV.rows(cfg)
    assert saved is None or kv_sink is None, "the KV sink reads roped K|V from the fused buffer; the training path keeps that buffer pre-norm"
    rope = _rope_table(L, D, theta, h.device)                          # cos/sin of positions 0..L-1, built once per (L, theta)
    for li, Lw in enumerate(W.layers):
        S = LayerSaved() if saved is not None else None
        if S is not None:
            xn, rstd1 = ops.rmsnorm(h, Lw.ln1, eps, want_rstd=True)
            S.h_in, S.rstd1, S.xn1 = h, rstd1, xn
        else:
            xn = ops.rmsnorm(h, Lw.ln1, eps)
        qkv = _linear(QKV, xn, Lw, li, lora, dropout, S)
        if S is not None:
            # training: the roped q|k go to their own buffer, the GEMM output keeps the pre-norm q|k (qk-norm backward) and V -- no copy
            S.qkv_pre = qkv
            qk = torch.empty(h.shape[0], k_rows.stop, device=h.device, dtype=torch.bfloat16)
            ops.qk_rope_(qkv, Hq, Hkv, D, positions, theta, q_norm_w=Lw.q_norm, k_norm_w=Lw.k_norm, eps=eps, mode=0, out=qk, rope=rope)
            q, k, v = qk[:, q_rows], qk[:, k_rows], qkv[:, v_rows]
            S.q, S.k, S.v = q, k, v
        else:
            ops.qk_rope_(qkv, Hq, Hkv, D, positions, theta, q_norm_w=Lw.q_norm, k_norm_w=Lw.k_norm, eps=eps, mode=0, rope=rope)
            q, k, v = qkv[:, q_rows], qkv[:, k_rows], qkv[:, v_rows]
        if kv_sink is not None:
            kv_sink(li, qkv)
        if layout is not None:
            res = ops.attn_fwd_shared(q, k, v, layout.U, layout.G, layout.Lp, layout.Ls, Hq, Hkv, D, kv_start, kv_end, want_lse=S is not None)
            if S is not None:
                attn, S.lse = res
                S.attn = attn
            else:
                attn = res
        elif S is not None:
            attn, lse = ops.attn_fwd(q, k, v, B, L, Hq, Hkv, D, kv_start=kv_start, kv_end=kv_end, causal=True, want_lse=True)
            S.attn, S.lse = attn, lse
        else:
            attn = ops.attn_fwd(q, k, v, B, L, Hq, Hkv, D, kv_start=kv_start, kv_end=kv_end, causal=True)
        h2 = _linear(O, attn, Lw, li, lora, dropout, S, residual=h)
        if S is not None:
            xn2, rstd2 = ops.rmsnorm(h2, Lw.ln2, eps, want_rstd=True)
            S.h_mid, S.rstd2, S.xn2 = h2, rstd2, xn2
            gu = torch.empty(h.shape[0], Lw.w_gu.shape[0], device=h.device, dtype=torch.bfloat16)
        else:
            xn2 = ops.rmsnorm(h2, Lw.ln2, eps)
            gu = None
        act = _linear(GU, xn2, Lw, li, lora, dropout, S, act=1, aux_out=gu)
        if S is not None:
            S.gu, S.act = gu, act
        h = _linear(DOWN, act, Lw, li, lora, dropout, S, residual=h2)
        if S is not None:
            saved.append(S)
    if not final_norm:
        return h
    return ops.rmsnorm(h, W.final_norm, eps)


def encoder_forward(W: EncoderW, input_ids: torch.Tensor, attention_mask: torch.Tensor) -> torch.Tensor:
    """NT-v2 / ESM encoder, forward only (the reference wraps it in no_grad, dna_llm.py:121): last hidden state
    after the final LayerNorm (== hidden_states[-1], HF esm/modeling_esm.py:511-512).  Returns [n_seq*S, d] bf16."""
    cfg = W.cfg
    n_seq, S = input_ids.shape
    nh = cfg.num_attention_heads
    D = cfg.hidden_size // nh
    d = cfg.hidden_size
    eps = cfg.layer_norm_eps
    x = ops.embed_gather(input_ids, W.embed, keep=attention_mask)          # embeddings * attention_mask (esm:232-233)
    ks, ke = mask_window(attention_mask)
    pos = torch.arange(S, device=x.device, dtype=torch.int32).repeat(n_seq)
    for Lw in W.layers:
        xn = ops.layernorm(x, Lw.ln1_w, Lw.ln1_b, eps)
        qkv = ops.gemm(xn, Lw.w_qkv, bias=Lw.b_qkv)
        ops.qk_rope_(qkv, nh, nh, D, pos, 10000.0, q_scale=D ** -0.5, mode=1)
        a = ops.attn_fwd(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], n_seq, S, nh, nh, D, kv_start=ks, kv_end=ke, scale=1.0, causal=False)
        x = ops.gemm(a, Lw.w_o, bias=Lw.b_o, residual=x)
        xn = ops.layernorm(x, Lw.ln2_w, Lw.ln2_b, eps)
        act = ops.gemm(xn, Lw.w_gu, bias=Lw.b_gu, act=1)
        x = ops.gemm(act, Lw.w_down, bias=Lw.b_down, residual=x)
    return ops.layernorm(x, W.final_ln_w, W.final_ln_b, eps)


def dna_row_map(input_ids: torch.Tensor, dna_token_id: int, dna_mask: torch.Tensor, batch_idx_map: List[int]):
    """Destination row (in the flattened [B*L] embedding buffer) of every encoder output row, or -1 for DNA pads.

    Restates dna_llm.py:166-177 + :216-229 without the per-sequence host syncs: valid tokens of the sequences, taken
    in (batch item, sequence) order, fill the <|dna_pad|> slots in row-major order.  Returns (row_map int32
    [n_seq*S], n_features, n_slots) with the two counts still on the device.
    """
    n_seq, S = dna_mask.shape
    dev = input_ids.device
    order = sorted(range(n_seq), key=lambda i: batch_idx_map[i])           # stable: regroup by batch item
    order_t = torch.tensor(order, device=dev, dtype=torch.long)
    valid_len = dna_mask.sum(dim=1)                                        # [:valid_length] slicing (dna_llm.py:168-169)
    tok = torch.arange(S, device=dev)
    valid = tok[None, :] < valid_len[:, None]                              # [n_seq, S] (first valid_len tokens)
    valid_sorted = valid[order_t]
    rank_sorted = valid_sorted.reshape(-1).long().cumsum(0) - 1            # feature index of each valid token
    slot_mask = (input_ids == dna_token_id).reshape(-1)
    n_slots = slot_mask.sum()
    n_feat = valid.sum()
    # position of the r-th slot
    slot_rank = slot_mask.long().cumsum(0) - 1
    N = slot_mask.numel()
    pos_of_rank = torch.full((N + 1,), -1, device=dev, dtype=torch.long)
    pos_of_rank.scatter_(0, torch.where(slot_mask, slot_rank, torch.full_like(slot_rank, N)), torch.arange(N, device=dev))
    dest_sorted = torch.where(valid_sorted.reshape(-1), pos_of_rank[rank_sorted.clamp(min=0, max=N)], torch.full_like(rank_sorted, -1))
    dest = torch.empty(n_seq, S, device=dev, dtype=torch.long)
    dest[order_t] = dest_sorted.view(n_seq, S)
    return dest.reshape(-1).to(torch.int32), n_feat, n_slots
