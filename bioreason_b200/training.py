"""Policy forward with saved activations + the hand-written backward through the LoRA-adapted Qwen3 decoder,
the fused lm_head log-prob, and the DNA projector (SURVEY.md §8a A7-A9, §2.3 K6/K12).

`policy_logps` is the differentiable equivalent of `_get_per_token_logps(...)[:, P-1:]` (grpo_trainer.py:510-520, :779):
gradients flow to the LoRA A/B masters and to `dna_projection` only -- the base weights are frozen and the encoder
is under no_grad in the reference (dna_llm.py:121).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import torch

from . import engine, ops
from .engine import LayerSaved
from .packing import LINEARS


class PolicyCtx:
    pass


def activation_bytes_per_token(model) -> int:
    """Bytes `policy_forward(save=True)` keeps per token for the backward: per decoder layer the block input and its RMSNorm, the QKV
    GEMM output, the roped q|k, the attention output and log-sum-exp, the mid-block residual and its RMSNorm, the gate|up
    pre-activations and the SwiGLU output (bf16 unless noted), plus the LoRA intermediates."""
    cfg = model._dec.cfg
    d, F = cfg.hidden_size, cfg.intermediate_size
    Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
    r = model._lora.r if getattr(model, "_lora", None) is not None else 0
    bf16 = 2 * (4 * d + (Hq + 2 * Hkv) * D + (Hq + Hkv) * D + Hq * D + 2 * F + F + 4 * r)
    fp32 = 4 * (2 + Hq)                                                    # two rstd values, one lse per query head
    return cfg.num_hidden_layers * (bf16 + fp32) + 2 * d                   # + the final hidden state


SHARED_TILE = 64          # tile height of the attention kernels: the shared prefix is a whole number of tiles


@dataclass
class SharedPrefixPlan:
    """Shared-prefix token layout of U groups x G rows [prompt P | completion], L positions each (see plan_shared_prefix)."""
    U: int
    G: int
    P: int
    L: int
    Lp: int                      # shared prefix length: positions 0 .. Lp-1 of a group are computed once
    Ls: int                      # L - Lp positions per row suffix
    N: int                       # buffer rows: U * Lp + U * G * Ls
    src: torch.Tensor            # int32 [N]: dense row (r * L + t) each buffer row holds (the group's first row for prefix rows)
    owner: torch.Tensor          # int32 [U*G*L]: buffer row of every dense row; -1 for the prefix positions of rows g > 0 of a group
    positions: torch.Tensor      # int32 [N]: arange over the padded row
    kv_start: torch.Tensor       # int32 [U]: attention window start of each group
    kv_end: torch.Tensor         # int32 [U*G]: attention window end of each row
    scored: torch.Tensor         # int32 [U*G*(L-P)]: buffer rows of positions P-1 .. L-2, row-major (the [B, L-P] log-prob order)

    def owner_of(self, dense_rows: torch.Tensor) -> torch.Tensor:
        """Buffer row owning each dense row index (-1 stays -1; prefix positions of rows g > 0 map to -1, so every (DNA feature,
        destination) pair of the shared layout is counted once)."""
        return torch.where(dense_rows >= 0, self.owner[dense_rows.clamp(min=0).long()], torch.full_like(dense_rows, -1)).to(torch.int32)


def plan_shared_prefix(G: int, P: int, L: int, kv_start: torch.Tensor, kv_end: torch.Tensor) -> Optional[SharedPrefixPlan]:
    """Shared-prefix layout of a batch of U = R / G groups whose G consecutive rows repeat one left-padded prompt of P columns,
    followed by L - P completion positions (host side, pure; index bookkeeping only, on kv_end's device, no host sync).

    The prefix is the prompt's full 64-position tiles minus one: Lp = 64 * floor((P - 1) / 64), so position P - 1 and every scored
    position (P - 1 .. L - 2) lie in a row's own suffix; like the rollout's page plan, full tiles are shared and the tail is private.
    Buffer rows: group u's positions 0 .. Lp-1 at u * Lp + t, row r = u * G + g's positions Lp + t at U * Lp + r * Ls + t.
    kv_start / kv_end are the dense rows' windows (engine.mask_window); the rows of a group share kv_start, and every window ends past
    the prefix (a completion follows the prompt).  Returns None (no sharing: the dense path) when G = 1 or Lp = 0."""
    R = int(kv_end.numel())
    if G <= 1 or R % G != 0 or P > L or P < 1:
        return None
    Lp = SHARED_TILE * ((P - 1) // SHARED_TILE)
    if Lp <= 0:
        return None
    U, Ls = R // G, L - Lp
    N = U * Lp + R * Ls
    dev = kv_end.device
    i64 = dict(device=dev, dtype=torch.long)
    t_p, t_s = torch.arange(Lp, **i64), torch.arange(Ls, **i64)
    u, r = torch.arange(U, **i64), torch.arange(R, **i64)
    src = torch.cat([((u * G * L)[:, None] + t_p[None, :]).reshape(-1), ((r * L + Lp)[:, None] + t_s[None, :]).reshape(-1)])
    owner = torch.full((R, L), -1, **i64)
    owner[::G, :Lp] = (u * Lp)[:, None] + t_p[None, :]
    owner[:, Lp:] = (U * Lp + r * Ls)[:, None] + t_s[None, :]
    positions = torch.cat([t_p.repeat(U), (Lp + t_s).repeat(R)])
    n = L - P
    scored = ((U * Lp + r * Ls + (P - 1 - Lp))[:, None] + torch.arange(n, **i64)[None, :]).reshape(-1)
    i32 = lambda x: x.to(torch.int32).contiguous()
    return SharedPrefixPlan(U=U, G=G, P=P, L=L, Lp=Lp, Ls=Ls, N=N, src=i32(src), owner=i32(owner.reshape(-1)), positions=i32(positions),
                            kv_start=i32(kv_start[::G]), kv_end=i32(kv_end), scored=i32(scored))


def policy_forward(model, input_ids, attention_mask, dna_tokenized, batch_idx_map, keep_last: int, *, save: bool = True,
                   lora="policy", targets: Optional[torch.Tensor] = None, dropout: bool = False, dropout_pass: Optional[int] = None,
                   row_offset: int = 0, group_size: Optional[int] = None, want_entropy: bool = False):
    """Returns (logps [B, keep_last] fp32, ctx), or with want_entropy (logps, ctx, entropies [B, keep_last] fp32): the entropy of the
    full-vocabulary softmax at every scored position (T = 1), from the same lm-head pass; the log-probs are the same bits.  lora: "policy" (adapters on), None (base weights = reference policy).
    targets: optional [B, keep_last] class ids scored at the last keep_last positions before the end (default: the realised next
    tokens input_ids[:, L-keep_last:]); entries < 0 are ignored (log-prob 0, no gradient) -- the SFT label mask.
    dropout: apply the LoRA dropout set by `model.set_lora_dropout` (no-op while it is off or with lora=None).  Row chunks of one pass
    share `dropout_pass` (from `model.new_lora_dropout_pass()`; None draws a new pass) and give `row_offset` = the batch row of their
    first row, so the masks do not depend on the chunking.  policy_backward regenerates the same masks from ctx.
    group_size: G > 1 declares that every G consecutive rows repeat one prompt, the first L - keep_last columns (left-padded, as the GRPO
    trainer builds them).  The decoder then runs on the shared-prefix layout (plan_shared_prefix): each group's full prompt tiles are
    computed once.  The log-probs are the same, in the same [B, keep_last] order.  Not combinable with an active LoRA dropout (its masks
    differ between the G copies of a prompt): ValueError."""
    W = model._dec
    dev = W.embed.device
    input_ids = input_ids.to(dev)
    attention_mask = attention_mask.to(dev)
    B, L = input_ids.shape
    use_lora = model._lora.w if (lora == "policy" and model._lora is not None) else None
    if lora is None and getattr(model, "_proj_ref", None) is not None:
        # the reference's ref_model is a deep copy taken at init (grpo_trainer.py:314-316): initial projector too
        pw, pb = model._proj_w16, model._proj_b16
        model._proj_w16, model._proj_b16 = model._proj_ref
        try:
            emb, aux = model.merged_embeddings(input_ids, dna_tokenized, batch_idx_map, return_proj_inputs=True)
        finally:
            model._proj_w16, model._proj_b16 = pw, pb
    else:
        emb, aux = model.merged_embeddings(input_ids, dna_tokenized, batch_idx_map, return_proj_inputs=True)
    ks, ke = engine.mask_window(attention_mask)
    saved: Optional[List[LayerSaved]] = [] if save else None
    drop = None
    if dropout and use_lora is not None and model._lora.dropout is not None:
        if group_size is not None and group_size > 1:
            raise ValueError("group_size > 1 (shared prompt prefix) cannot be combined with LoRA dropout: its masks are drawn per token row, "
                             "so the G copies of a prompt are not identical")
        pid = model._lora.new_dropout_pass() if dropout_pass is None else dropout_pass
        drop = model._lora.dropout_for(pid, row_offset * L)
    plan = plan_shared_prefix(group_size, L - keep_last, L, ks, ke) if group_size is not None and group_size > 1 else None
    if plan is None:
        pos = engine.forward_positions(B, L, dev)
        h = engine.decoder_forward(W, emb, B, L, pos, ks, ke, lora=use_lora, saved=saved, final_norm=False, dropout=drop)
    else:
        pos = plan.positions
        x = ops.gather_rows(emb, plan.src)                                 # the dense embeddings (DNA features included), prefix once
        del emb
        h = engine.decoder_forward(W, x, B, L, pos, plan.kv_start, plan.kv_end, lora=use_lora, saved=saved, final_norm=False, layout=plan)
    eps = W.cfg.rms_norm_eps
    if save:
        hn, rstd_f = ops.rmsnorm(h, W.final_norm, eps, want_rstd=True)
    else:
        hn, rstd_f = ops.rmsnorm(h, W.final_norm, eps), None
    n = keep_last
    if plan is None:
        cols = torch.arange(L - 1 - n, L - 1, device=dev)
        rows = (torch.arange(B, device=dev)[:, None] * L + cols[None, :]).reshape(-1).to(torch.int32)
    else:
        rows = plan.scored
    h_sel = ops.gather_rows(hn, rows)
    tgt = (input_ids[:, L - n:] if targets is None else targets.to(dev)).reshape(-1).to(torch.int32)
    if want_entropy:
        logp, lse, ent = ops.lmhead_logprob(h_sel, W.lm_head, tgt, want_entropy=True)
    else:
        logp, lse = ops.lmhead_logprob(h_sel, W.lm_head, tgt)
    ctx = None
    if save:
        ctx = PolicyCtx()
        ctx.B, ctx.L, ctx.n = B, L, n
        ctx.saved, ctx.h_final, ctx.rstd_f = saved, h, rstd_f
        ctx.rows, ctx.h_sel, ctx.tgt, ctx.lse = rows, h_sel, tgt, lse
        ctx.pos, ctx.ks, ctx.ke, ctx.aux = pos, ks, ke, aux
        ctx.use_lora = use_lora is not None
        ctx.drop = drop
        ctx.layout = plan
    if want_entropy:
        return logp.view(B, n), ctx, ent.view(B, n)
    return logp.view(B, n), ctx


@torch.no_grad()
def policy_backward(model, ctx: PolicyCtx, dlogp: torch.Tensor, on_layer_done=None):
    """Accumulates d(sum dlogp * logp) into the LoRA flat gradient buffer and the projector's .grad buffers.
    on_layer_done(layer_index): called right after the kernels producing that layer's adapter gradients were enqueued (the
    trainer hangs the overlapped gradient all-reduce of that layer's slice on it)."""
    W = model._dec
    W.build_transposes()
    cfg = W.cfg
    Hq, Hkv, D, d = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim, cfg.hidden_size
    theta = cfg.rope_parameters["rope_theta"] if hasattr(cfg, "rope_parameters") else cfg.rope_theta
    eps = cfg.rms_norm_eps
    B, L = ctx.B, ctx.L
    layout = getattr(ctx, "layout", None)
    M = B * L if layout is None else layout.N
    dev = W.embed.device
    lora = model._lora if ctx.use_lora else None
    r = lora.r if lora else 0
    s = lora.scale if lora else 1.0
    QKV, O, GU, DOWN = LINEARS

    # ---- lm_head: dlogits tiles recomputed from (h_sel, W) and the saved LSE, then dH = dlogits @ W
    g = dlogp.reshape(-1).float().contiguous()
    dlogits = ops.lmhead_dlogits(ctx.h_sel, W.lm_head, ctx.tgt, ctx.lse, g)
    dh_sel = ops.gemm(dlogits, W.lm_head_T)
    del dlogits
    dhn = torch.zeros(M, d, device=dev, dtype=torch.bfloat16)
    ops.scatter_rows_(dhn, dh_sel, ctx.rows)
    dh = ops.rmsnorm_bwd(ctx.h_final, W.final_norm, ctx.rstd_f, dhn)
    del dhn

    drop = getattr(ctx, "drop", None)

    def dd(li, j):
        """mask descriptor of projection j (packing.TARGETS index) in layer li, or None without dropout"""
        return ops.lora_dropout_desc(drop, li, j, r) if drop is not None else None

    def linear_bwd(f, li, dy, x, S):
        """dx = dy @ W of fused linear f (+ the LoRA path), then its adapter gradients.  With dropout the u @ A segment is masked per
        projection: dx = dy @ W + sum_i m_i * inv_keep * (u_i @ A_i)."""
        w_T = W.layers[li].w_T[f.name]
        if lora is None:
            return ops.gemm(dy, w_T)
        ad = lora.w.layers[li][f.name]
        u = ops.gemm(dy, ad.b_T, alpha=s)                                 # [M, n r] = s * dy @ B
        dx = ops.gemm(dy, w_T, a2=u, b2=ad.a_T, dropout=dd(li, f.proj0))
        # dB = dy^T t: one product over all of the linear's rows; each target keeps its rows and its own r columns (cross blocks are
        # discarded).  Blocked rows (gate/up) take mode 2.
        ops.lora_grad_tn(dy, S.t[f.name], [(lora.grad_view(li, t, "B"), rows.start, rows.stop, i * r, r)
                                           for i, (t, rows) in enumerate(zip(f.targets, f.rows(cfg)))], mode=2 if f.blocked else 0)
        for i, t in enumerate(f.targets):                                  # dA = u^T x
            ops.lora_grad_tn(x, u[:, i * r:(i + 1) * r], [(lora.grad_view(li, t, "A"), 0, x.shape[1], 0, r)], mode=1,
                             dropout=dd(li, f.proj0 + i))
        return dx

    for li in range(len(W.layers) - 1, -1, -1):
        Lw, S = W.layers[li], ctx.saved[li]
        # ---------------- MLP: h_out = h_mid + down(act)
        dact = linear_bwd(DOWN, li, dh, S.act, S)
        dgu = ops.swiglu_bwd(S.gu, dact)
        del dact
        dxn2 = linear_bwd(GU, li, dgu, S.xn2, S)
        del dgu
        dh_mid = ops.rmsnorm_bwd(S.h_mid, Lw.ln2, S.rstd2, dxn2, dres=dh)
        del dxn2
        # ---------------- attention: h_mid = h_in + o_proj(attn)
        dattn = linear_bwd(O, li, dh_mid, S.attn, S)
        dqkv = torch.empty(M, (Hq + 2 * Hkv) * D, device=dev, dtype=torch.bfloat16)
        dq, dk, dv = (dqkv[:, rows] for rows in QKV.rows(cfg))
        if layout is None:
            ops.attn_bwd(S.q, S.k, S.v, S.attn, dattn, S.lse, dq, dk, dv, B, L, Hq, Hkv, D, kv_start=ctx.ks, kv_end=ctx.ke)
        else:
            ops.attn_bwd_shared(S.q, S.k, S.v, S.attn, dattn, S.lse, dq, dk, dv, layout.U, layout.G, layout.Lp, layout.Ls, Hq, Hkv, D,
                                layout.kv_start, layout.kv_end)
        del dattn
        ops.qk_rope_bwd_(dqkv, S.qkv_pre, Hq, Hkv, D, Lw.q_norm, Lw.k_norm, ctx.pos, theta, eps)
        dxn1 = linear_bwd(QKV, li, dqkv, S.xn1, S)
        del dqkv
        dh = ops.rmsnorm_bwd(S.h_in, Lw.ln1, S.rstd1, dxn1, dres=dh_mid)
        del dxn1, dh_mid
        ctx.saved[li] = None                                              # free this layer's activations
        if on_layer_done is not None and lora is not None:
            on_layer_done(li)

    # ---------------- projector: emb rows that came from DNA features
    if ctx.aux is not None and model.dna_projection.weight.requires_grad:
        enc, row_map = ctx.aux
        if layout is not None:
            # each (feature, buffer row) pair once: a prefix row carries the gradient of the whole group and is owned by the group's
            # first row; a tail feature of every row lands in that row's suffix
            row_map = layout.owner_of(row_map)
        dE = ops.gather_rows(dh, row_map)                                  # rows with row_map < 0 (DNA pads) come back as zeros
        dE_T = ops.transpose(dE)                                           # [d_text, n']
        enc_T = ops.transpose(enc)                                         # [d_dna, n']
        gw = ops.gemm(dE_T, enc_T, out_dtype=torch.float32)                # [d_text, d_dna]
        model._proj_grad_w.add_(gw)
        ops.colsum_accumulate_(model._proj_grad_b, dE)
    return dh


def sft_step(model, input_ids, attention_mask, dna_tokenized, batch_idx_map, labels, *, backward: bool = True, grad_scale: float = 1.0):
    """One supervised step (train_dna_qwen.py:179-213 -> HF ForCausalLMLoss, loss/loss_utils.py:28-67): shift, ignore -100, mean CE.
    Returns the loss; with backward=True accumulates d(loss * grad_scale) into the LoRA / projector gradient buffers (through the LoRA
    dropout when it is on; the forward-only loss is undropped, like eval mode)."""
    dev = model._dec.embed.device
    labels = labels.to(dev)
    B, L = labels.shape
    tgt = torch.where(labels[:, 1:] == -100, torch.full_like(labels[:, 1:], -1), labels[:, 1:])           # position t predicts label t+1
    valid = tgt >= 0
    n = valid.sum().clamp(min=1).float()
    lp, ctx = policy_forward(model, input_ids, attention_mask, dna_tokenized, batch_idx_map, L - 1, save=backward, targets=tgt,
                             dropout=backward)
    loss = -(lp * valid).sum() / n
    if backward:
        policy_backward(model, ctx, (-(valid.float()) / n) * grad_scale)
    return loss


class _PolicyLogps(torch.autograd.Function):
    """Autograd bridge so `loss.backward()` (HF Trainer style) reaches the hand-written backward."""

    @staticmethod
    def forward(ctx, model, input_ids, attention_mask, dna_tokenized, batch_idx_map, keep_last, *trainable):
        logp, pctx = policy_forward(model, input_ids, attention_mask, dna_tokenized, batch_idx_map, keep_last, save=True, dropout=True)
        ctx.model, ctx.pctx, ctx.n_train = model, pctx, len(trainable)
        return logp

    @staticmethod
    def backward(ctx, dlogp):
        model = ctx.model
        lora = model._lora
        before = lora.flat_grad.clone() if lora is not None else None
        pw, pb = model._proj_grad_w.clone(), model._proj_grad_b.clone()
        policy_backward(model, ctx.pctx, dlogp)
        grads = []
        if lora is not None:
            delta = lora.flat_grad - before
            lora.flat_grad.copy_(before)                                   # autograd does the accumulation into .grad
            off = 0
            for p in lora.params:
                grads.append(delta[off:off + p.numel()].view_as(p)); off += p.numel()
        gw, gb = model._proj_grad_w - pw, model._proj_grad_b - pb
        model._proj_grad_w.copy_(pw); model._proj_grad_b.copy_(pb)
        grads += [gw, gb]
        return (None, None, None, None, None, None, *grads[:ctx.n_train])


def policy_logps_autograd(model, input_ids, attention_mask, dna_tokenized, batch_idx_map, keep_last):
    trainable = (list(model._lora.params) if model._lora is not None else []) + [model.dna_projection.weight, model.dna_projection.bias]
    return _PolicyLogps.apply(model, input_ids, attention_mask, dna_tokenized, batch_idx_map, keep_last, *trainable)
