"""Thin Python wrappers: PyTorch tensors in, PyTorch tensors out, math in libbioreason_b200 (C ABI).

PyTorch here is plumbing only: it owns device memory and streams.  Every op raises if its tensors
are not CUDA tensors -- there is no CPU path.
"""
from __future__ import annotations

from typing import Optional

import torch

from ._lib import COUNTER as LAUNCHES_RAW, check, ffi, lib, ptr

BF16, F32 = 0, 1
LAUNCHES = LAUNCHES_RAW   # kernels launched through the C ABI (bench.py's gpu_launches); graph replays add their captured count


def _stream():
    return ffi.cast("void*", torch.cuda.current_stream().cuda_stream)


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("bioreason_b200 ops run on CUDA tensors only (no CPU fallback)")


# ------------------------------------------------------------------ GRPO
def grpo_advantages(rewards_per_func: torch.Tensor, num_generations: int, return_stats: bool = False):
    """grpo_trainer.py:682-692."""
    _need_cuda(rewards_per_func)
    r = rewards_per_func.float().contiguous()
    rows, nf = r.shape
    adv = torch.empty(rows, device=r.device, dtype=torch.float32)
    gm = torch.empty(rows // num_generations, device=r.device, dtype=torch.float32)
    gs = torch.empty_like(gm)
    check(lib().br_grpo_advantages(ptr(r, "float*"), rows, nf, num_generations, ptr(adv, "float*"),
                                   ptr(gm, "float*"), ptr(gs, "float*"), _stream()), "grpo_advantages")
    return (adv, gm, gs) if return_stats else adv


def grpo_loss_raw(lp, old_lp, ref_lp, adv, mask, beta, eps_low, eps_high, want_grad=True):
    _need_cuda(lp, adv, mask)
    B, C = lp.shape
    lp = lp.float().contiguous()
    old_lp = None if old_lp is None else old_lp.float().contiguous()
    ref_lp = None if ref_lp is None else ref_lp.float().contiguous()
    adv = adv.float().contiguous()
    mask = mask.to(torch.int32).contiguous()
    out3 = torch.empty(3, device=lp.device, dtype=torch.float32)
    dlp = torch.empty_like(lp) if want_grad else None
    check(lib().br_grpo_loss_fwd_bwd(ptr(lp, "float*"), ptr(old_lp, "float*"), ptr(ref_lp, "float*"), ptr(adv, "float*"),
                                     ptr(mask, "int32_t*"), B, C, float(beta), float(eps_low), float(eps_high),
                                     ptr(out3, "float*"), ptr(dlp, "float*"), _stream()), "grpo_loss")
    return out3, dlp


def grpo_loss_is_raw(lp, old_lp, ref_lp, rollout_lp, adv, mask, beta, eps_low, eps_high, is_cap, want_grad=True):
    """grpo_loss_raw with truncated importance sampling against the rollout's log-probs (br_grpo_loss_is_fwd_bwd): each token's
    policy-gradient term is weighted by min(exp(o - rollout_lp), is_cap), o = old_lp (lp when None), the KL term is not.
    Returns (out3, is_stats, dlp); is_stats = masked token means of [w, capped, o - rollout_lp, exp(o - rollout_lp) - 1 - (o - rollout_lp)]."""
    _need_cuda(lp, rollout_lp, adv, mask)
    B, C = lp.shape
    lp = lp.float().contiguous()
    old_lp = None if old_lp is None else old_lp.float().contiguous()
    ref_lp = None if ref_lp is None else ref_lp.float().contiguous()
    rollout_lp = rollout_lp.float().contiguous()
    assert rollout_lp.shape == (B, C), (rollout_lp.shape, lp.shape)
    adv = adv.float().contiguous()
    mask = mask.to(torch.int32).contiguous()
    out3 = torch.empty(3, device=lp.device, dtype=torch.float32)
    stats = torch.empty(4, device=lp.device, dtype=torch.float32)
    dlp = torch.empty_like(lp) if want_grad else None
    check(lib().br_grpo_loss_is_fwd_bwd(ptr(lp, "float*"), ptr(old_lp, "float*"), ptr(ref_lp, "float*"), ptr(rollout_lp, "float*"),
                                        ptr(adv, "float*"), ptr(mask, "int32_t*"), B, C, float(beta), float(eps_low), float(eps_high),
                                        float(is_cap), ptr(out3, "float*"), ptr(stats, "float*"), ptr(dlp, "float*"), _stream()), "grpo_loss_is")
    return out3, stats, dlp


def grpo_loss_ent_raw(lp, old_lp, ref_lp, rollout_lp, adv, mask, entropy, tau, beta, eps_low, eps_high, is_cap=2.0, want_grad=True):
    """grpo_loss_raw (grpo_loss_is_raw when rollout_lp is given) with high-entropy token selection (br_grpo_loss_ent_fwd_bwd): a token's
    policy-gradient term is kept only where mask and entropy >= tau (fp32 [1] on the device, entropy_threshold); the KL term is not
    masked.  tau = -inf gives the plain (or IS) loss bit for bit.
    Returns (out3, is_stats or None, ent_sum [1] = sum of mask * entropy, dlp)."""
    _need_cuda(lp, adv, mask, entropy, tau)
    B, C = lp.shape
    lp = lp.float().contiguous()
    old_lp = None if old_lp is None else old_lp.float().contiguous()
    ref_lp = None if ref_lp is None else ref_lp.float().contiguous()
    rollout_lp = None if rollout_lp is None else rollout_lp.float().contiguous()
    entropy = entropy.float().contiguous()
    assert entropy.shape == (B, C) and tau.dtype == torch.float32 and tau.numel() == 1, (entropy.shape, lp.shape, tau.dtype)
    adv = adv.float().contiguous()
    mask = mask.to(torch.int32).contiguous()
    out3 = torch.empty(3, device=lp.device, dtype=torch.float32)
    stats = torch.empty(4, device=lp.device, dtype=torch.float32) if rollout_lp is not None else None
    ent_sum = torch.empty(1, device=lp.device, dtype=torch.float32)
    dlp = torch.empty_like(lp) if want_grad else None
    check(lib().br_grpo_loss_ent_fwd_bwd(ptr(lp, "float*"), ptr(old_lp, "float*"), ptr(ref_lp, "float*"), ptr(rollout_lp, "float*"),
                                         ptr(adv, "float*"), ptr(mask, "int32_t*"), ptr(entropy, "float*"), ptr(tau, "float*"), B, C,
                                         float(beta), float(eps_low), float(eps_high), float(is_cap), ptr(out3, "float*"),
                                         ptr(stats, "float*"), ptr(ent_sum, "float*"), ptr(dlp, "float*"), _stream()), "grpo_loss_ent")
    return out3, stats, ent_sum, dlp


def grpo_objective_raw(lp, old_lp, ref_lp, adv, mask, beta, eps_low, eps_high, *, norm_rows=0, norm=None, sequence_level=False,
                       delta=None, rollout_lp=None, is_cap=2.0, entropy=None, tau=None, want_grad=True):
    """The GRPO objectives of later TRL releases (br_grpo_objective_fwd_bwd): token or sequence-level (GSPO) ratios, two-sided clipping
    with delta (None: off), optional truncated IS (rollout_lp) and entropy selection (entropy, tau).  Aggregation: norm_rows = B of the
    whole local batch gives "grpo" (row means / B); otherwise norm, a device fp32 [1], divides the token sum (bnpo, dr_grpo, dapo).
    Returns (out7, is_sums or None, ent_sum or None, dlp); out7 = [loss, sum of row-mean kl, clip, low, high, region, tokens] are
    sums over this call's rows, so row chunks add up; is_sums are the masked sums behind grpo_loss_is_raw's means."""
    _need_cuda(lp, adv, mask, norm, rollout_lp, entropy, tau)
    B, C = lp.shape
    assert (norm_rows > 0) != (norm is not None), "give norm_rows (grpo) or norm (bnpo / dr_grpo / dapo)"
    lp = lp.float().contiguous()
    old_lp = None if old_lp is None else old_lp.float().contiguous()
    ref_lp = None if ref_lp is None else ref_lp.float().contiguous()
    adv = adv.float().contiguous()
    mask = mask.to(torch.int32).contiguous()
    opt = ffi.new("br_grpo_objective*")
    opt.sequence_level = 1 if sequence_level else 0
    opt.delta = float("inf") if delta is None else float(delta)
    opt.norm_rows = int(norm_rows)
    if norm is not None:
        norm = norm.float().reshape(1).contiguous()
        opt.norm = ptr(norm, "float*")
    is_sums = ent_sum = None
    if rollout_lp is not None:
        rollout_lp = rollout_lp.float().contiguous()
        assert rollout_lp.shape == (B, C), (rollout_lp.shape, lp.shape)
        is_sums = torch.empty(4, device=lp.device, dtype=torch.float32)
        opt.rollout_lp, opt.is_cap, opt.is_sums = ptr(rollout_lp, "float*"), float(is_cap), ptr(is_sums, "float*")
    if entropy is not None:
        entropy = entropy.float().contiguous()
        assert entropy.shape == (B, C) and tau is not None and tau.dtype == torch.float32 and tau.numel() == 1, (entropy.shape, lp.shape)
        ent_sum = torch.empty(1, device=lp.device, dtype=torch.float32)
        opt.entropy, opt.tau, opt.ent_sum = ptr(entropy, "float*"), ptr(tau, "float*"), ptr(ent_sum, "float*")
    out7 = torch.empty(7, device=lp.device, dtype=torch.float32)
    dlp = torch.empty_like(lp) if want_grad else None
    check(lib().br_grpo_objective_fwd_bwd(ptr(lp, "float*"), ptr(old_lp, "float*"), ptr(ref_lp, "float*"), ptr(adv, "float*"),
                                          ptr(mask, "int32_t*"), B, C, float(beta), float(eps_low), float(eps_high), opt,
                                          ptr(out7, "float*"), ptr(dlp, "float*"), _stream()), "grpo_objective")
    return out7, is_sums, ent_sum, dlp


SCALE_REWARDS = {"group": 0, "batch": 1, "none": 2}


def grpo_advantages_scaled(rewards_per_func: torch.Tensor, num_generations: int, scale_rewards: str = "group"):
    """TRL's scale_rewards: (r - group mean) / (std + 1e-4) with the group std ("group", grpo_advantages' bits) or the std of all rows
    ("batch"), or r - group mean ("none"); unbiased stds.  Returns (advantages, std_used [rows], zero_std [rows] int32); in "none"
    mode std_used is the group std."""
    _need_cuda(rewards_per_func)
    r = rewards_per_func.float().contiguous()
    rows, nf = r.shape
    adv = torch.empty(rows, device=r.device, dtype=torch.float32)
    sd = torch.empty_like(adv)
    zero = torch.empty(rows, device=r.device, dtype=torch.int32)
    check(lib().br_grpo_advantages_scaled(ptr(r, "float*"), rows, nf, num_generations, SCALE_REWARDS[scale_rewards], ptr(adv, "float*"),
                                          ptr(sd, "float*"), ptr(zero, "int32_t*"), _stream()), "grpo_advantages_scaled")
    return adv, sd, zero


def eos_mask_truncated(completion_ids: torch.Tensor, eos_id: int):
    """eos_mask with the rows that hold no EOS zeroed (mask_truncated_completions); returns (mask int32 [B, C], lengths int32 [B]), the
    lengths counted before the zeroing."""
    _need_cuda(completion_ids)
    ids = completion_ids.to(torch.int64).contiguous()
    B, C = ids.shape
    m = torch.empty(B, C, device=ids.device, dtype=torch.int32)
    n = torch.empty(B, device=ids.device, dtype=torch.int32)
    check(lib().br_eos_mask_truncated(ptr(ids, "int64_t*"), B, C, int(eos_id), ptr(m, "int32_t*"), ptr(n, "int32_t*"), _stream()),
          "eos_mask_truncated")
    return m, n


def entropy_threshold(entropy: torch.Tensor, mask: torch.Tensor, level: float) -> torch.Tensor:
    """fp32 [1] on the device: torch.quantile(entropy[mask != 0].float(), level) bit for bit (+inf when no entry is valid), without a
    host sync.  TRL's top_entropy_quantile rho takes level = 1 - rho."""
    _need_cuda(entropy, mask)
    x = entropy.reshape(-1).float().contiguous()
    m = mask.reshape(-1).to(torch.int32).contiguous()
    assert x.numel() == m.numel(), (x.shape, m.shape)
    tau = torch.empty(1, device=x.device, dtype=torch.float32)
    check(lib().br_entropy_threshold(ptr(x, "float*"), ptr(m, "int32_t*"), x.numel(), float(level), ptr(tau, "float*"), _stream()),
          "entropy_threshold")
    return tau


class _GRPOLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, lp, old_lp, ref_lp, adv, mask, beta, eps_low, eps_high):
        out3, dlp = grpo_loss_raw(lp.detach(), old_lp, ref_lp, adv, mask, beta, eps_low, eps_high)
        ctx.save_for_backward(dlp)
        ctx.mark_non_differentiable(out3)
        return out3[0].clone(), out3

    @staticmethod
    def backward(ctx, g, _g3):
        (dlp,) = ctx.saved_tensors
        return dlp * g, None, None, None, None, None, None, None


def grpo_loss(lp, old_lp, ref_lp, adv, mask, beta=0.04, eps_low=0.2, eps_high=0.2):
    """grpo_trainer.py:786-812 -> (loss, out3=[loss, mean_kl, clip_ratio]); differentiable w.r.t. lp."""
    return _GRPOLoss.apply(lp, old_lp, ref_lp, adv, mask, beta, eps_low, eps_high)


def eos_mask(completion_ids: torch.Tensor, eos_id: int) -> torch.Tensor:
    """grpo_trainer.py:605-609."""
    _need_cuda(completion_ids)
    ids = completion_ids.to(torch.int64).contiguous()
    B, C = ids.shape
    m = torch.empty(B, C, device=ids.device, dtype=torch.int32)
    check(lib().br_eos_mask(ptr(ids, "int64_t*"), B, C, int(eos_id), ptr(m, "int32_t*"), _stream()), "eos_mask")
    return m


# ------------------------------------------------------------------ GEMM
def _row_major_2d(t):
    assert t.dim() == 2 and t.stride(1) == 1, "need a 2-D tensor with contiguous last dim"
    return t.stride(0)


def lora_dropout_desc(drop, layer: int, proj: int, r: int):
    """br_lora_dropout for projection `proj` (packing.TARGETS index; block i of a fused linear is FusedLinear.proj0 + i, see
    packing.LINEARS) of decoder layer `layer`.
    drop: engine.LoraDropout (seed, pass id, threshold, row offset)."""
    d = ffi.new("br_lora_dropout*")
    d.seed = int(drop.seed) & 0xFFFFFFFFFFFFFFFF
    setattr(d, "pass", int(drop.pass_id) & 0xFFFFFFFF)
    d.layer, d.proj, d.r = int(layer), int(proj), int(r)
    d.threshold = int(drop.threshold)
    d.inv_keep = 65536.0 / (65536 - int(drop.threshold))
    d.row_offset = int(drop.row_offset)
    return d


def gemm(a: torch.Tensor, b: torch.Tensor, *, bias=None, residual=None, alpha: float = 1.0, act: int = 0,
         out: Optional[torch.Tensor] = None, out_dtype=torch.bfloat16, row_map=None, aux_out=None,
         a2=None, b2=None, dropout=None) -> torch.Tensor:
    """out[M,N] = epilogue(a[M,K] @ b[N,K].T (+ a2[M,K2] @ b2[N,K2].T)) on wgmma (bf16 in, fp32 accumulate).
    dropout: optional br_lora_dropout (lora_dropout_desc): the a2 @ b2.T segment is a LoRA up-path whose r-wide K blocks are masked."""
    _need_cuda(a, b)
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16
    M, K = a.shape
    N, Kb = b.shape
    assert K == Kb
    n_out = N // 2 if act == 1 else N
    if out is None:
        out = torch.empty(M, n_out, device=a.device, dtype=out_dtype)
    e = ffi.new("br_gemm_epilogue*")
    e.alpha = alpha
    e.act = act
    e.out_dtype = F32 if out.dtype == torch.float32 else BF16
    keep = [a, b, out]
    if bias is not None:
        e.bias = ptr(bias); e.bias_dtype = F32 if bias.dtype == torch.float32 else BF16; keep.append(bias)
    if residual is not None:
        assert residual.dtype == torch.bfloat16
        e.residual = ptr(residual); e.ldr = _row_major_2d(residual); keep.append(residual)
    if row_map is not None:
        assert row_map.dtype == torch.int32
        e.row_map = ptr(row_map, "int32_t*"); keep.append(row_map)
    if aux_out is not None:
        e.aux_out = ptr(aux_out); e.ld_aux = _row_major_2d(aux_out); keep.append(aux_out)
    if a2 is not None:
        assert a2.dtype == torch.bfloat16 and b2.dtype == torch.bfloat16 and a2.shape[0] == M and b2.shape[0] == N
        e.A2 = ptr(a2); e.lda2 = _row_major_2d(a2); e.B2 = ptr(b2); e.ldb2 = _row_major_2d(b2); e.K2 = a2.shape[1]
        keep += [a2, b2]
    if dropout is not None:
        assert a2 is not None, "the dropout mask applies to the second (LoRA) segment"
        e.lora_dropout = dropout
    check(lib().br_gemm_bf16(ptr(a), _row_major_2d(a), ptr(b), _row_major_2d(b), ptr(out), _row_major_2d(out),
                             M, N, K, e, _stream()), "gemm_bf16")
    return out


def lmhead_logprob(h: torch.Tensor, w: torch.Tensor, target: torch.Tensor, scale: float = 1.0, want_entropy: bool = False):
    """Fused lm_head + log_softmax + gather (grpo_trainer.py:511-520): returns (logp[M], lse[M]) fp32.
    want_entropy: also the entropy of every row's softmax, (logp, lse, entropy[M]); logp and lse are the same bits."""
    _need_cuda(h, w, target)
    M, K = h.shape
    V = w.shape[0]
    tgt = target.to(torch.int32).contiguous()
    logp = torch.empty(M, device=h.device, dtype=torch.float32)
    lse = torch.empty(M, device=h.device, dtype=torch.float32)
    if want_entropy:
        ent = torch.empty(M, device=h.device, dtype=torch.float32)
        ws = torch.empty(lib().br_lmhead_entropy_workspace_bytes(M, V), device=h.device, dtype=torch.uint8)
        check(lib().br_lmhead_logprob_entropy_fwd(ptr(h), _row_major_2d(h), ptr(w), _row_major_2d(w), ptr(tgt, "int32_t*"), M, V, K,
                                                  float(scale), ptr(logp, "float*"), ptr(lse, "float*"), ptr(ent, "float*"), ptr(ws),
                                                  _stream()), "lmhead_logprob_entropy_fwd")
        return logp, lse, ent
    ws = torch.empty(lib().br_lmhead_workspace_bytes(M, V), device=h.device, dtype=torch.uint8)
    check(lib().br_lmhead_logprob_fwd(ptr(h), _row_major_2d(h), ptr(w), _row_major_2d(w), ptr(tgt, "int32_t*"), M, V, K,
                                      float(scale), ptr(logp, "float*"), ptr(lse, "float*"), ptr(ws), _stream()),
          "lmhead_logprob_fwd")
    return logp, lse


def lmhead_dlogits(h, w, target, lse, gscale, scale: float = 1.0, out: Optional[torch.Tensor] = None):
    """bf16 [M, V] tile-recomputed gradient of sum_m gscale[m] * logp[m] w.r.t. the logits.
    out: optional bf16 [M, V] destination with contiguous rows (any row stride that is a multiple of 8)."""
    _need_cuda(h, w, target)
    M, K = h.shape
    V = w.shape[0]
    tgt = target.to(torch.int32).contiguous()
    if out is None:
        d = torch.empty(M, V, device=h.device, dtype=torch.bfloat16)
    else:
        assert out.dtype == torch.bfloat16 and out.shape == (M, V), (out.dtype, out.shape)
        d = out
    check(lib().br_lmhead_dlogits(ptr(h), _row_major_2d(h), ptr(w), _row_major_2d(w), ptr(tgt, "int32_t*"),
                                  ptr(lse, "float*"), ptr(gscale.float().contiguous(), "float*"), M, V, K, float(scale),
                                  ptr(d), _row_major_2d(d), _stream()), "lmhead_dlogits")
    return d


# ------------------------------------------------------------------ row kernels
def rmsnorm(x, w, eps: float, out=None, want_rstd: bool = False):
    _need_cuda(x, w)
    M, d = x.shape
    if out is None:
        out = torch.empty(M, d, device=x.device, dtype=torch.bfloat16)
    rstd = torch.empty(M, device=x.device, dtype=torch.float32) if want_rstd else None
    check(lib().br_rmsnorm(ptr(x), _row_major_2d(x), ptr(w), ptr(out), _row_major_2d(out), ptr(rstd, "float*"), M, d, float(eps),
                           _stream()), "rmsnorm")
    return (out, rstd) if want_rstd else out


def seqcls_score(h, input_ids, pad_id, norm_w, eps: float, score_w, out=None, want_index: bool = False):
    """Pooled score head of a sequence-classification reward model (br_seqcls_score): h bf16 [B*L, d], the last decoder layer's
    output before the final norm; input_ids [B, L].  Per row, the rightmost column whose id != pad_id (None: the last column) is
    final-normed with norm_w and scored against score_w [n_labels, d].  Returns fp32 [B, n_labels] (and the pooled index int32 [B]
    with want_index).  out: optional fp32 [B, n_labels] destination with contiguous rows, e.g. a column of rewards_per_func."""
    _need_cuda(h, input_ids, norm_w, score_w, out)
    B, L = input_ids.shape
    n_labels, d = score_w.shape
    assert h.dtype == torch.bfloat16 and score_w.dtype == torch.bfloat16 and norm_w.dtype == torch.bfloat16
    assert h.shape == (B * L, d) and norm_w.shape == (d,), (h.shape, norm_w.shape, B, L, d)
    ids = input_ids.to(torch.int64).contiguous()
    if out is None:
        out = torch.empty(B, n_labels, device=h.device, dtype=torch.float32)
    assert out.dtype == torch.float32 and out.shape == (B, n_labels) and out.stride(1) == 1, (out.dtype, out.shape, out.stride())
    idx = torch.empty(B, device=h.device, dtype=torch.int32) if want_index else None
    check(lib().br_seqcls_score(ptr(h), _row_major_2d(h), ptr(ids, "int64_t*"), B, L, -1 if pad_id is None else int(pad_id), ptr(norm_w),
                                float(eps), ptr(score_w), _row_major_2d(score_w), n_labels, d, ptr(out, "float*"), out.stride(0),
                                ptr(idx, "int32_t*"), _stream()), "seqcls_score")
    return (out, idx) if want_index else out


def layernorm(x, w, b, eps: float, out=None):
    _need_cuda(x, w, b)
    M, d = x.shape
    if out is None:
        out = torch.empty(M, d, device=x.device, dtype=torch.bfloat16)
    check(lib().br_layernorm(ptr(x), _row_major_2d(x), ptr(w), ptr(b), ptr(out), _row_major_2d(out), M, d, float(eps), _stream()),
          "layernorm")
    return out


def qk_rope_(qkv, n_q, n_k, head_dim, positions, theta, *, q_norm_w=None, k_norm_w=None, eps=1e-6, q_scale=1.0, mode=0, out=None, rope=None):
    """On the fused QKV buffer [M, >= (n_q+n_k)*head_dim]: in place, or (out=) into a separate [M, >= (n_q+n_k)*head_dim] buffer so the
    pre-norm values stay available for the backward.  rope: optional cos/sin table from rope_table() (decoder rows, mode 0)."""
    _need_cuda(qkv, positions)
    assert positions.dtype == torch.int32 and positions.numel() == qkv.shape[0]
    check(lib().br_qk_rope_ex(ptr(qkv), _row_major_2d(qkv), ptr(out), _row_major_2d(out) if out is not None else 0, qkv.shape[0], n_q, n_k, head_dim,
                              ptr(q_norm_w), ptr(k_norm_w), ptr(positions, "int32_t*"), float(theta), float(eps), float(q_scale), mode,
                              ptr(rope, "float*"), rope.shape[0] if rope is not None else 0, _stream()), "qk_rope")
    return qkv if out is None else out


def embed_gather(ids, table, keep=None, out=None):
    _need_cuda(ids, table)
    ids = ids.reshape(-1).to(torch.int64).contiguous()
    M, d = ids.numel(), table.shape[1]
    if out is None:
        out = torch.empty(M, d, device=table.device, dtype=torch.bfloat16)
    if keep is not None:
        keep = keep.reshape(-1).to(torch.int32).contiguous()
    check(lib().br_embed_gather(ptr(ids, "int64_t*"), ptr(table), _row_major_2d(table), table.shape[0], ptr(out),
                                _row_major_2d(out), M, d, ptr(keep, "int32_t*"), _stream()), "embed_gather")
    return out


def scatter_rows_(dst, src, row_map):
    _need_cuda(dst, src, row_map)
    assert row_map.dtype == torch.int32
    check(lib().br_scatter_rows(ptr(src), _row_major_2d(src), ptr(row_map, "int32_t*"), ptr(dst), _row_major_2d(dst),
                                src.shape[0], src.shape[1], _stream()), "scatter_rows")
    return dst


def gather_rows(src, idx, out=None):
    _need_cuda(src, idx)
    assert idx.dtype == torch.int32
    if out is None:
        out = torch.empty(idx.numel(), src.shape[1], device=src.device, dtype=torch.bfloat16)
    check(lib().br_gather_rows(ptr(src), _row_major_2d(src), ptr(idx, "int32_t*"), ptr(out), _row_major_2d(out),
                               idx.numel(), src.shape[1], _stream()), "gather_rows")
    return out


# ------------------------------------------------------------------ attention
def attn_fwd(q, k, v, B, L, n_q, n_kv, head_dim, *, kv_start=None, kv_end=None, scale=None, causal=True, want_lse=False, out=None):
    """q/k/v: 2-D views [B*L, heads*head_dim] (may alias one fused QKV buffer)."""
    _need_cuda(q, k, v)
    if out is None:
        out = torch.empty(B * L, n_q * head_dim, device=q.device, dtype=torch.bfloat16)
    lse = torch.empty(B, n_q, L, device=q.device, dtype=torch.float32) if want_lse else None
    if scale is None:
        scale = head_dim ** -0.5
    check(lib().br_attn_fwd(ptr(q), _row_major_2d(q), ptr(k), _row_major_2d(k), ptr(v), _row_major_2d(v), ptr(out), _row_major_2d(out),
                            ptr(lse, "float*"), B, L, n_q, n_kv, head_dim, ptr(kv_start, "int32_t*"), ptr(kv_end, "int32_t*"),
                            float(scale), 1 if causal else 0, _stream()), "attn_fwd")
    return (out, lse) if want_lse else out


def attn_fwd_shared(q, k, v, U, G, Lp, Ls, n_q, n_kv, head_dim, kv_start, kv_end, *, scale=None, want_lse=False, out=None):
    """Causal attention over the shared-prefix layout (br_attn_fwd_shared): q/k/v are 2-D views [U*Lp + U*G*Ls, heads*head_dim];
    kv_start [U] per group, kv_end [U*G] per row.  Returns out (and (lse_prefix [U, Hq, Lp], lse_suffix [U*G, Hq, Ls]))."""
    _need_cuda(q, k, v, kv_start, kv_end)
    N = U * Lp + U * G * Ls
    assert q.shape[0] == N and kv_start.dtype == torch.int32 and kv_end.dtype == torch.int32
    if out is None:
        out = torch.empty(N, n_q * head_dim, device=q.device, dtype=torch.bfloat16)
    lse_p = torch.empty(U, n_q, Lp, device=q.device, dtype=torch.float32)
    lse_s = torch.empty(U * G, n_q, Ls, device=q.device, dtype=torch.float32)
    if scale is None:
        scale = head_dim ** -0.5
    check(lib().br_attn_fwd_shared(ptr(q), _row_major_2d(q), ptr(k), _row_major_2d(k), ptr(v), _row_major_2d(v), ptr(out), _row_major_2d(out),
                                   ptr(lse_p, "float*"), ptr(lse_s, "float*"), U, G, Lp, Ls, n_q, n_kv, head_dim, ptr(kv_start, "int32_t*"),
                                   ptr(kv_end, "int32_t*"), float(scale), _stream()), "attn_fwd_shared")
    return (out, (lse_p, lse_s)) if want_lse else out


# ------------------------------------------------------------------ decode
def skinny_scratch(max_n: int, device) -> torch.Tensor:
    return torch.zeros(lib().br_skinny_scratch_bytes(max_n), device=device, dtype=torch.uint8)


class Fp8Weight:
    """A decode weight [N, K] in weight-only FP8: `q` is br_quantize_rows_e4m3's opaque e4m3 buffer, `scale` the fp32 per-row scales."""
    __slots__ = ("q", "scale", "shape")

    def __init__(self, q: torch.Tensor, scale: torch.Tensor, shape):
        self.q, self.scale, self.shape = q, scale, tuple(shape)


def fp8_weight_empty(N: int, K: int, device) -> Fp8Weight:
    q = torch.empty(lib().br_fp8_weight_bytes(N, K), device=device, dtype=torch.uint8)
    return Fp8Weight(q, torch.empty(N, device=device, dtype=torch.float32), (N, K))


def quantize_rows_e4m3(w: torch.Tensor, out: Optional[Fp8Weight] = None) -> Fp8Weight:
    """Per-row e4m3 quantization of a bf16 [N, K] matrix: scale = amax|row| / 448 (1 for a zero row), codes = RNE(w / scale)."""
    _need_cuda(w)
    assert w.dtype == torch.bfloat16 and w.dim() == 2
    N, K = w.shape
    if out is None:
        out = fp8_weight_empty(N, K, w.device)
    assert out.shape == (N, K)
    check(lib().br_quantize_rows_e4m3(ptr(w), _row_major_2d(w), N, K, ptr(out.q), ptr(out.scale, "float*"), _stream()), "quantize_rows_e4m3")
    return out


def skinny_gemm(x, w, scratch, *, mode=0, residual=None, out=None, sumsq_in=None, sumsq_in_n=1, sumsq_out=None, eps=0.0):
    """out[R, N] = x[R, K] @ w[N, K].T for R <= 32 decode rows (optionally with the folded-RMSNorm statistics).  `w` is a bf16
    tensor or an Fp8Weight (then w's per-row scales multiply the sums before the epilogue)."""
    if isinstance(w, Fp8Weight):
        return _skinny_gemm_fp8(x, w, scratch, mode=mode, residual=residual, out=out, sumsq_in=sumsq_in, sumsq_in_n=sumsq_in_n,
                                sumsq_out=sumsq_out, eps=eps)
    _need_cuda(x, w)
    R, K = x.shape
    N = w.shape[0]
    if out is None:
        if mode == 3:
            out = torch.empty(R, N, device=x.device, dtype=torch.float32)
        else:
            out = torch.empty(R, N // 2 if mode == 2 else N, device=x.device, dtype=torch.bfloat16)
    check(lib().br_skinny_gemm(ptr(x), _row_major_2d(x), ptr(w), _row_major_2d(w), ptr(out), _row_major_2d(out), R, N, K, mode,
                               ptr(residual), _row_major_2d(residual) if residual is not None else 0, ptr(scratch),
                               ptr(sumsq_in, "float*"), int(sumsq_in_n) if sumsq_in is not None else 0, ptr(sumsq_out, "float*"),
                               float(eps), _stream()),
          "skinny_gemm")
    return out


def _skinny_gemm_fp8(x, w, scratch, *, mode, residual, out, sumsq_in, sumsq_in_n, sumsq_out, eps):
    _need_cuda(x, w.q)
    R, K = x.shape
    N = w.shape[0]
    assert w.shape[1] == K, (w.shape, x.shape)
    if out is None:
        if mode == 3:
            out = torch.empty(R, N, device=x.device, dtype=torch.float32)
        else:
            out = torch.empty(R, N // 2 if mode == 2 else N, device=x.device, dtype=torch.bfloat16)
    check(lib().br_skinny_gemm_fp8(ptr(x), _row_major_2d(x), ptr(w.q), K, ptr(w.scale, "float*"), ptr(out), _row_major_2d(out), R, N, K, mode,
                                   ptr(residual), _row_major_2d(residual) if residual is not None else 0, ptr(scratch),
                                   ptr(sumsq_in, "float*"), int(sumsq_in_n) if sumsq_in is not None else 0, ptr(sumsq_out, "float*"),
                                   float(eps), _stream()),
          "skinny_gemm_fp8")
    return out


def embed_gather_sumsq(ids, table, out, sumsq):
    ids = ids.reshape(-1)
    assert ids.dtype == torch.int64
    check(lib().br_embed_gather_sumsq(ptr(ids, "int64_t*"), ptr(table), _row_major_2d(table), table.shape[0], ptr(out), _row_major_2d(out),
                                      ids.numel(), table.shape[1], ptr(sumsq, "float*"), _stream()), "embed_gather_sumsq")
    return out


def scale_columns_(w, scale):
    check(lib().br_scale_columns(ptr(w), _row_major_2d(w), w.shape[0], w.shape[1], ptr(scale), _stream()), "scale_columns")
    return w


def kv_write_pages(qkv_from_first_token, n_tok, n_q, n_kv, head_dim, pages, kcache, vcache):
    check(lib().br_kv_write_pages(ptr(qkv_from_first_token), _row_major_2d(qkv_from_first_token), n_tok, n_q, n_kv, head_dim,
                                  ptr(pages, "int32_t*"), ptr(kcache), ptr(vcache), _stream()), "kv_write_pages")


def decode_fused_workspace(R, n_q, n_kv, head_dim, n_slots, device):
    return torch.zeros(lib().br_decode_fused_workspace_bytes(R, n_q, n_kv, head_dim, n_slots), device=device, dtype=torch.uint8)


def rope_table(n_pos, head_dim, theta, device):
    t = torch.empty(n_pos, head_dim // 2, 2, device=device, dtype=torch.float32)
    check(lib().br_rope_table(ptr(t, "float*"), n_pos, head_dim, float(theta), _stream()), "rope_table")
    return t


def decode_attn_fused(qkv_raw, q_norm_w, k_norm_w, kcache, vcache, page_table, cur_len, G, n_q, n_kv, head_dim, n_shared_pages,
                      splits_shared, splits_private, theta, eps, workspace, out, scale=None, rope=None):
    R = qkv_raw.shape[0]
    if scale is None:
        scale = head_dim ** -0.5
    check(lib().br_decode_attn_fused(ptr(qkv_raw), _row_major_2d(qkv_raw), ptr(q_norm_w), ptr(k_norm_w), ptr(kcache), ptr(vcache),
                                     ptr(page_table, "int32_t*"), page_table.shape[1], ptr(cur_len, "int32_t*"), R, G, n_q, n_kv,
                                     head_dim, n_shared_pages, splits_shared, splits_private, float(scale), float(theta), float(eps),
                                     ptr(rope, "float*"), rope.shape[0] if rope is not None else 0,
                                     ptr(workspace), ptr(out), _row_major_2d(out), _stream()), "decode_attn_fused")
    return out


def sample_workspace(R, V, device, logp: bool = False):
    """Two-stage sampler workspace; logp=True: large enough for sample_next(..., logp=) as well."""
    n = lib().br_sample_logp_workspace_bytes(R, V) if logp else lib().br_sample_workspace_bytes(R, V)
    return torch.empty(n, device=device, dtype=torch.uint8)


def sample_next(logits, *, temperature=1.0, top_k=20, top_p=1.0, do_sample=True, uniforms=None, step=None, max_steps=1,
                eos_id=-1, pad_id=0, finished=None, tokens=None, next_ids=None, workspace=None, logp=None,
                repetition_penalty=1.0, min_p=0.0, min_new_tokens=0, presence=None):
    """logp: optional fp32 [R, max_steps]; receives log_softmax(logits)[r, token] at column step (0 for finished rows).
    repetition_penalty / min_new_tokens / min_p: HF's logits processors (br_sample_next*_proc).  presence: int32 [R, ceil(V / 32)] bitmap
    of the tokens each row has emitted (zeroed by the caller before the first draw, updated by every call), needed when
    repetition_penalty != 1.  With all three at their defaults the launches are those of the sampler without processors."""
    R, V = logits.shape
    assert logits.dtype == torch.float32
    if repetition_penalty != 1.0 or min_p != 0.0 or min_new_tokens != 0:
        _sample_next_proc(logits, R, V, temperature, top_k, top_p, do_sample, uniforms, step, max_steps, eos_id, pad_id, finished, tokens,
                          next_ids, workspace, logp, repetition_penalty, min_p, min_new_tokens, presence)
        return
    if logp is not None:
        _sample_next_logp(logits, R, V, temperature, top_k, top_p, do_sample, uniforms, step, max_steps, eos_id, pad_id, finished, tokens,
                          next_ids, workspace, logp)
        return
    if workspace is not None and (not do_sample or top_k <= 32):
        check(lib().br_sample_next_2stage(ptr(logits, "float*"), _row_major_2d(logits), R, V, float(temperature), int(top_k), float(top_p),
                                          1 if do_sample else 0, ptr(uniforms, "float*"), ptr(step, "int32_t*"), int(max_steps), int(eos_id),
                                          int(pad_id), ptr(finished, "int32_t*"), ptr(tokens, "int64_t*"), ptr(next_ids, "int64_t*"),
                                          ptr(workspace), _stream()), "sample_next_2stage")
        return
    check(lib().br_sample_next(ptr(logits, "float*"), _row_major_2d(logits), R, V, float(temperature), int(top_k), float(top_p),
                               1 if do_sample else 0, ptr(uniforms, "float*"), ptr(step, "int32_t*"), int(max_steps), int(eos_id),
                               int(pad_id), ptr(finished, "int32_t*"), ptr(tokens, "int64_t*"), ptr(next_ids, "int64_t*"), _stream()),
          "sample_next")


def _sample_next_logp(logits, R, V, temperature, top_k, top_p, do_sample, uniforms, step, max_steps, eos_id, pad_id, finished, tokens,
                      next_ids, workspace, logp):
    _need_cuda(logits, logp)
    assert logp.dtype == torch.float32 and logp.is_contiguous() and logp.shape == (R, max_steps), (logp.shape, R, max_steps)
    if workspace is not None and (not do_sample or top_k <= 32):
        assert workspace.numel() >= lib().br_sample_logp_workspace_bytes(R, V), "logp needs sample_workspace(R, V, device, logp=True)"
        check(lib().br_sample_next_2stage_logp(ptr(logits, "float*"), _row_major_2d(logits), R, V, float(temperature), int(top_k), float(top_p),
                                               1 if do_sample else 0, ptr(uniforms, "float*"), ptr(step, "int32_t*"), int(max_steps), int(eos_id),
                                               int(pad_id), ptr(finished, "int32_t*"), ptr(tokens, "int64_t*"), ptr(next_ids, "int64_t*"),
                                               ptr(logp, "float*"), ptr(workspace), _stream()), "sample_next_2stage_logp")
        return
    check(lib().br_sample_next_logp(ptr(logits, "float*"), _row_major_2d(logits), R, V, float(temperature), int(top_k), float(top_p),
                                    1 if do_sample else 0, ptr(uniforms, "float*"), ptr(step, "int32_t*"), int(max_steps), int(eos_id),
                                    int(pad_id), ptr(finished, "int32_t*"), ptr(tokens, "int64_t*"), ptr(next_ids, "int64_t*"),
                                    ptr(logp, "float*"), _stream()), "sample_next_logp")


def presence_bitmap(R, V, device):
    """The processed sampler's emitted-token bitmap: int32 [R, ceil(V / 32)], zeroed."""
    return torch.zeros(R, (V + 31) // 32, device=device, dtype=torch.int32)


def _sample_next_proc(logits, R, V, temperature, top_k, top_p, do_sample, uniforms, step, max_steps, eos_id, pad_id, finished, tokens,
                      next_ids, workspace, logp, repetition_penalty, min_p, min_new_tokens, presence):
    _need_cuda(logits, logp, presence)
    if presence is not None:
        assert presence.dtype == torch.int32 and presence.is_contiguous() and presence.shape == (R, (V + 31) // 32), \
            ("presence must be int32 [R, ceil(V / 32)] contiguous", tuple(presence.shape), R, V)
    if logp is not None:
        assert logp.dtype == torch.float32 and logp.is_contiguous() and logp.shape == (R, max_steps), (logp.shape, R, max_steps)
    proc = ffi.new("br_sample_proc*")
    proc.repetition_penalty = float(repetition_penalty)
    proc.min_p = float(min_p)
    proc.min_new_tokens = int(min_new_tokens)
    proc.presence = ptr(presence, "uint32_t*")
    if workspace is not None and (not do_sample or top_k <= 32):
        if logp is not None:
            assert workspace.numel() >= lib().br_sample_logp_workspace_bytes(R, V), "logp needs sample_workspace(R, V, device, logp=True)"
        check(lib().br_sample_next_2stage_proc(ptr(logits, "float*"), _row_major_2d(logits), R, V, float(temperature), int(top_k), float(top_p),
                                               1 if do_sample else 0, ptr(uniforms, "float*"), ptr(step, "int32_t*"), int(max_steps), int(eos_id),
                                               int(pad_id), ptr(finished, "int32_t*"), ptr(tokens, "int64_t*"), ptr(next_ids, "int64_t*"),
                                               ptr(logp, "float*"), proc, ptr(workspace), _stream()), "sample_next_2stage_proc")
        return
    check(lib().br_sample_next_proc(ptr(logits, "float*"), _row_major_2d(logits), R, V, float(temperature), int(top_k), float(top_p),
                                    1 if do_sample else 0, ptr(uniforms, "float*"), ptr(step, "int32_t*"), int(max_steps), int(eos_id),
                                    int(pad_id), ptr(finished, "int32_t*"), ptr(tokens, "int64_t*"), ptr(next_ids, "int64_t*"),
                                    ptr(logp, "float*"), proc, _stream()), "sample_next_proc")


def sample_full_workspace(R, V, device):
    """Workspace of sample_next_full (no initialisation needed)."""
    return torch.empty(lib().br_sample_full_workspace_bytes(R, V), device=device, dtype=torch.uint8)


def sample_next_full(logits, *, temperature=1.0, top_k=0, top_p=1.0, uniforms=None, step=None, max_steps=1, eos_id=-1, pad_id=0,
                     finished=None, tokens=None, next_ids=None, workspace=None, logp=None, repetition_penalty=1.0, min_p=0.0,
                     min_new_tokens=0, presence=None):
    """Sample from the full vocabulary (br_sample_next_full): any top_k >= 0 (0: top-k off), no cap on the kept set.  The keyword
    arguments mean what they mean in sample_next; workspace: sample_full_workspace(R, V, device)."""
    R, V = logits.shape
    assert logits.dtype == torch.float32
    _need_cuda(logits, logp, presence)
    assert workspace is not None and workspace.numel() >= lib().br_sample_full_workspace_bytes(R, V), \
        "sample_next_full needs sample_full_workspace(R, V, device)"
    if logp is not None:
        assert logp.dtype == torch.float32 and logp.is_contiguous() and logp.shape == (R, max_steps), (logp.shape, R, max_steps)
    proc = ffi.NULL
    if repetition_penalty != 1.0 or min_p != 0.0 or min_new_tokens != 0:
        if presence is not None:
            assert presence.dtype == torch.int32 and presence.is_contiguous() and presence.shape == (R, (V + 31) // 32), \
                ("presence must be int32 [R, ceil(V / 32)] contiguous", tuple(presence.shape), R, V)
        proc = ffi.new("br_sample_proc*")
        proc.repetition_penalty = float(repetition_penalty)
        proc.min_p = float(min_p)
        proc.min_new_tokens = int(min_new_tokens)
        proc.presence = ptr(presence, "uint32_t*")
    check(lib().br_sample_next_full(ptr(logits, "float*"), _row_major_2d(logits), R, V, float(temperature), int(top_k), float(top_p),
                                    ptr(uniforms, "float*"), ptr(step, "int32_t*"), int(max_steps), int(eos_id), int(pad_id),
                                    ptr(finished, "int32_t*"), ptr(tokens, "int64_t*"), ptr(next_ids, "int64_t*"), ptr(logp, "float*"),
                                    proc, ptr(workspace), _stream()), "sample_next_full")
    LAUNCHES[0] += (3 if 1 <= top_k < V else 0) + (3 if top_p < 1.0 else 0) + 1      # stats, the cuts' radix passes, draw


def decode_advance(step, cur_len):
    check(lib().br_decode_advance(ptr(step, "int32_t*"), ptr(cur_len, "int32_t*"), cur_len.numel(), _stream()), "decode_advance")


# ------------------------------------------------------------------ backward
def attn_bwd(q, k, v, o, dout, lse, dq, dk, dv, B, L, n_q, n_kv, head_dim, *, kv_start=None, kv_end=None, scale=None):
    if scale is None:
        scale = head_dim ** -0.5
    ws = torch.empty(lib().br_attn_bwd_workspace_bytes(B, L, n_q, head_dim), device=q.device, dtype=torch.uint8)
    check(lib().br_attn_bwd(ptr(q), _row_major_2d(q), ptr(k), _row_major_2d(k), ptr(v), _row_major_2d(v), ptr(o), _row_major_2d(o),
                            ptr(dout), _row_major_2d(dout), ptr(lse, "float*"), ptr(dq), _row_major_2d(dq), ptr(dk), _row_major_2d(dk),
                            ptr(dv), _row_major_2d(dv), B, L, n_q, n_kv, head_dim, ptr(kv_start, "int32_t*"), ptr(kv_end, "int32_t*"),
                            float(scale), ptr(ws), _stream()), "attn_bwd")


def attn_bwd_shared(q, k, v, o, dout, lse, dq, dk, dv, U, G, Lp, Ls, n_q, n_kv, head_dim, kv_start, kv_end, *, scale=None):
    """Backward of attn_fwd_shared; lse = the (lse_prefix, lse_suffix) pair it returned."""
    _need_cuda(q, k, v, o, dout, dq, dk, dv, kv_start, kv_end)
    if scale is None:
        scale = head_dim ** -0.5
    lse_p, lse_s = lse
    ws = torch.empty(lib().br_attn_bwd_shared_workspace_bytes(U, G, Lp, Ls, n_q, head_dim), device=q.device, dtype=torch.uint8)
    check(lib().br_attn_bwd_shared(ptr(q), _row_major_2d(q), ptr(k), _row_major_2d(k), ptr(v), _row_major_2d(v), ptr(o), _row_major_2d(o),
                                   ptr(dout), _row_major_2d(dout), ptr(lse_p, "float*"), ptr(lse_s, "float*"), ptr(dq), _row_major_2d(dq),
                                   ptr(dk), _row_major_2d(dk), ptr(dv), _row_major_2d(dv), U, G, Lp, Ls, n_q, n_kv, head_dim,
                                   ptr(kv_start, "int32_t*"), ptr(kv_end, "int32_t*"), float(scale), ptr(ws), _stream()), "attn_bwd_shared")


def rmsnorm_bwd(x, w, rstd, dy, dres=None, out=None):
    M, d = x.shape
    if out is None:
        out = torch.empty(M, d, device=x.device, dtype=torch.bfloat16)
    check(lib().br_rmsnorm_bwd(ptr(x), _row_major_2d(x), ptr(w), ptr(rstd, "float*"), ptr(dy), _row_major_2d(dy), ptr(dres),
                               _row_major_2d(dres) if dres is not None else 0, ptr(out), _row_major_2d(out), M, d, _stream()), "rmsnorm_bwd")
    return out


def swiglu_bwd(gu, dact, out=None):
    M, F2 = gu.shape
    if out is None:
        out = torch.empty(M, F2, device=gu.device, dtype=torch.bfloat16)
    check(lib().br_swiglu_bwd(ptr(gu), _row_major_2d(gu), ptr(dact), _row_major_2d(dact), ptr(out), _row_major_2d(out), M, F2 // 2,
                              _stream()), "swiglu_bwd")
    return out


def qk_rope_bwd_(dqkv, qk_pre, n_q, n_k, head_dim, q_norm_w, k_norm_w, positions, theta, eps):
    check(lib().br_qk_rope_bwd(ptr(dqkv), _row_major_2d(dqkv), ptr(qk_pre), _row_major_2d(qk_pre), dqkv.shape[0], n_q, n_k, head_dim,
                               ptr(q_norm_w), ptr(k_norm_w), ptr(positions, "int32_t*"), float(theta), float(eps), _stream()), "qk_rope_bwd")
    return dqkv


_LORA_WS = {}


def lora_grad_tn(big, small, segs, *, mode=0, dropout=None):
    """Deterministic wgmma TN GEMM: product[P, N] = big[M, P]^T @ small[M, N]; the blocks named by `segs` are ADDED into fp32 views.
    segs: list of (dst fp32 2-D view with contiguous rows, row_lo, row_hi, col_lo, n_cols); mode 1: one segment, dst[n, p] (transposed);
    mode 2: gate/up-blocked product rows (segment 0 = gate rows, 1 = up rows).
    dropout: optional br_lora_dropout (lora_dropout_desc): `big` is the adapter input x, masked, and the product is scaled by
    1 / (1 - p_eff), i.e. dA += inv_keep * u^T (x * m)."""
    _need_cuda(big, small)
    assert big.dtype == torch.bfloat16 and small.dtype == torch.bfloat16 and big.shape[0] == small.shape[0]
    M, P = big.shape
    N = small.shape[1]
    dev = big.device
    ws = _LORA_WS.get(dev)
    if ws is None:
        ws = _LORA_WS[dev] = torch.zeros(lib().br_lora_grad_workspace_bytes(), device=dev, dtype=torch.uint8)
    arr = ffi.new("br_lora_grad_seg[]", len(segs))
    for i, (dst, row_lo, row_hi, col_lo, n_cols) in enumerate(segs):
        assert dst.dtype == torch.float32 and dst.dim() == 2 and dst.stride(1) == 1
        arr[i].dst = ptr(dst, "float*"); arr[i].ld = dst.stride(0)
        arr[i].row_lo, arr[i].row_hi, arr[i].col_lo, arr[i].n_cols = int(row_lo), int(row_hi), int(col_lo), int(n_cols)
    if dropout is not None:
        check(lib().br_lora_grad_tn_dropout(ptr(big), _row_major_2d(big), ptr(small), _row_major_2d(small), M, P, N, int(mode), arr, len(segs),
                                            dropout, ptr(ws), _stream()), "lora_grad_tn_dropout")
        return
    check(lib().br_lora_grad_tn(ptr(big), _row_major_2d(big), ptr(small), _row_major_2d(small), M, P, N, int(mode), arr, len(segs), ptr(ws),
                                _stream()), "lora_grad_tn")


def lora_down_dropout(x, a, scale: float, dropout, out=None):
    """t[M, n_proj * r] = scale / (1 - p_eff) * ((x * m_j) @ A_j.T) for the stacked adapters a [n_proj * r, K] of one fused linear."""
    _need_cuda(x, a)
    assert x.dtype == torch.bfloat16 and a.dtype == torch.bfloat16
    M, K = x.shape
    n_proj = a.shape[0] // dropout.r
    assert a.shape[0] == n_proj * dropout.r and a.shape[1] == K
    if out is None:
        out = torch.empty(M, a.shape[0], device=x.device, dtype=torch.bfloat16)
    check(lib().br_lora_down_dropout(ptr(x), _row_major_2d(x), ptr(a), _row_major_2d(a), ptr(out), _row_major_2d(out), M, K, n_proj,
                                     float(scale), dropout, _stream()), "lora_down_dropout")
    return out


def lora_dropout_mask(dropout, M: int, K: int, device) -> torch.Tensor:
    """uint8 [M, K]: 1 where element (row_offset + m, k) of projection dropout.proj's input is kept."""
    keep = torch.empty(M, K, device=device, dtype=torch.uint8)
    check(lib().br_lora_dropout_mask(dropout, M, K, ffi.cast("uint8_t*", keep.data_ptr()), K, _stream()), "lora_dropout_mask")
    return keep


def transpose(x, out=None, pad_cols_to: int = 8):
    """bf16 [M, N] -> [N, M'] with M' = M rounded up to `pad_cols_to` (zero padded) so it can feed the TMA GEMM."""
    M, N = x.shape
    Mp = (M + pad_cols_to - 1) // pad_cols_to * pad_cols_to
    if out is None:
        out = torch.zeros(N, Mp, device=x.device, dtype=torch.bfloat16) if Mp != M else torch.empty(N, Mp, device=x.device, dtype=torch.bfloat16)
    check(lib().br_transpose_bf16(ptr(x), _row_major_2d(x), ptr(out), _row_major_2d(out), M, N, _stream()), "transpose")
    return out


def colsum_accumulate_(out, x):
    M, N = x.shape
    check(lib().br_colsum_accumulate(ptr(x), _row_major_2d(x), ptr(out, "float*"), M, N, _stream()), "colsum")
    return out
