"""fp64 references of the NT-v2 (ESM) encoder's forward kernels -- LayerNorm, the ESM rotary (qk_rope_ mode 1) and one encoder layer
as the chain of launches engine.encoder_forward makes -- and of the decoder's RMSNorm forward, with per-element error bounds for the
bf16-storage / fp32-math row kernels of elementwise.cu, and one-bug variants.  Test infrastructure: torch only, runs on CPU or GPU.

Every reference is computed in float64 from the exact bf16 inputs.  u = bf16 unit roundoff, e = 2^-24 (fp32 unit roundoff), and
n = 8 ceil(d / 256) + 5 is the longest chain of fp32 adds in a row reduction: a lane adds up to 8 ceil(d / 256) elements of its
16-byte vectors, then a 5-step warp tree.  Every bound is SAFETY times the derived value.
  LayerNorm  mu = sum(x) / d, V = sum((x - mu)^2) / d (biased, as torch's layer_norm), r = (V + eps)^-1/2, y = bf16((x - mu) r w + b)
             dmu    = n e sum|x| / d + e |mu|                                the fp32 sum and the division
             dr / r = ((n + 3) e V + dmu^2) / (2 (V + eps)) + 2^-22 + e      the fp32 squares, their sum, the division (V also picks up
                                                                              dmu^2 from the rounded mean, as sum(x - mu) = 0), the eps add
                                                                              and rsqrtf (2 ulp)
             E      = |w| r dmu + |w| |x - mu| r (dr / r + 3 e) + e (|x - mu| r |w| + |b|)   the subtraction, two products, the add
             bound  = E + u (|y| + E)                                        the output rounding.  dmu dominates on rows of large mean.
  RMSNorm    r = (mean(x^2) + eps)^-1/2 in fp32: dr / r = (n + 3) e / 2 + 2^-22;  y = bf16(w bf16(x r)) (HF Qwen3RMSNorm):
             Ez = |x| r (dr / r + e) + u (|x| r + ...)   (x r in fp32, rounded to bf16);  Ey = |w| Ez + e |w| (|x| r + Ez);
             bound = Ey + u (|y| + Ey)
  rotary     (mode 1, ESM) a = bf16(q s) on the q heads (kernel semantics, reproduced exactly by a torch bf16 multiply), a = k on the k
             heads; out_j = a_j cos t_j - a_{j+D/2} sin t_j, out_{j+D/2} = a_{j+D/2} cos t_j + a_j sin t_j (rotate-half), exact angles
             t_j = pos 10000^(-2j/D).  The kernel's angle is off by dt = 2 pos ulp(inv_freq_j) + ulp(angle) + 2^-21 (powf and the
             reciprocal, the fp32 product, sincosf), its two products and one add are fp32:
             E = (|a_j| + |a_{j+D/2}|) dt + 2 e (|a_j cos| + |a_{j+D/2} sin|),  bound = E + u (|out| + E)
  layer      encoder_layer(): ln1 -> qkv GEMM (+bias) -> rotary -> attention (D = 64, bidirectional, scale 1 on the pre-scaled q) ->
             o GEMM (+bias, +residual) -> ln2 -> gated GEMM (SiLU of the gate half) -> down GEMM (+residual).  Each step's reference
             and bound come from the bf16 tensor that step actually received (gemm_ref / attn_ref carry the GEMM and attention models).
Exact values get a bound of exactly 0 only where the tests check them bit for bit (zero LayerNorm rows give y = b).

Bugs out of reach (below the bound by construction, so no variant claims them):
  - unbiased LayerNorm variance scales r by sqrt(1 - 1/d): a relative change of ~0.5 / d, under u for every d >= 128;
  - the order of the fp32 adds in any reduction (all orders are inside n e).
"""
import math

import torch

import attn_ref as ar
import gemm_ref as gr

U = ar.U_BF16
E32 = gr.E32
SAFETY = ar.SAFETY
ROPE_THETA = 10000.0
RSQRT_REL = 2.0 ** -22          # rsqrtf: 2 ulp

# one typical kernel bug each (layernorm_ref / rmsnorm_ref / rope_esm_ref(variant=...))
VARIANTS = (
    "ln_no_bias",              # LayerNorm: b never added
    "ln_wb_swapped",           # LayerNorm: w and b exchanged
    "ln_tail_vec",             # LayerNorm: statistics over the first 256 (ceil(d / 256) - 1) columns (each lane's last vector dropped)
    "rope_k_scaled",           # rotary: k multiplied by the q scale too
    "rope_interleaved",        # rotary: GPT-J pairs (2i, 2i + 1) instead of rotate-half (i, i + D/2)
    "rope_pos_plus_1",         # rotary: angle of position + 1
    "rms_d_minus_8",           # RMSNorm: rstd over the first d - 8 columns
)


def chain_len(d):
    """n of the module doc: the longest chain of fp32 adds in a row reduction over d columns."""
    return 8 * math.ceil(d / 256) + 5


def _f64(t):
    return None if t is None else t.to(torch.float64)


# ------------------------------------------------------------------------------------------------------------------ LayerNorm
def layernorm_ref(x, w, b, eps, variant=None):
    """y = (x - mu) r w + b over rows of x [M, d] in float64, with the bound of the module doc.  Returns {"y", "b_y"}."""
    M, d = x.shape
    x, w, b = _f64(x), _f64(w)[None], _f64(b)[None]
    xs = x[:, :256 * (math.ceil(d / 256) - 1)] if variant == "ln_tail_vec" else x
    mu = xs.mean(1, keepdim=True)
    V = (xs - mu).pow(2).mean(1, keepdim=True)
    r = torch.rsqrt(V + eps)
    if variant == "ln_wb_swapped":
        w, b = b, w
    y = (x - mu) * r * w + (0.0 if variant == "ln_no_bias" else b)
    n = chain_len(d)
    xm = (x - mu).abs()
    dmu = n * E32 * x.abs().sum(1, keepdim=True) / d + E32 * mu.abs()
    rel_r = ((n + 3) * E32 * V + dmu ** 2) / (2 * (V + eps)) + RSQRT_REL + E32
    E = w.abs() * r * dmu + w.abs() * xm * r * (rel_r + 3 * E32) + E32 * (xm * r * w.abs() + b.abs())
    return {"y": y, "b_y": SAFETY * (E + U * (y.abs() + E))}


LN_FAMILIES = ("normal", "large_mean", "zero", "constant")


def layernorm_inputs(family, M, d, seed, device="cpu"):
    """Seeded bf16 rows x [M, d], w, b of one LayerNorm input family on `device` (drawn on the CPU).

    normal: N(0.3, 2^2);  large_mean: 40 + N(0, 0.5^2) (the fp32 mean's error dominates the bound);  zero: every pad token's
    embedding (y must be b bit for bit);  constant: one value per row (V = 0: r = eps^-1/2)."""
    gen = torch.Generator().manual_seed(seed)
    if family == "normal":
        x = torch.randn(M, d, generator=gen) * 2 + 0.3
    elif family == "large_mean":
        x = 40 + torch.randn(M, d, generator=gen) * 0.5
    elif family == "zero":
        x = torch.zeros(M, d)
    elif family == "constant":
        x = (torch.randn(M, 1, generator=gen) * 3).expand(M, d).clone()
    else:
        raise ValueError(family)
    w = 1 + 0.1 * torch.randn(d, generator=gen)
    b = 0.1 * torch.randn(d, generator=gen)
    return tuple(t.to(torch.bfloat16).to(device) for t in (x, w, b))


# -------------------------------------------------------------------------------------------------------------------- RMSNorm
def rmsnorm_ref(x, w, eps, variant=None):
    """rstd = (mean(x^2) + eps)^-1/2 and y = w (x rstd) in float64 with their bounds.  Returns {"y", "b_y", "rstd", "b_rstd"}."""
    M, d = x.shape
    x, w = _f64(x), _f64(w)[None]
    xs = x[:, :d - 8] if variant == "rms_d_minus_8" else x
    r = torch.rsqrt(xs.pow(2).mean(1, keepdim=True) + eps)
    rel_r = (chain_len(d) + 3) * E32 / 2 + RSQRT_REL
    y = w * x * r
    xr = x.abs() * r
    Ez = xr * (rel_r + E32)
    Ez = Ez + U * (xr + Ez)
    Ey = w.abs() * Ez + E32 * w.abs() * (xr + Ez)
    return {"y": y, "b_y": SAFETY * (Ey + U * (y.abs() + Ey)), "rstd": r[:, 0], "b_rstd": SAFETY * rel_r * r[:, 0]}


# --------------------------------------------------------------------------------------------------------------- ESM rotary
def rope_esm_ref(qk, pos, n_q, n_k, D, q_scale, variant=None):
    """The rotated q | k heads of qk [M, >= (n_q + n_k) D] (mode 1 of qk_rope_) in float64 with the bound of the module doc.

    The q heads are first scaled by q_scale and rounded to qk's dtype (the kernel's bf16(q s); a no-op for float64 input).
    pos: [M] int positions.  Returns {"y", "b_y"} of shape [M, n_q + n_k, D]."""
    M = qk.shape[0]
    H = n_q + n_k
    x = qk[:, :H * D].reshape(M, H, D)
    ks = q_scale if variant == "rope_k_scaled" else 1.0
    a = torch.cat([(x[:, :n_q] * q_scale).to(qk.dtype), (x[:, n_q:] * ks).to(qk.dtype)], 1).to(torch.float64)
    dev = a.device
    pos = pos.to(dev)
    p64 = pos.to(torch.float64) + (1.0 if variant == "rope_pos_plus_1" else 0.0)
    j = torch.arange(D // 2, device=dev, dtype=torch.float64)
    ang = p64[:, None] * ROPE_THETA ** (-2 * j / D)[None]                          # [M, D/2]
    c, s = ang.cos()[:, None], ang.sin()[:, None]
    if variant == "rope_interleaved":
        lo, hi = a[..., 0::2], a[..., 1::2]
        y = torch.stack([lo * c - hi * s, hi * c + lo * s], -1).reshape(M, H, D)
    else:
        lo, hi = a[..., :D // 2], a[..., D // 2:]
        y = torch.cat([lo * c - hi * s, hi * c + lo * s], -1)
    lo, hi = a[..., :D // 2], a[..., D // 2:]
    inv32 = (1.0 / torch.pow(torch.tensor(ROPE_THETA, dtype=torch.float32), (2 * j / D).float())).to(dev)
    dth = (2 * pos.to(torch.float64)[:, None] * gr.ulp32(inv32)[None] + gr.ulp32(pos.float()[:, None] * inv32[None]) + 2.0 ** -21)[:, None]
    E = torch.cat([(lo.abs() + hi.abs()) * dth + 2 * E32 * (lo.abs() * c.abs() + hi.abs() * s.abs()),
                   (lo.abs() + hi.abs()) * dth + 2 * E32 * (hi.abs() * c.abs() + lo.abs() * s.abs())], -1)
    return {"y": y, "b_y": SAFETY * (E + U * (y.abs() + E))}


# ------------------------------------------------------------------------------------------------------------- encoder layer
STEPS = ("ln1", "qkv", "rope", "attn", "o", "ln2", "gu", "down")


def encoder_layer(x, Lw, n_seq, S, nh, windows, eps, got=None):
    """One NT-v2 encoder layer on rows x [n_seq S, d] as engine.encoder_forward runs it, step by step.

    Lw: the layer's weights in kernel layout (packing.EncoderLayerW, or anything with its attributes; w_gu gate/up-blocked).
    windows: [(kv_start, kv_end)] per sequence.  got: the kernel's output of every step (keys of STEPS; "rope" is the rotated q | k
    columns [M, 2d]); each step's reference is then computed from the previous step's kernel output.  Without `got` the steps
    are chained on their own references, which for float64 x and weights is the layer in exact arithmetic.
    Returns {step: (ref, bound)}; ref is shaped like the kernel output of the step ([M, 2d] for "rope", [M, d] for "attn")."""
    d = x.shape[1]
    D = d // nh
    M = n_seq * S
    dev = x.device
    pos = torch.arange(S, device=dev).repeat(n_seq)
    out = {}
    inp = lambda step, ref: got[step] if got is not None else ref

    r = layernorm_ref(x, Lw.ln1_w, Lw.ln1_b, eps)
    out["ln1"] = (r["y"], r["b_y"])
    r = gr.gemm_ref(inp("ln1", r["y"]), Lw.w_qkv, bias=Lw.b_qkv)
    out["qkv"] = (r["y"], r["b_y"])
    qkv = inp("qkv", r["y"])
    r = rope_esm_ref(qkv, pos, nh, nh, D, D ** -0.5)
    out["rope"] = (r["y"].reshape(M, 2 * d), r["b_y"].reshape(M, 2 * d))
    qk = inp("rope", r["y"].reshape(M, 2 * d))
    q, k, v = (t.reshape(n_seq, S, nh, D) for t in (qk[:, :d], qk[:, d:], qkv[:, 2 * d:3 * d]))
    r = ar.attn_ref(q, k, v, None, windows, scale=1.0, causal=False)
    out["attn"] = (r["o"].reshape(M, d), r["b_o"].reshape(M, d))
    r = gr.gemm_ref(inp("attn", r["o"].reshape(M, d)), Lw.w_o, bias=Lw.b_o, residual=x)
    out["o"] = (r["y"], r["b_y"])
    x_mid = inp("o", r["y"])
    r = layernorm_ref(x_mid, Lw.ln2_w, Lw.ln2_b, eps)
    out["ln2"] = (r["y"], r["b_y"])
    r = gr.gemm_ref(inp("ln2", r["y"]), Lw.w_gu, bias=Lw.b_gu, act=1)
    out["gu"] = (r["y"], r["b_y"])
    r = gr.gemm_ref(inp("gu", r["y"]), Lw.w_down, bias=Lw.b_down, residual=x_mid)
    out["down"] = (r["y"], r["b_y"])
    return out
