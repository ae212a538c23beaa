"""fp64 references of the training-pass GEMMs -- the wgmma GEMM of gemm_tc5.cu with its epilogues, its fused lm-head modes (log-prob
and softmax gradient) and the LoRA-gradient GEMM of lora_grad_tc5.cu -- with a per-element error bound for the bf16-in /
fp32-accumulate kernels, seeded input families in which the tile edges decide an O(1) share of the result, and one-bug variants.
Test infrastructure: torch only, runs on CPU or GPU; oracle/ is not involved.

Every reference is computed in float64 from the exact bf16 input values.

Error model (every bound is SAFETY times the derived value).  u = bf16 unit roundoff, e = 2^-24 (fp32 unit roundoff), w = W_ACC: a
deliberately loose model of one fp32 tensor-core accumulation relative to the sum of |terms| (as in attn_ref.py).  How the tensor
cores round inside a k16 step is not documented, so w is an assumption, not a derived constant.  Where the terms of a row share a sign
(same_sign: the peaked and tail_max lm-head rows) the running sum is as large as the result, and the ceil(K/16) k16 chunks added one
after another are charged in full: w = max(W_ACC, (ceil(K/16) + 1) e).  S = sum_k |a_k b_k| per output (a masked segment adds
inv_keep * its kept |terms|), E(x) = 2^-21 + 2^-23 |x| is the relative error of __expf(x) (ex2.approx plus the rounding of x log2 e).
  GEMM acc   dacc = |alpha| w S + 2e (|alpha acc| + |bias|)                lin = alpha acc + bias, formed in fp32
  GEMM out   fp32: dacc (+ u |lin| + e |y| with a residual: lin is rounded to bf16 before the add);  bf16 out: the same + u |y|
  aux        dacc + u |lin|                                                the pre-activation, rounded to bf16
  SiLU       (1.1 eg + |G| E(G) / 4 + (u + e) |silu G|) (|U| + eu) + |silu G| eu + (u + e) |y|     y = silu(G) U;  gate G, up U are
             lin columns, eg = dacc_G + u |G|, eu = dacc_U + u |U| (both rounded to bf16 before the activation); |silu'| <= 1.1;
             silu(g) = g / (1 + __expf(-g)) is rounded to bf16, the product to bf16
  lse        sum_j p_j dz_j + 2^-20 + 2^-22 sum_j p_j (zmax - z_j) + (40 + ceil(nt / 32)) e + ulp(log s) + ulp(lse)
             dz_j = |scale| w S_j + e |z_j| (z = scale * acc in fp32); the __expf terms: each exp argument x - m is at most zmax - z_j
             in size, twice (in the tile and in the combine); the positive sums: 32 adds in a tile, 2 shuffles, ceil(nt / 32)
             partials per lane of the combine and a 5-step warp sum; then logf (1 ulp) and the final add.  nt = ceil(V / 128).
  logp       dz_t + b_lse + e |logp|                                       exactly 0 for t = -1
  dlogits    |gs| p expm1(dz + e |a| + E(a)) + 2e |gs| (p + onehot) + u |d| + |gs| 2^-125 + 2^-134
             a = z - L with L the fp32 lse the kernel is given, p = exp(a), d = gs (onehot - p).  |gs| 2^-125: an exp that underflows
             fp32 (a < -87.3: __expf flushes to 0).  2^-134: the kernels are built without -ftz, so a product gs p below 2^-126 stays
             an fp32 subnormal and is rounded to a bf16 subnormal; those are 2^-133 apart, so u |d| does not cover its rounding
  LoRA grad  w inv_keep S + 2e (|prev| + |prev + v|)                      v = big^T small summed over the tokens in fp32, split-K
             partials added in fp32 (at most 16 adds, inside w), then added to the destination in fp32
Outputs that must be exact get a bound of exactly 0: an all-zero product (a zero row, a row of a tail family outside its tile), logp of
a t = -1 row.  Whatever a kernel must not write is checked bit for bit by the tests, not through a bound.
"""
import math

import torch

from attn_ref import SAFETY, U_BF16, W_ACC

E32 = 2.0 ** -24
TILE = 128                    # column tile of the lm-head partials, row tile of the LoRA-gradient product
BK = 64                       # K block of the GEMM, token block of the LoRA gradient

GEMM_VARIANTS = ("bias_half", "no_k_tail", "wrong_mask")
LMHEAD_VARIANTS = ("no_last_tile", "no_rescale", "tgt_neighbour", "no_scale_dlogits", "no_onehot_odd")
LORA_VARIANTS = ("no_last_split", "gate_up_swapped", "no_token_tail")


def acc_weight(K, same_sign=False):
    """w of the module doc for a K-long accumulation."""
    return max(W_ACC, (math.ceil(K / 16) + 1) * E32) if same_sign else W_ACC


def ulp32(x):
    """Unit in the last place of the fp32 values nearest x (float64 result)."""
    _, e = torch.frexp(x.to(torch.float32).abs())
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), (e - 24).to(torch.int64))


def exp_err(x):
    """E(x): relative error of __expf(x)."""
    return 2.0 ** -21 + 2.0 ** -23 * x.abs()


def _f64(t):
    return None if t is None else t.to(torch.float64)


def worst_ratio(got, ref, bound):
    """max |got - ref| / bound (float64).  Where bound == 0 the values must be equal (0 / inf otherwise); NaN counts as inf."""
    got, ref, bound = got.to(torch.float64), ref.to(torch.float64), bound.to(torch.float64)
    eq = got == ref
    diff = torch.where(eq, torch.zeros_like(got), (got - ref).abs())
    ratio = torch.where(bound > 0, diff / torch.where(bound > 0, bound, 1.0), torch.where(diff > 0, math.inf, 0.0))
    ratio = torch.where(torch.isnan(ratio), math.inf, ratio)
    return ratio.max().item() if ratio.numel() else 0.0


# ------------------------------------------------------------------------------------------------------------------------ GEMM
def gemm_ref(a, b, *, alpha=1.0, bias=None, residual=None, act=0, out_f32=False, a2=None, b2=None, masks=None, inv_keep=1.0,
             same_sign=False, variant=None):
    """y = epilogue(alpha (a b^T + a2 b2^T) + bias), as ops.gemm computes it, in float64 (see the module doc), with its bound.

    masks: with a2 / b2, the LoRA dropout of the second segment: one bool [M, N] keep mask per r-wide K block (projection) of a2,
    and that block's product is multiplied by mask * inv_keep.  act=1: gated SiLU over column blocks of 16 = 8 gate | 8 up.
    variant: one of GEMM_VARIANTS (compare it against the bounds of the correct reference).
    Returns a dict of float64 tensors: y, b_y and, for act=1, aux, b_aux (the pre-activation lin)."""
    dev = a.device
    M, K = a.shape
    N = b.shape[0]
    a, b = _f64(a), _f64(b)
    w = acc_weight(K + (0 if a2 is None else a2.shape[1]), same_sign)
    kk = (K // BK) * BK if variant == "no_k_tail" else K
    acc = a[:, :kk] @ b[:, :kk].T
    S = a.abs() @ b.abs().T
    if a2 is not None:
        a2, b2 = _f64(a2), _f64(b2)
        K2 = a2.shape[1]
        k2 = (K2 // BK) * BK if variant == "no_k_tail" else K2
        if masks is None:
            acc = acc + a2[:, :k2] @ b2[:, :k2].T
            S = S + a2.abs() @ b2.abs().T
        else:
            n = len(masks)
            r = K2 // n
            assert r * n == K2
            if variant == "wrong_mask":
                assert n >= 2, "wrong_mask needs two projections"
            for j in range(n):
                sl = slice(j * r, min((j + 1) * r, k2))
                m = masks[(j + 1) % n if variant == "wrong_mask" else j].to(dev, torch.float64) * inv_keep
                acc = acc + m * (a2[:, sl] @ b2[:, sl].T)
                S = S + masks[j].to(dev, torch.float64) * inv_keep * (a2[:, j * r:(j + 1) * r].abs() @ b2[:, j * r:(j + 1) * r].abs().T)
    lin = alpha * acc
    babs = torch.zeros(N, dtype=torch.float64, device=dev)
    if bias is not None:
        bias = _f64(bias).to(dev)
        babs = bias.abs()
        if variant == "bias_half":
            src = torch.arange(N, device=dev) ^ TILE
            bias = torch.where(src < N, bias[src.clamp(max=N - 1)], 0.0)
        lin = lin + bias[None]
    dacc = abs(alpha) * w * S + 2 * E32 * (abs(alpha) * acc.abs() + babs[None])
    u = U_BF16
    out = {}
    if act == 1:
        G = lin.view(M, N // 16, 2, 8)[:, :, 0].reshape(M, N // 2)
        U = lin.view(M, N // 16, 2, 8)[:, :, 1].reshape(M, N // 2)
        dG = dacc.view(M, N // 16, 2, 8)[:, :, 0].reshape(M, N // 2)
        dU = dacc.view(M, N // 16, 2, 8)[:, :, 1].reshape(M, N // 2)
        sg = torch.nn.functional.silu(G)
        y = sg * U
        eg, eu = dG + u * G.abs(), dU + u * U.abs()
        es = 1.1 * eg + G.abs() * exp_err(G) / 4 + (u + E32) * sg.abs()
        out["y"] = y
        out["b_y"] = SAFETY * (es * (U.abs() + eu) + sg.abs() * eu + (u + E32) * y.abs())
        out["aux"] = lin
        out["b_aux"] = SAFETY * (dacc + u * lin.abs())
        return out
    if residual is not None:
        y = lin + _f64(residual).to(dev)
        b_y = dacc + u * lin.abs() + E32 * y.abs()
    else:
        y = lin
        b_y = dacc
    if not out_f32:
        b_y = b_y + u * y.abs()
    out["y"] = y
    out["b_y"] = SAFETY * b_y
    return out


def make_gemm_inputs(family, M, N, K, *, seed=0, device="cpu"):
    """Seeded bf16 a [M, K], b [N, K] on `device`.

    random : a ~ N(0, 1), b ~ N(0, 1 / K).
    tail_k : only the last K % 64 columns (the partial last K block; the last 64 when K % 64 == 0) are non-zero.
    tail_mn: a is non-zero only in the rows of the last 128-row tile, b only in the rows of the last 128-column tile: every
             non-zero output lies in the last, partial M / N tile."""
    gen = torch.Generator(device=device).manual_seed(seed)
    a = torch.randn(M, K, generator=gen, device=device)
    b = torch.randn(N, K, generator=gen, device=device) / math.sqrt(K)
    if family == "tail_k":
        k0 = K - (K % BK or BK)
        a[:, :k0] = 0
        b[:, :k0] = 0
    elif family == "tail_mn":
        a[:((M - 1) // TILE) * TILE] = 0
        b[:((N - 1) // TILE) * TILE] = 0
    elif family != "random":
        raise ValueError(family)
    return a.to(torch.bfloat16), b.to(torch.bfloat16)


# --------------------------------------------------------------------------------------------------------------------- lm-head
def lmhead_ref(h, w, tgt, scale=1.0, *, lse_used=None, gs=None, same_sign=False, variant=None, vchunk=16384):
    """z = scale h w^T;  lse = logsumexp(z);  logp = z[t] - lse (0 for t = -1);  with lse_used (the fp32 lse handed to the dlogits
    kernel) and gs: d = gs (onehot(t) - exp(z - lse_used)).  All float64, with the bounds of the module doc.  w is read in chunks of
    `vchunk` rows so only [M, V] float64 buffers are held (call it on row blocks of a large M).
    variant: one of LMHEAD_VARIANTS (the bounds it returns are those of the correct reference).
    Returns a dict: lse, logp, b_lse, b_logp and, with lse_used, d, b_d ([M, V])."""
    dev = h.device
    M, K = h.shape
    V = w.shape[0]
    h = _f64(h)
    ww = acc_weight(K, same_sign)
    z = torch.empty(M, V, dtype=torch.float64, device=dev)
    S = torch.empty_like(z)
    for v0 in range(0, V, vchunk):
        wc = _f64(w[v0:v0 + vchunk])
        z[:, v0:v0 + vchunk] = h @ wc.T
        S[:, v0:v0 + vchunk] = h.abs() @ wc.abs().T
        del wc
    z *= scale
    dz = abs(scale) * ww * S + E32 * z.abs()
    del S
    nt = math.ceil(V / TILE)
    tgt = tgt.to(dev, torch.int64)
    has = tgt >= 0
    tc = tgt.clamp(min=0)
    zmax = z.amax(1, keepdim=True)
    ez = torch.exp(z - zmax)
    s = ez.sum(1)
    lse = torch.log(s) + zmax[:, 0]
    p = ez / s[:, None]
    del ez
    b_lse = ((p * dz).sum(1) + 2.0 ** -20 + 2.0 ** -22 * (p * (zmax - z)).sum(1) + (40 + math.ceil(nt / 32)) * E32
             + ulp32(torch.log(s)) + ulp32(lse))
    out = {"b_lse": SAFETY * b_lse}
    if variant == "no_last_tile":
        zl = z[:, :(nt - 1) * TILE]
        out["lse"] = torch.logsumexp(zl, 1) if zl.shape[1] else torch.full_like(lse, -math.inf)
    elif variant == "no_rescale":
        zp = torch.nn.functional.pad(z, (0, nt * TILE - V), value=-math.inf).view(M, nt, TILE)
        mt = zp.amax(2)
        out["lse"] = torch.log(torch.exp(zp - mt[..., None]).sum((1, 2))) + mt.amax(1)
    else:
        out["lse"] = lse
    src = tc ^ 1 if variant == "tgt_neighbour" else tc
    out["logp"] = torch.where(has, z.gather(1, src.clamp(max=V - 1)[:, None])[:, 0] - out["lse"], 0.0)
    logp = z.gather(1, tc[:, None])[:, 0] - lse
    out["b_logp"] = torch.where(has, SAFETY * (dz.gather(1, tc[:, None])[:, 0] + b_lse + E32 * logp.abs()), 0.0)
    if lse_used is not None:
        L = _f64(lse_used).to(dev)[:, None]
        g = _f64(gs).to(dev)[:, None]
        onehot = torch.zeros_like(z)
        oh_rows = has & (tgt % 2 == 0) if variant == "no_onehot_odd" else has
        onehot[torch.nonzero(oh_rows)[:, 0], tc[oh_rows]] = 1.0
        a = z - L
        pe = torch.exp(a)
        zz = z / scale if variant == "no_scale_dlogits" else z
        out["d"] = g * (onehot - torch.exp(zz - L))
        onehot_true = torch.zeros_like(z)
        onehot_true[torch.nonzero(has)[:, 0], tc[has]] = 1.0
        d_true = g * (onehot_true - pe)
        out["b_d"] = SAFETY * (g.abs() * pe * torch.expm1(dz + E32 * a.abs() + exp_err(a)) + 2 * E32 * g.abs() * (pe + onehot_true)
                               + U_BF16 * d_true.abs() + g.abs() * 2.0 ** -125 + 2.0 ** -134)
    return out


def lmhead_targets(M, V, seed=0):
    """int64 [M]: random classes, -1 on every 7th row, and the edge classes 0, 1, V - 1, V - 2 and the first and last column of the
    last two 128-column tiles on the first rows that are not -1."""
    gen = torch.Generator().manual_seed(seed)
    t = torch.randint(0, V, (M,), generator=gen)
    nt = math.ceil(V / TILE)
    edge = [0, 1, V - 1, V - 2, (nt - 2) * TILE, (nt - 1) * TILE - 1, (nt - 1) * TILE, V - 1]
    edge = [c for c in edge if 0 <= c < V]
    rows = [m for m in range(M) if m % 7]
    for m, c in zip(rows, edge):
        t[m] = c
    t[::7] = -1
    return t


LM_FAMILIES = ("random", "zero_row", "peaked", "tail_max", "far_negative")


def make_lmhead_weight(V, K, *, seed=0, device="cpu"):
    """Seeded bf16 lm-head weight [V, K] ~ N(0, 9 / K)."""
    gen = torch.Generator(device=device).manual_seed(seed)
    return (torch.randn(V, K, generator=gen, device=device) * (3.0 / math.sqrt(K))).to(torch.bfloat16)


def _logits32(x, w, chunk=16384):
    """fp32 x [M, K] @ w[V, K]^T, reading w in row chunks."""
    return torch.cat([x.float() @ w[v0:v0 + chunk].float().T for v0 in range(0, w.shape[0], chunk)], 1)


def make_lmhead_inputs(family, w, M, tgt, *, scale=1.0, seed=0):
    """Seeded bf16 h [M, K] on w's device for one input family (w from make_lmhead_weight); returns (h, tgt, same_sign).

    random      : h ~ N(0, 1): logits with std ~ 3 |scale|.
    zero_row    : random, with every other row 0 (z = 0, lse = log V).
    peaked      : h = alpha w_c with c the target (a random class on t = -1 rows): z_c exceeds every other logit by >= 30, so p_c
                  rounds to 1 and d_c cancels.  The terms of z_c share a sign.
    tail_max    : h = alpha (w_c + beta (w_a + w_b)), beta = 0.5 (less where that would bring a, b level with c): the row's largest
                  logit c, ahead by >= 8, sits in the last (partial) 128-column tile, a second cluster a, b in tile 0; every third row
                  (but the t = -1 rows) gets c as its target.
    far_negative: h ~ N(0, 15^2): logits with std ~ 45, most of them more than 87 below the lse (exp underflows fp32)."""
    V, K = w.shape
    device = w.device
    gen = torch.Generator(device=device).manual_seed(seed)
    tgt = tgt.clone()
    h = torch.randn(M, K, generator=gen, device=device)
    same_sign = False
    if family == "zero_row":
        h[::2] = 0
    elif family == "far_negative":
        h *= 15.0
    elif family in ("peaked", "tail_max"):
        same_sign = True
        lo = (math.ceil(V / TILE) - 1) * TILE
        g2 = torch.Generator().manual_seed(seed + 1)
        rnd = lambda n, a, b: torch.randint(a, b, (n,), generator=g2)
        wf = lambda idx: w[idx.to(device)].float()
        if family == "peaked":
            c = torch.where(tgt >= 0, tgt, rnd(M, 0, V))
            need = 30.0
            dirs = wf(c)
        else:
            c = torch.where(tgt >= lo, tgt, rnd(M, lo, V))
            pick = (torch.arange(M) % 3 == 2) & (tgt >= 0)
            tgt[pick] = c[pick]
            n0 = min(TILE, V)                                 # two classes of tile 0 other than c and each other
            ab = torch.tensor([[x for x in torch.randperm(n0, generator=g2).tolist() if x != int(c[m])][:2] for m in range(M)])
            need = 8.0
            cluster = wf(ab[:, 0]) + wf(ab[:, 1])
        cd = c.to(device)[:, None]

        def gap(x):
            z = abs(scale) * _logits32(x, w)
            return z.gather(1, cd)[:, 0] - z.scatter(1, cd, -math.inf).amax(1)
        if family == "tail_max":                             # a weaker cluster on the rows where it would rival c (small K, V)
            dirs = wf(c) + 0.5 * cluster
            for beta in (0.25, 0.1):
                weak = gap(dirs) < 1.0
                dirs[weak] = wf(c)[weak] + beta * cluster[weak]
        unit = gap(dirs).clamp(min=1e-3)
        for margin in (1.1, 1.3, 1.6, 2.0):                 # h is rounded to bf16: solve with a margin, check on the rounded h
            h = (((need * margin) / unit)[:, None] * dirs).to(torch.bfloat16).float()
            if (gap(h) >= need).all():
                break
        assert (gap(h) >= need).all(), f"{family}: logit gap {need} not reached"
    elif family != "random":
        raise ValueError(family)
    return h.to(torch.bfloat16), tgt, same_sign


# ---------------------------------------------------------------------------------------------------------------- LoRA gradient
def lora_splits(M, P, n_sms):
    """Token ranges [lo, hi) of the non-empty split-K partials of br_lora_grad_tn (its host rule), in the order they are summed."""
    tiles = math.ceil(P / TILE)
    kb_total = math.ceil(M / BK)
    splits = max(1, n_sms // tiles)
    splits = min(splits, 16, kb_total)
    if tiles > n_sms:
        splits = 1
    kb_per = math.ceil(kb_total / splits)
    return [(s * kb_per * BK, min(M, (s + 1) * kb_per * BK)) for s in range(splits) if s * kb_per < kb_total]


def lora_grad_ref(big, small, segs, mode, prev, *, mask=None, inv_keep=1.0, n_sms=132, variant=None, tok_chunk=2048):
    """dst (+)= big[M, P]^T small[M, N] placed as ops.lora_grad_tn places it, in float64, with the bound of the module doc.

    segs: [(row_lo, row_hi, col_lo, n_cols)] as ops.lora_grad_tn takes them (without the destination).  prev: the destinations'
    contents before the call, one per segment, in the shape the kernel writes: [row_hi - row_lo, n_cols] (mode 0), [N, P] (mode 1:
    dst[n, p], one segment), [P / 2, n_cols] (mode 2: product row p = 16 i + 8 s + e goes to segment s, row 8 i + e).
    mask: bool [M, P] keep mask of `big` (LoRA dropout), the product then scaled by inv_keep.  variant: one of LORA_VARIANTS.
    Returns [(ref, bound)] per segment."""
    dev = big.device
    M, P = big.shape
    N = small.shape[1]
    keep = torch.ones(M, dtype=torch.bool, device=dev)
    if variant == "no_last_split":
        lo, hi = lora_splits(M, P, n_sms)[-1]
        keep[lo:hi] = False
    elif variant == "no_token_tail":
        keep[(M // BK) * BK:] = False
    prod = torch.zeros(P, N, dtype=torch.float64, device=dev)
    S = torch.zeros_like(prod)
    for t0 in range(0, M, tok_chunk):
        bc = _f64(big[t0:t0 + tok_chunk])
        if mask is not None:
            bc = bc * mask[t0:t0 + tok_chunk].to(dev, torch.float64)
        sc = _f64(small[t0:t0 + tok_chunk])
        k = keep[t0:t0 + tok_chunk].to(torch.float64)[:, None]
        prod += (bc * k).T @ sc
        S += bc.abs().T @ sc.abs()
        del bc, sc
    prod *= inv_keep
    S *= inv_keep
    out = []
    for i, (row_lo, row_hi, col_lo, n_cols) in enumerate(segs):
        if mode == 1:
            v, s = prod.T, S.T
        elif mode == 2:
            sg = 1 - i if variant == "gate_up_swapped" else i
            v = prod.view(P // 16, 2, 8, N)[:, sg].reshape(P // 2, N)[:, col_lo:col_lo + n_cols]
            s = S.view(P // 16, 2, 8, N)[:, i].reshape(P // 2, N)[:, col_lo:col_lo + n_cols]
        else:
            v, s = prod[row_lo:row_hi, col_lo:col_lo + n_cols], S[row_lo:row_hi, col_lo:col_lo + n_cols]
        pv = _f64(prev[i]).to(dev)
        ref = pv + v
        out.append((ref, SAFETY * (W_ACC * s + 2 * E32 * (pv.abs() + ref.abs()))))
    return out


LORA_FAMILIES = ("random", "tail_token", "tail_split")


def make_lora_inputs(family, M, P, N, *, n_sms=132, seed=0, device="cpu"):
    """Seeded bf16 big [M, P] ~ N(0, 1), small [M, N] ~ N(0, 1) on `device`.

    tail_token: only the tokens past the last full 64-token block are non-zero (the whole last block when M % 64 == 0).
    tail_split: only the tokens of the last split-K partial (lora_splits) are non-zero."""
    gen = torch.Generator(device=device).manual_seed(seed)
    big = torch.randn(M, P, generator=gen, device=device)
    small = torch.randn(M, N, generator=gen, device=device)
    if family == "tail_token":
        t0 = M - (M % BK or BK)
    elif family == "tail_split":
        t0 = lora_splits(M, P, n_sms)[-1][0]
    elif family == "random":
        t0 = 0
    else:
        raise ValueError(family)
    big[:t0] = 0
    small[:t0] = 0
    return big.to(torch.bfloat16), small.to(torch.bfloat16)
