"""fp64 references of the rollout's decode step -- the skinny GEMM of decode_gemm_tc5.cu (bf16 or dequantized FP8 weights, with the
folded RMSNorm and its sum-of-squares partials), the q/k RMSNorm + RoPE of qk_rope_ mode 0 and of the fused decode attention, and the
fused paged attention of decode_attn_fused.cu (append, shared-prefix and private split passes, slot merge) -- with a per-element
error bound, seeded input families in which the page edges, the newest slot and the rotary position decide an O(1) share of the
result, and one-bug variants.  Test infrastructure: torch only, runs on CPU or GPU; oracle/ is not involved.

Every reference is computed in float64 from the exact bf16 (or fp32) input values the kernel received.

Error model.  u = U_BF16, e = 2^-24 (fp32 unit roundoff), w = W_ACC (attn_ref.py: a loose model of one fp32 tensor-core accumulation
relative to the sum of |terms|), E(x) = 2^-21 + 2^-23 |x| (gemm_ref.exp_err: __expf).  Bounds of the GEMM are the values derived below;
every other bound is SAFETY times the derived value.
  GEMM acc     tb = (w S + 2^-20 |acc|) rs       S = sum_k |x_k w_k|, rs = the row's rstd (1 without the norm): fp32 accumulation, the
               fp32 rstd (sum of fp32 partials, rsqrtf) and the products with it
  GEMM out     mode 3: tb;  mode 0: tb + u |v| + u tb;  mode 1: tb + u |v| + u |y| + 2u tb (v rounded to bf16, + residual, rounded);
               mode 2: 1.1 dg (|U| + du) + |silu G| du + 2u (|silu G| + 1.1 dg)(|U| + du) + 1e-6 |silu G| |U|,  dg = tb_G + u |G|,
               du = tb_U + u |U| (gate / up rounded to bf16, |silu'| <= 1.1, silu and the product rounded)
  sumsq_out    SAFETY (5 e Sq + 32 2^-149)          Sq = sum of the 32 squares of the kernel's own bf16 outputs of one warp: the
               squares of bf16 values are exact in fp32, the 5-level warp tree rounds each partial sum once
  embed sumsq  SAFETY (d / 32 + 5) e Sq + 2^-140     (each lane sums its d / 32 exact squares in order, then the 5-level warp tree)
  q/k prep     0 for every element none of whose rounding inputs is at risk; else 3 ulp_bf16(max(|p1|, |p2|, |y|)).  HF's rounding
               points are emulated in float64: t = bf16(x rstd), a = bf16(g t), p1 = bf16(a cos), p2 = bf16(-b sin) (resp. b cos,
               a sin), y = bf16(p1 + p2), with rstd in float64 and cos / sin from the kernel's own table (exact inputs).  The kernel's
               rstd is fp32 (shuffle-order sum of squares, rsqrtf), relative error < 2^-21, so x rstd can round the other way when it
               lies within that of a rounding boundary (a midpoint between bf16 neighbours).  The later rounding inputs are no risk of their
               own: a product of two bf16 values is exact in fp32 (and often lands exactly ON a midpoint, a tie both sides break to
               even), and p1 + p2 is formed in fp32 and rounded to bf16 by the kernel and the reference alike.  So an element is at risk
               when x rstd of either half of its rotary pair lies within a relative 2^-20 of a midpoint.  One flipped ulp of t moves a
               and each product by at most an ulp, so p1 + p2 moves by up to two ulps of the larger product, and the final rounding
               can add one ulp of y: 3 ulps (2 ulps was measured to be reached exactly on the H100).
  attention O  SAFETY ((2u + 2w a)(P|V|) + Eq + Em + u |O|)
               (2u + 2w a)(P|V|): attn_ref's O bound (P rounded to bf16 before P V, score and normaliser error), a = max over visible j
               of scale sum_d |q_d| |k_jd|;
               Eq = sum_j P_j |ds_j - <ds>| |V_j| <= P(ds |V|) + <ds> (P|V|), ds_j = scale sum_d dq_d |k_jd|, <ds> = sum_j P_j ds_j: the
               first-order effect of the q allowance dq (the at-risk elements of the query prep) on the scores;
               Em: the merge.  Slot j (one split of one pass) hands over o_j = O_j / l_j (fp32 divide: e) and lse_j = m_j ln2 + log l_j
               (fp32: 2 ulp32(lse_j) absolute); its weight is __expf(lse_j - mx) / sum, so it carries a relative error
               d_j = E(lse_j - mx) + 2 ulp32(lse_j) + 2 ulp32(mx) + 2e, and after the normalisation d_j + <d> (<d> = sum_k W_k d_k,
               W_k the exact slot weights).  The weighted sum of <= 32 slots adds (n_slots + 1) e relative to sum_j W_j |o_j|.  With
               W_j |o_j| <= (P|V|)_slot j:  Em = sum_j (d_j + <d>)(P|V|)_j + (n_slots + 2) e (P|V|);
               u |O|: the bf16 output.
Outputs that must be exact (appended V, kv_write_pages, gathered rows, scale_columns_) are checked bit for bit by the tests.
"""
import math

import torch

from attn_ref import SAFETY, U_BF16, W_ACC, worst_ratio  # noqa: F401  (worst_ratio: re-exported for the tests)
from gemm_ref import E32, exp_err, ulp32

PAGE = 64
BM, BK = 128, 64               # skinny GEMM: feature tile, k block
E_RS = 2.0 ** -20              # the fp32 rstd and the products with it (relative)
RISK = 2.0 ** -20              # relative distance to a bf16 rounding boundary below which a rounding may flip
FAR = 300.0

SKINNY_VARIANTS = ("no_last_kblock", "drop_contributor", "rstd_short", "rstd_over_n", "gate_up_swapped")
ATTN_VARIANTS = ("no_new", "stale_plus1", "rope_prev", "private_from_0", "skip_shared", "drop_last_slot", "head_mod", "group_row0_q",
                 "before_append")
FAMILIES = ("random", "decoy", "newest_wins", "rope_probe", "shared_edge")
# the family on which each attention variant is exposed (the case must also have the structure it needs: shared pages, G > 1, ...)
EXPOSED_BY = {"no_new": "newest_wins", "stale_plus1": "decoy", "rope_prev": "rope_probe", "private_from_0": "shared_edge",
              "skip_shared": "shared_edge", "drop_last_slot": "newest_wins", "head_mod": "newest_wins", "group_row0_q": "newest_wins",
              "before_append": "newest_wins"}


def _f64(t):
    return None if t is None else t.to(torch.float64)


def bf16(x):
    """Round to bf16 (through fp32, as the kernels do) and return float64."""
    return x.to(torch.float32).to(torch.bfloat16).to(torch.float64)


def ulp_bf16(x):
    """Spacing of the bf16 values at |x| (float64; 0 where x == 0)."""
    m, e = torch.frexp(x.to(torch.float64).abs())
    return torch.where(x != 0, torch.ldexp(torch.ones_like(m), (e - 8).to(torch.int64)), torch.zeros_like(m))


def near_boundary(x):
    """x (float64) lies within a relative RISK of a bf16 rounding boundary (a midpoint between two bf16 neighbours)."""
    m, _ = torch.frexp(x.to(torch.float64).abs())
    s = m * 256.0                                                    # in [128, 256): the bf16 mantissa and the rounded-off bits
    frac = s - torch.floor(s)
    return (x != 0) & ((frac - 0.5).abs() < RISK * s)


# ------------------------------------------------------------------------------------------------------------------- skinny GEMM
def streamk_plan(N, K, n_sms):
    """(chunk, KB): the units (tile * KB + k block) CTA c owns are [c chunk, (c + 1) chunk) -- br_skinny_gemm's host rule."""
    tiles, KB = -(-N // BM), -(-K // BK)
    units = tiles * KB
    grid = min(units, n_sms)
    return -(-units // grid), KB


def skinny_ref(x, w, mode, residual=None, sumsq_in=None, sumsq_in_n=1, eps=1e-6, *, variant=None, n_sms=132):
    """out = epilogue(rs (x w^T)) as br_skinny_gemm computes it, in float64 (see the module doc), with its bound.

    x [R, K], w [N, K] (bf16, or the dequantized FP8 weights in any float type), residual [R, N] (mode 1), sumsq_in [>= n, >= R] fp32
    partial sums of squares of the row (n = sumsq_in_n; rs = 1 / sqrt(sum / K + eps)).  variant: one of SKINNY_VARIANTS (n_sms sets the
    stream-K chunks of drop_contributor).  Returns (ref, bound), float64 [R, N] (mode 2: [R, N / 2])."""
    x, w = _f64(x), _f64(w)
    R, K = x.shape
    N = w.shape[0]
    dev = x.device
    xk, wk = x, w
    if variant == "no_last_kblock":
        kk = ((K - 1) // BK) * BK
        xk, wk = x[:, :kk], w[:, :kk]
    acc = xk @ wk.T
    if variant == "drop_contributor":                               # the last CTA of every tile that spans several loses its k blocks
        chunk, KB = streamk_plan(N, K, n_sms)
        for t in range(-(-N // BM)):
            first_c, last_c = (t * KB) // chunk, ((t + 1) * KB - 1) // chunk
            if last_c > first_c:
                k0 = (last_c * chunk - t * KB) * BK
                f = slice(t * BM, min(N, (t + 1) * BM))
                acc[:, f] -= x[:, k0:] @ w[f, k0:].T
    terms = x.abs() @ w.abs().T
    rs = torch.ones(R, 1, dtype=torch.float64, device=dev)
    if sumsq_in is not None:
        n = sumsq_in_n - 1 if variant == "rstd_short" else sumsq_in_n
        ss = _f64(sumsq_in[:n, :R]).to(dev).sum(0)
        rs_ref = 1.0 / torch.sqrt(_f64(sumsq_in[:sumsq_in_n, :R]).to(dev).sum(0) / K + eps)
        div = N if variant == "rstd_over_n" else K
        rs = (1.0 / torch.sqrt(ss / div + eps))[:, None]
        rs_b = rs_ref[:, None]
    else:
        rs_b = rs
    v = acc * rs
    v_true = (acc if variant is None else x @ w.T) * rs_b          # the bound is that of the correct result
    tb = (W_ACC * terms + E_RS * (x @ w.T).abs()) * rs_b
    u = U_BF16
    if mode == 3:
        return v, tb
    if mode == 0:
        return v, tb + u * v_true.abs() + u * tb
    if mode == 1:
        res = _f64(residual).to(dev)
        return v + res, tb + u * v_true.abs() + u * (v_true + res).abs() + 2 * u * tb
    vg = v.view(R, N // 16, 2, 8)
    G, U = (vg[:, :, 1], vg[:, :, 0]) if variant == "gate_up_swapped" else (vg[:, :, 0], vg[:, :, 1])
    vt = v_true.view(R, N // 16, 2, 8)
    eg, eu = tb.view(R, N // 16, 2, 8)[:, :, 0], tb.view(R, N // 16, 2, 8)[:, :, 1]
    silu = G * torch.sigmoid(G)
    ref = (silu * U).reshape(R, N // 2)
    Gt, Ut = vt[:, :, 0], vt[:, :, 1]
    st = Gt * torch.sigmoid(Gt)
    dg, du = eg + u * Gt.abs(), eu + u * Ut.abs()
    bound = 1.1 * dg * (Ut.abs() + du) + st.abs() * du + 2 * u * (st.abs() + 1.1 * dg) * (Ut.abs() + du) + 1e-6 * st.abs() * Ut.abs()
    return ref, bound.reshape(R, N // 2)


def sumsq_out_ref(out_bf16, N):
    """The sumsq_out partials [(tile 4 + warp), r] from the kernel's own bf16 outputs [R, >= N], with their bound (module doc).
    Feature columns past N count 0 (the kernel writes a 0 partial for a warp with no live feature)."""
    y = _f64(out_bf16[:, :N])
    R = y.shape[0]
    tiles = -(-N // BM)
    sq = torch.zeros(R, tiles * BM, dtype=torch.float64, device=y.device)
    sq[:, :N] = y * y
    ref = sq.view(R, tiles * 4, 32).sum(2).T.contiguous()
    return ref, SAFETY * (5 * E32 * ref + 32 * 2.0 ** -149)


# --------------------------------------------------------------------------------------------------------------- q/k norm + RoPE
def rope_table_ref(n_pos, D, theta):
    """A stand-in for br_rope_table on the CPU (fp32 angle, cos / sin rounded to bf16).  The GPU tests use the kernel's own table."""
    j = torch.arange(D // 2, dtype=torch.float32)
    inv = 1.0 / torch.pow(torch.tensor(theta, dtype=torch.float32), (2 * j) / D)
    ang = (torch.arange(n_pos, dtype=torch.float32)[:, None] * inv[None]).to(torch.float64)
    return torch.stack([bf16(torch.cos(ang)), bf16(torch.sin(ang))], -1).to(torch.float32)


def qk_prep_ref(raw, norm_w, pos, rope, eps):
    """y = RoPE(bf16(g * bf16(x * rstd))) at HF's rounding points (module doc), per head vector of raw [M, H, D].

    norm_w [D] bf16, pos [M] ints (clamped to the table like the fused kernel), rope [n_pos, D / 2, 2] fp32 (cos, sin).
    Returns (y [M, H, D] float64 (bf16 values), allow [M, H, D] float64 (0 where no rounding is at risk), risk bool [M, H, D])."""
    x = _f64(raw)
    M, H, D = x.shape
    h = D // 2
    dev = x.device
    g = _f64(norm_w).to(dev)
    p = pos.to(dev, torch.int64).clamp(0, rope.shape[0] - 1)
    cs = _f64(rope.to(dev)[p])                                       # [M, D/2, 2]
    c, s = cs[..., 0][:, None], cs[..., 1][:, None]
    rstd = 1.0 / torch.sqrt((x * x).mean(-1, keepdim=True) + eps)
    xr = x * rstd
    t = bf16(xr)
    a_ = bf16(g * t)
    a, b = a_[..., :h], a_[..., h:]
    p1, p2, p3, p4 = bf16(a * c), bf16(-b * s), bf16(b * c), bf16(a * s)
    y = torch.cat([bf16(p1 + p2), bf16(p3 + p4)], -1)
    nt = near_boundary(xr)                                           # the only rounding input the kernel does not compute exactly
    pair = nt[..., :h] | nt[..., h:]
    risk = torch.cat([pair, pair], -1)
    big = torch.cat([torch.maximum(p1.abs(), p2.abs()), torch.maximum(p3.abs(), p4.abs())], -1)
    big = torch.maximum(big, y.abs())
    allow = torch.where(risk, 3 * ulp_bf16(big), torch.zeros_like(big))
    return y, allow, risk


# ----------------------------------------------------------------------------------------------------------- fused decode attention
def decode_slots(n_shared, SS, SP):
    """(n_sh, SS) as the kernel sees them: the shared pass runs only with n_shared > 0 and SS > 0."""
    return (n_shared, SS) if n_shared > 0 and SS > 0 else (0, 0)


def key_slot(j, n_sh, SS, SP):
    """Merge slot of key position j: shared split (page % SS) for the first n_sh pages, SS + private split after them."""
    pg = j // PAGE
    return torch.where(pg < n_sh, pg % max(SS, 1), SS + (pg - n_sh) % SP)


def decode_step_ref(qkv, Hq, Hkv, qw, kw, kc0, vc0, table, cur, G, n_shared, SS, SP, rope, eps, *, D=128, scale=None, variant=None,
                    bounds=True, rows=None):
    """One decode step of br_decode_attn_fused in float64: the q/k prep of the raw projection qkv [R, >= (Hq + 2 Hkv) D], the append of
    the new K / V at position T = cur[r] of each row, and attention of each query over keys [0, T] through the page table.

    kc0 / vc0: the caches before the step [n_pages, Hkv, 64, D]; table [R, max_pages]; rope: the cos / sin table.  rows: the rows to
    compute (default all).  variant: one of ATTN_VARIANTS (compare against the bound of the correct reference).
    Returns a dict: o [R, Hq D], b_o (bounds=True), k_new / k_allow [R, Hkv, D] (the appended K and its allowance), v_new [R, Hkv, D]."""
    R = qkv.shape[0]
    GQ = Hq // Hkv
    dev = qkv.device
    scale = D ** -0.5 if scale is None else scale
    cur = cur.to(dev, torch.int64)
    raw = qkv[:, :(Hq + 2 * Hkv) * D].reshape(R, Hq + 2 * Hkv, D)
    q, qa, _ = qk_prep_ref(raw[:, :Hq], qw, cur - 1 if variant == "rope_prev" else cur, rope, eps)
    if variant == "group_row0_q":
        q = q[(torch.arange(R, device=dev) // G) * G]
    kn, ka, _ = qk_prep_ref(raw[:, Hq:Hq + Hkv], kw, cur, rope, eps)
    vn = _f64(raw[:, Hq + Hkv:])
    n_sh, SSe = decode_slots(n_shared, SS, SP)
    n_slots = SSe + SP
    u, w = U_BF16, W_ACC
    out = {"o": torch.zeros(R, Hq, D, dtype=torch.float64, device=dev), "k_new": kn, "k_allow": ka, "v_new": vn}
    if bounds:
        out["b_o"] = torch.zeros_like(out["o"])
    kv_of = (lambda hh: hh % Hkv) if variant == "head_mod" else (lambda hh: hh // GQ)
    table = table.to(dev, torch.int64)
    for r in (range(R) if rows is None else rows):
        T = int(cur[r])
        n_keys = T + 2 if variant == "stale_plus1" else T + 1
        j = torch.arange(n_keys, device=dev)
        pg = table[r, j // PAGE]
        sl = j % PAGE
        K = _f64(kc0.to(dev)[pg, :, sl])                             # [n, Hkv, D]
        V = _f64(vc0.to(dev)[pg, :, sl])
        if variant != "before_append":
            K[T], V[T] = kn[r], vn[r]
        mult = torch.ones(n_keys, dtype=torch.float64, device=dev)  # how often the kernel counts each key
        if variant == "no_new":
            mult[T] = 0
        elif variant == "private_from_0" and n_sh:
            mult[j < n_sh * PAGE] = 2
        elif variant == "skip_shared" and n_sh:
            mult[j < n_sh * PAGE] = 0
        elif variant == "drop_last_slot":
            mult[key_slot(j, n_sh, SSe, SP) == n_slots - 1] = 0
        slot = key_slot(torch.arange(T + 1, device=dev), n_sh, SSe, SP)
        for hk in range(Hkv):
            heads = [hh for hh in range(Hq) if kv_of(hh) == hk]
            if not heads:
                continue
            qh = q[r, heads]                                           # [g, D]
            Kh, Vh = K[:, hk], V[:, hk]
            S = scale * (qh @ Kh.T)                                    # [g, n]
            Sm = torch.where(mult > 0, S + torch.log(mult.clamp(min=1e-300)), -math.inf)
            P = torch.nan_to_num(torch.softmax(Sm, -1))                 # no key left (a variant): the kernel's merge writes 0
            out["o"][r, heads] = P @ Vh
            if not bounds:
                continue
            # bounds: the correct step (keys [0, T], each once)
            St, Pt = S[:, :T + 1], torch.softmax(S[:, :T + 1], -1)
            Ka, Va = Kh[:T + 1].abs(), Vh[:T + 1].abs()
            PV = Pt @ Va                                               # [g, D]
            a = (scale * (qh.abs() @ Ka.T)).amax(-1)                   # [g]
            eo = (2 * u + 2 * w * a)[:, None] * PV
            ds = scale * (qa[r, heads] @ Ka.T)                         # [g, n]
            dsm = (Pt * ds).sum(-1, keepdim=True)
            eq = (Pt * ds) @ Va + dsm * PV
            lse_s = torch.full((len(heads), n_slots), -math.inf, dtype=torch.float64, device=dev)
            PV_s = torch.zeros(len(heads), n_slots, D, dtype=torch.float64, device=dev)
            for sidx in range(n_slots):
                m = slot == sidx
                if m.any():
                    lse_s[:, sidx] = torch.logsumexp(St[:, m], -1)
                    PV_s[:, sidx] = Pt[:, m] @ Va[m]
            mx = lse_s.amax(-1, keepdim=True)
            Ws = torch.exp(lse_s - mx)
            Ws = Ws / Ws.sum(-1, keepdim=True)
            fin = torch.isfinite(lse_s)
            lf = torch.where(fin, lse_s, mx)
            dj = exp_err(lf - mx) + 2 * ulp32(lf) + 2 * ulp32(mx.expand_as(lf)) + 2 * E32
            dj = torch.where(fin, dj, torch.zeros_like(dj))
            dbar = (Ws * dj).sum(-1, keepdim=True)
            em = ((dj + dbar)[..., None] * PV_s).sum(1) + (n_slots + 2) * E32 * PV
            o_true = Pt @ Vh[:T + 1]
            out["b_o"][r, heads] = SAFETY * (eo + eq + em + u * o_true.abs())
    out["o"] = out["o"].reshape(R, Hq * D)
    if bounds:
        out["b_o"] = out["b_o"].reshape(R, Hq * D)
    return out


# ------------------------------------------------------------------------------------------------------------------ input families
def page_layout(plen, G, cur, *, extra=3, seed=0):
    """A scattered page table for U = len(plen) groups of G rows: the first n_shared = min(plen) // 64 (G > 1) prompt pages are shared
    by a group, every row owns the pages after them up to the page of position cur[r].  Entries past a row's last page point at
    `extra` unreferenced decoy pages (never out of range).  Returns (table [R, max_pages] int32, n_pages, n_shared)."""
    U, R = len(plen), len(cur)
    n_shared = min(l // PAGE for l in plen) if G > 1 else 0
    need = [int(c) // PAGE + 1 for c in cur]
    priv = [n - n_shared for n in need]
    max_pages = max(need) + 1
    n_pages = U * n_shared + sum(priv) + extra
    perm = torch.randperm(n_pages, generator=torch.Generator().manual_seed(seed)).tolist()
    spare = perm[n_pages - extra:]
    table = torch.zeros(R, max_pages, dtype=torch.int32)
    nxt = 0
    for uu in range(U):
        sh = perm[nxt:nxt + n_shared]; nxt += n_shared
        for g in range(G):
            r = uu * G + g
            mine = perm[nxt:nxt + priv[r]]; nxt += priv[r]
            row = sh + mine
            row += [spare[i % extra] for i in range(max_pages - len(row))]
            table[r] = torch.tensor(row, dtype=torch.int32)
    return table, n_pages, n_shared


def make_decode_case(family, plen, G, cur, Hq, Hkv, rope, *, D=128, extra_width=0, seed=0, eps=1e-6):
    """Seeded bf16 inputs of one decode step (CPU tensors): dict(qkv [R, (Hq + 2 Hkv) D + extra_width] raw projection, qw, kw, kc, vc
    (caches before the step), table, cur (int32), n_shared).  plen[u]: prompt length of group u (its rows share its first
    plen // 64 pages' contents, and the rest of the prompt is copied into every row, as the rollout's tail copies do); cur[r] >= plen.

    random     : raw q / k / v ~ N(0, 1); cached K ~ N(0, 1), V ~ N(0, 1); slots past a row's position and unreached pages random too.
    decoy      : random, but every cache slot past cur[r] in the newest page and every slot of a page the row does not reach holds
                 K = 30 sign(q-hat of the first q head of its kv head group) (a score far above every visible key) and V = +-300.
    newest_wins: random with cached K scaled by 0.5; the raw k of the new token equals the raw q of the group's first q head, so after
                 norm + RoPE at the same position it outscores every cached key (score ~ scale |q-hat|^2 ~ 11); the stale slot at cur[r]
                 holds -k-hat and -v (reading the page before the append gives an O(1) error).
    rope_probe : q and k put their energy in the highest-frequency rotary pair (dims 0 and 64, inv_freq = 1); cached keys point in
                 random directions of that pair with |k| = 3, so a query roped one position off turns every score by 1 rad.
    shared_edge: random with the raw q of a group's rows equal, plus one dominant key (score ~ 25 above the rest) in BOTH the last
                 slot of the last shared page and the first slot of the first private page (the same K, different V): the two edges
                 split the attention evenly."""
    gen = torch.Generator().manual_seed(seed)
    R, U = len(cur), len(plen)
    assert R == U * G and all(int(cur[r]) >= plen[r // G] for r in range(R))
    GQ = Hq // Hkv
    table, n_pages, n_shared = page_layout(plen, G, cur, seed=seed)
    width = (Hq + 2 * Hkv) * D
    qkv = torch.randn(R, width + extra_width, generator=gen)
    qw = (1 + 0.1 * torch.randn(D, generator=gen)).to(torch.bfloat16)
    kw = (1 + 0.1 * torch.randn(D, generator=gen)).to(torch.bfloat16)
    kc = torch.randn(n_pages, Hkv, PAGE, D, generator=gen)
    vc = torch.randn(n_pages, Hkv, PAGE, D, generator=gen)
    curt = torch.tensor([int(c) for c in cur], dtype=torch.int32)
    if family == "rope_probe":
        qkv[:, :width] *= 0.02
        ang = torch.rand(R, Hq + Hkv, generator=gen) * 2 * math.pi
        qkv[:, :(Hq + Hkv) * D].view(R, Hq + Hkv, D)[:, :, 0] = 4 * torch.cos(ang)
        qkv[:, :(Hq + Hkv) * D].view(R, Hq + Hkv, D)[:, :, D // 2] = 4 * torch.sin(ang)
        kc *= 0.02
        phi = torch.rand(n_pages, Hkv, PAGE, generator=gen) * 2 * math.pi
        kc[..., 0], kc[..., D // 2] = 3 * torch.cos(phi), 3 * torch.sin(phi)
    elif family == "newest_wins":
        kc *= 0.5
        v3 = qkv[:, :(Hq + Hkv) * D].view(R, Hq + Hkv, D)
        v3[:, Hq:] = v3[:, 0:Hq:GQ]
    elif family == "shared_edge":                                    # one query per group: the dominant key wins in every row
        for uu in range(U):
            qkv[uu * G:(uu + 1) * G, :Hq * D] = qkv[uu * G, :Hq * D].clone()
    elif family not in ("random", "decoy"):
        raise ValueError(family)
    qkv = qkv.to(torch.bfloat16)
    kc, vc = kc.to(torch.bfloat16), vc.to(torch.bfloat16)
    # the prompt of a group is the same in every row: private prompt pages of rows g > 0 copy row 0's
    for uu in range(U):
        r0 = uu * G
        for g in range(1, G):
            for p in range(n_shared, -(-plen[uu] // PAGE)):
                kc[table[r0 + g, p]] = kc[table[r0, p]]
                vc[table[r0 + g, p]] = vc[table[r0, p]]
    raw = qkv[:, :width].reshape(R, Hq + 2 * Hkv, D)
    qh, _, _ = qk_prep_ref(raw[:, :Hq], qw, curt, rope, eps)
    kh, _, _ = qk_prep_ref(raw[:, Hq:Hq + Hkv], kw, curt, rope, eps)
    if family == "decoy":
        reached = set()
        for r in range(R):
            T = int(cur[r])
            reached |= {int(table[r, p]) for p in range(T // PAGE + 1)}
        for p in range(n_pages):
            if p not in reached:
                kc[p] = (30 * torch.sign(qh[0, 0:Hq:GQ]))[:, None].expand(Hkv, PAGE, D).to(torch.bfloat16)
                vc[p] = (FAR * torch.sign(torch.randn(Hkv, PAGE, D, generator=gen))).to(torch.bfloat16)
        for r in range(R):
            T = int(cur[r])
            p = int(table[r, T // PAGE])
            s0 = T % PAGE + 1
            if s0 < PAGE:
                kc[p, :, s0:] = (30 * torch.sign(qh[r, 0:Hq:GQ]))[:, None].expand(Hkv, PAGE - s0, D).to(torch.bfloat16)
                vc[p, :, s0:] = (FAR * torch.sign(torch.randn(Hkv, PAGE - s0, D, generator=gen))).to(torch.bfloat16)
    elif family == "newest_wins":
        for r in range(R):
            T = int(cur[r])
            p = int(table[r, T // PAGE])
            kc[p, :, T % PAGE] = (-kh[r]).to(torch.bfloat16)
            vc[p, :, T % PAGE] = (-raw[r, Hq + Hkv:].double()).to(torch.bfloat16)
    elif family == "shared_edge":
        for uu in range(U):
            r0 = uu * G
            kstar = (3 * torch.sign(qh[r0, 0:Hq:GQ])).to(torch.bfloat16)        # [Hkv, D]: score ~ scale 3 sum |q-hat| ~ 25
            edges = []
            if n_shared:
                edges.append((int(table[r0, n_shared - 1]), PAGE - 1, [r0]))
            for g in range(G):
                r = r0 + g
                if int(cur[r]) >= n_shared * PAGE:
                    edges.append((int(table[r, n_shared]), 0, [r]))
            for p, s, _ in edges:
                kc[p, :, s] = kstar
    return dict(qkv=qkv, qw=qw, kw=kw, kc=kc, vc=vc, table=table, cur=curt, n_shared=n_shared)
