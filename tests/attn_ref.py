"""fp64 reference of the training attention (causal GQA, one key window [ks, ke) per row), its analytic backward, a per-element
error bound for the bf16-in / fp32-accumulate kernels, and seeded input families in which the mask edges decide an O(1) share of
the result.  causal=False gives the bidirectional encoder attention (every query of a row sees the whole window; the rows past
kv_end are pad queries and still get a result).  Test infrastructure: torch only, runs on CPU or GPU; oracle/ is not involved.

Layouts: q, do [B, L, Hq, D]; k, v [B, L, Hkv, D]; lse [B, Hq, L].  The shared-prefix layout ([U * Lp prefix rows | U * G suffixes])
is checked through its dense equivalent: expand_shared() builds the [U * G, Lp + Ls] rows, fold_shared() maps dense results back
(prefix dK / dV summed over the G rows of a group, prefix O / lse taken from row g = 0).

Error model (every bound is SAFETY times the derived value; u = bf16 unit roundoff, w = a deliberately loose model of one fp32
tensor-core accumulation, relative to the sum of |terms|; a_i = max over visible j of scale * sum_d |q_id| |k_jd|):
  O     |dO_id|   <= (2u + 2w a_i) (P|V|)_id          P rounded to bf16 before P V, the bf16 output, score (and normaliser) error
  lse   |dlse_i|  <= 2w a_i + 1e-5
  dV    |ddV_jd|  <= sum_i P_ij (2u + 2w a_i) |dO_id|  summed over the q heads of the KV group
  dQ    |ddQ_id|  <= scale sum_j W_ij |K_jd|,  dK: scale sum_i W_ij |Q_id| (summed over the group), with
        W_ij = P_ij (2u |dP_ij - delta_i| + Edelta_i + w sum_d |dO_id| |V_jd| + 2w a_i |dP_ij - delta_i|)
        Edelta_i: the error delta = rowsum(dO o O) picks up from the O the backward reads (the kernel's own bf16 O when given).
Outputs that must be exactly 0 get a bound of exactly 0: O / dQ rows with no visible key, dK / dV rows of keys outside the window.
"""
import math

import torch

U_BF16 = 2.0 ** -8
W_ACC = 2.0 ** -16
SAFETY = 2.0
LSE_FLOOR = 1e-5
BN = 64                      # key tile of the kernels (the online-softmax variant below walks the same tiles)
FAR = 300.0                  # magnitude of the k / v rows outside the window in the adversarial families

# one typical kernel bug each; attn_ref(variant=...) computes attention as a kernel carrying it would
VARIANTS = ("diag_strict", "diag_plus_1", "ks_minus_1", "ke_included", "head_mod", "no_rescale")
# the same for the bidirectional (causal=False) kernel; tail_tile_unmasked: the keys from ke to the end of the 64-key tile that holds
# ke - 1 (the last tile the kernel loads) are left visible
NONCAUSAL_VARIANTS = ("causal_applied", "ke_included", "ks_minus_1", "tail_tile_unmasked", "no_rescale")


def visible(L, ks, ke, device, variant=None, causal=True):
    """[L, L] bool: query i sees key j."""
    i = torch.arange(L, device=device)[:, None]
    j = torch.arange(L, device=device)[None, :]
    lo = ks - 1 if variant == "ks_minus_1" and ks > 0 else ks
    hi = ke + 1 if variant == "ke_included" and ke < L else ke
    if variant == "tail_tile_unmasked":
        hi = min(L, -(-ke // BN) * BN)
    if causal:
        diag = (j < i) if variant == "diag_strict" else (j <= i + 1) if variant == "diag_plus_1" else (j <= i)
    else:
        diag = (j <= i) if variant == "causal_applied" else torch.ones(L, L, dtype=torch.bool, device=device)
    return (j >= lo) & (j < hi) & diag


def _online_softmax_fwd(S, vis, vh, rescale):
    """Flash forward over 64-key tiles in fp64: running max, running sum, O accumulator; rescale=False skips the correction of
    l and O when the running max grows (the bug)."""
    G, L, _ = S.shape
    m = torch.full((G, L), -math.inf, dtype=S.dtype, device=S.device)
    l = torch.zeros(G, L, dtype=S.dtype, device=S.device)
    o = torch.zeros(G, L, vh.shape[-1], dtype=S.dtype, device=S.device)
    for t0 in range(0, L, BN):
        st = S[..., t0:t0 + BN].masked_fill(~vis[:, t0:t0 + BN], -math.inf)
        m_new = torch.maximum(m, st.amax(-1))
        fin = torch.isfinite(m_new)
        p = torch.where(fin[..., None], torch.exp(st - torch.where(fin, m_new, 0.0)[..., None]), 0.0)
        alpha = torch.where(torch.isfinite(m), torch.exp(m - torch.where(fin, m_new, 0.0)), 0.0)
        if not rescale:
            alpha = torch.where(torch.isfinite(m), torch.ones_like(alpha), alpha)
        l = l * alpha + p.sum(-1)
        o = o * alpha[..., None] + p @ vh[t0:t0 + BN]
        m = m_new
    has = l > 0
    o = o / torch.where(has, l, 1.0)[..., None]
    lse = torch.where(has, m + torch.log(torch.where(has, l, 1.0)), math.inf)
    return o, lse


def attn_ref(q, k, v, do, windows, *, scale=None, o_used=None, variant=None, bounds=True, causal=True):
    """Forward and analytic backward in float64 from the exact input values, plus the per-element bounds (see the module doc).

    windows: [(ks, ke)] per row.  o_used: the O the backward under test reads ([B, L, Hq, D]); it sets Edelta.  Without it Edelta
    is derived from the O bound.  variant: one of VARIANTS (the bounds are then meaningless; pass bounds=False), or "online": the
    correct forward computed tile by tile like the kernel (the baseline of "no_rescale").
    Returns a dict of float64 tensors: o, lse, dq, dk, dv and (bounds=True) b_o, b_lse, b_dq, b_dk, b_dv."""
    B, L, Hq, D = q.shape
    Hkv = k.shape[2]
    GQ = Hq // Hkv
    dev = q.device
    f64 = lambda t: t.to(torch.float64)
    q, k, v = f64(q), f64(k), f64(v)
    do = torch.zeros_like(q) if do is None else f64(do)
    o_used = None if o_used is None else f64(o_used)
    scale = D ** -0.5 if scale is None else scale
    u, w = U_BF16, W_ACC
    r = {n: torch.zeros(B, L, Hq, D, dtype=torch.float64, device=dev) for n in ("o", "dq")}
    r.update({n: torch.zeros(B, L, Hkv, D, dtype=torch.float64, device=dev) for n in ("dk", "dv")})
    r["lse"] = torch.zeros(B, Hq, L, dtype=torch.float64, device=dev)
    if bounds:
        r.update({"b_" + n: torch.zeros_like(r[n]) for n in ("o", "dq", "dk", "dv", "lse")})
    kv_of = (lambda h: h % Hkv) if variant == "head_mod" else (lambda h: h // GQ)
    for b in range(B):
        ks, ke = (int(x) for x in windows[b])
        vis = visible(L, ks, ke, dev, variant, causal)
        for hk in range(Hkv):
            heads = [h for h in range(Hq) if kv_of(h) == hk]
            if not heads:
                continue
            qh, doh = q[b][:, heads].transpose(0, 1), do[b][:, heads].transpose(0, 1)       # [G, L, D]
            kh, vh = k[b, :, hk], v[b, :, hk]                                                # [L, D]
            S = scale * (qh @ kh.T)                                                          # [G, L, L]
            if variant in ("online", "no_rescale"):
                o, lse = _online_softmax_fwd(S, vis, vh, rescale=variant == "online")
            else:
                o = None
                Sm = S.masked_fill(~vis, -math.inf)
                mx = Sm.amax(-1)
                fin = torch.isfinite(mx)
                l = torch.exp(Sm - torch.where(fin, mx, 0.0)[..., None]).sum(-1)
                lse = torch.where(fin, torch.where(fin, mx, 0.0) + torch.log(torch.where(fin, l, 1.0)), math.inf)
                del Sm
            # the backward recomputes P from the forward's lse, as the kernels do
            fin = torch.isfinite(lse)
            P = torch.where(vis & fin[..., None], torch.exp(S - torch.where(fin, lse, 0.0)[..., None]), 0.0)
            if o is None:
                o = P @ vh
            delta = (o * doh).sum(-1)                                                        # [G, L]
            dP = doh @ vh.T
            dS = P * (dP - delta[..., None])
            r["o"][b][:, heads] = o.transpose(0, 1)
            r["lse"][b, heads] = lse
            r["dq"][b][:, heads] = (scale * (dS @ kh)).transpose(0, 1)
            r["dk"][b, :, hk] += scale * (dS.transpose(-1, -2) @ qh).sum(0)
            r["dv"][b, :, hk] += (P.transpose(-1, -2) @ doh).sum(0)
            if not bounds:
                continue
            a = (scale * (qh.abs() @ kh.abs().T)).masked_fill(~vis, 0.0).amax(-1)            # [G, L]
            eo = (2 * u + 2 * w * a)[..., None] * (P @ vh.abs())                             # O bound before the safety factor
            if o_used is not None:
                ou = o_used[b][:, heads].transpose(0, 1)
                edelta = ((ou - o) * doh).sum(-1).abs() + w * (ou.abs() * doh.abs()).sum(-1)
            else:
                edelta = (eo * doh.abs()).sum(-1) + w * (o.abs() * doh.abs()).sum(-1)
            ad = (dP - delta[..., None]).abs()
            W = P * (2 * u * ad + edelta[..., None] + w * (doh.abs() @ vh.abs().T) + 2 * w * a[..., None] * ad)
            r["b_o"][b][:, heads] = SAFETY * eo.transpose(0, 1)
            r["b_lse"][b, heads] = torch.where(fin, SAFETY * (2 * w * a + LSE_FLOOR), 0.0)
            r["b_dq"][b][:, heads] = (SAFETY * scale * (W @ kh.abs())).transpose(0, 1)
            r["b_dk"][b, :, hk] += SAFETY * scale * (W.transpose(-1, -2) @ qh.abs()).sum(0)
            r["b_dv"][b, :, hk] += SAFETY * ((P * (2 * u + 2 * w * a)[..., None]).transpose(-1, -2) @ doh.abs()).sum(0)
            del S, P, dP, dS, W, ad
    return r


def worst_ratio(got, ref, bound):
    """max |got - ref| / bound (float64).  Where bound == 0 the values must be equal (0 / inf otherwise); NaN counts as inf."""
    got, ref, bound = got.to(torch.float64), ref.to(torch.float64), bound.to(torch.float64)
    eq = got == ref                                                  # also inf == inf
    diff = torch.where(eq, torch.zeros_like(got), (got - ref).abs())
    ratio = torch.where(bound > 0, diff / torch.where(bound > 0, bound, 1.0), torch.where(diff > 0, math.inf, 0.0))
    ratio = torch.where(torch.isnan(ratio), math.inf, ratio)
    return ratio.max().item() if ratio.numel() else 0.0


# ------------------------------------------------------------------------------------------------------- shared-prefix layout
def expand_shared(buf, U, G, Lp, Ls):
    """[U * Lp + U * G * Ls, ...] -> [U * G, Lp + Ls, ...]: row r = [prefix of group r // G | suffix r]."""
    R = U * G
    pre = buf[:U * Lp].reshape(U, Lp, *buf.shape[1:])
    suf = buf[U * Lp:].reshape(R, Ls, *buf.shape[1:])
    return torch.cat([pre.repeat_interleave(G, 0), suf], 1)


def fold_shared(t, U, G, Lp, Ls, prefix="sum"):
    """[U * G, Lp + Ls, ...] -> [U * Lp + U * G * Ls, ...]; the prefix of a group is the sum of its G rows (gradients, bounds)
    or the value of row g = 0 (prefix="first": O, which every row of the group computes identically)."""
    R = U * G
    pre = t[:, :Lp].reshape(U, G, Lp, *t.shape[2:])
    pre = pre.sum(1) if prefix == "sum" else pre[:, 0]
    return torch.cat([pre.reshape(U * Lp, *t.shape[2:]), t[:, Lp:].reshape(R * Ls, *t.shape[2:])])


# ------------------------------------------------------------------------------------------------------------- input families
def make_inputs(family, B, L, Hq, Hkv, windows, *, D=128, seed=0, device="cpu", group=None, causal=True):
    """Seeded bf16 q, k, v, do on `device` (drawn on the CPU, so every device sees the same values).

    random    : N(0, 0.7^2) q / k / v, N(0, 1) dO.
    decoy     : token i has a unit direction u_i per KV head, shared by the q heads of the group (q_i = c_h sqrt(D) u_i, c_h in
                [0.8, 1.2] per head); k_j = 11 u_j + 17 u_{j-1}, so the diagonal is the largest visible score (~11) and the key just
                past it a larger, masked decoy (~17).
    first_key : every query shares a direction e per KV head; k at ks = e scaled to a score of ~12, so the maximum sits in the
                first key tile and the later tiles must leave it alone.
    window_decoy (for causal=False): every query shares a direction e per KV head as in first_key, the key at ke - 1 is e scaled to a
                score of ~12 (the maximum sits in the last key tile, so every earlier tile must be rescaled), and every key outside
                the window is +300 e: any key that leaks through the mask takes every query row.
    In decoy and first_key the k / v rows outside the window are +-300 (finite: a leaked key takes the whole row), and the rows at
    ks - 1 and ke (where they exist) are explicit decoys: 300 * sign of the query at ks (resp. ke), the first query that would
    see them through an off-by-one (with causal=False every query sees them: both use the query at ks).
    group=(G, Lp): rows b of one group b // G share positions [0, Lp) (the shared-prefix layout's dense equivalent)."""
    gen = torch.Generator().manual_seed(seed)
    GQ = Hq // Hkv
    scale = D ** -0.5

    def row(ks, ke):
        if family == "random":
            return (torch.randn(L, Hq, D, generator=gen) * 0.7, torch.randn(L, Hkv, D, generator=gen) * 0.7,
                    torch.randn(L, Hkv, D, generator=gen) * 0.7)
        if family == "decoy":
            ud = torch.randn(L, Hkv, D, generator=gen)
            ud = ud / ud.norm(dim=-1, keepdim=True)
            ch = torch.tensor([0.8 + 0.4 * g / max(GQ - 1, 1) for g in range(GQ)] * Hkv)
            qr = ch[None, :, None] * math.sqrt(D) * ud.repeat_interleave(GQ, 1)
            kr = 11.0 * ud
            kr[1:] += 17.0 * ud[:-1]
        elif family in ("first_key", "window_decoy"):
            e = torch.randn(Hkv, D, generator=gen)
            e = e / e.norm(dim=-1, keepdim=True)
            t = 0.7 * math.sqrt(D)
            qr = torch.randn(L, Hq, D, generator=gen) * 0.7 + t * e.repeat_interleave(GQ, 0)[None]
            kr = torch.randn(L, Hkv, D, generator=gen) * 0.7
            if ks < ke:
                kr[ks if family == "first_key" else ke - 1] = (12.0 / (scale * t)) * e
        else:
            raise ValueError(family)
        vr = torch.randn(L, Hkv, D, generator=gen) * 0.7
        out = torch.ones(L, dtype=torch.bool)
        out[ks:ke] = False
        n_out = int(out.sum())
        kr[out] = FAR * torch.randn(n_out, Hkv, D, generator=gen).sign()
        vr[out] = FAR * torch.randn(n_out, Hkv, D, generator=gen).sign()
        if family == "window_decoy":
            kr[out] = FAR * e
            return qr, kr, vr
        for jd, iq in ((ks - 1, ks), (ke, ke if causal else ks)):
            if 0 <= jd < L and iq < L:
                kr[jd] = FAR * qr[iq, ::GQ].sign()
        return qr, kr, vr

    qs, ks_, vs = [], [], []
    for b in range(B):
        qr, kr, vr = row(*windows[b])
        if group is not None and b % group[0]:
            G, Lp = group
            b0 = b - b % G
            assert windows[b][0] == windows[b0][0] and windows[b][1] >= Lp, "rows of a group share kv_start and see the whole prefix"
            qr[:Lp], kr[:Lp], vr[:Lp] = qs[b0][:Lp], ks_[b0][:Lp], vs[b0][:Lp]
        qs.append(qr); ks_.append(kr); vs.append(vr)
    bf = lambda xs: torch.stack(xs).to(torch.bfloat16).to(device)
    do = torch.randn(B, L, Hq, D, generator=gen).to(torch.bfloat16).to(device)
    return bf(qs), bf(ks_), bf(vs), do
