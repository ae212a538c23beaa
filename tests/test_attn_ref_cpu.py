"""The fp64 attention reference and its error bound (tests/attn_ref.py), checked without a GPU: the reference equals torch autograd
in float64, and a reference carrying one typical kernel bug breaks the bound by >= 10x on the adversarial input families, so the
GPU tests built on it would catch that bug."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attn_ref as ar  # noqa: E402


def _autograd(q, k, v, do, windows):
    """Causal GQA attention with per-row windows through torch autograd in float64: (o, lse, dq, dk, dv)."""
    B, L, Hq, D = q.shape
    GQ = Hq // k.shape[2]
    qf, kf, vf = (t.to(torch.float64).clone().requires_grad_(True) for t in (q, k, v))
    qt = qf.transpose(1, 2)
    kt, vt = (t.transpose(1, 2).repeat_interleave(GQ, 1) for t in (kf, vf))
    vis = torch.stack([ar.visible(L, ks, ke, q.device) for ks, ke in windows])[:, None]
    s = (qt @ kt.transpose(-1, -2) * D ** -0.5).masked_fill(~vis, -math.inf)
    lse = torch.logsumexp(s, -1)
    p = torch.softmax(s, -1).nan_to_num(0.0)
    o = (p @ vt).transpose(1, 2)
    o.backward(do.to(torch.float64))
    lse = torch.where(torch.isfinite(lse), lse, math.inf).detach()
    return o.detach(), lse, qf.grad, kf.grad, vf.grad


def _close(a, b):
    torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("B,L,Hq,Hkv,windows", [
    (3, 9, 4, 1, [(0, 9), (2, 7), (0, 0)]),                   # GQA 4:1, an inner window, an empty window
    (2, 70, 4, 2, [(3, 66), (0, 70)]),                        # two 64-key tiles
    (2, 130, 8, 2, [(65, 130), (0, 0)]),                      # a window starting past a tile edge; every row masked
])
def test_reference_matches_autograd(B, L, Hq, Hkv, windows):
    q, k, v, do = ar.make_inputs("random", B, L, Hq, Hkv, windows, D=32, seed=L)
    r = ar.attn_ref(q, k, v, do, windows)
    o, lse, dq, dk, dv = _autograd(q, k, v, do, windows)
    for name, want in (("o", o), ("lse", lse), ("dq", dq), ("dk", dk), ("dv", dv)):
        _close(r[name], want)
    # the tiled (online-softmax) forward is the same computation
    r2 = ar.attn_ref(q, k, v, do, windows, variant="online", bounds=False)
    _close(r2["o"], o)
    _close(r2["lse"], lse)
    # exact zeros carry a zero bound: rows with no visible key, keys outside the window
    for b, (ks, ke) in enumerate(windows):
        no_key = torch.arange(L) < (ks if ks < ke else L)
        assert (r["b_o"][b][no_key] == 0).all() and (r["b_dq"][b][no_key] == 0).all()
        assert torch.isinf(r["lse"][b][:, no_key]).all()
        out = (torch.arange(L) < ks) | (torch.arange(L) >= ke)
        assert (r["b_dk"][b][out] == 0).all() and (r["b_dv"][b][out] == 0).all()
        assert (r["b_o"][b][~no_key] > 0).all() and (r["b_dv"][b][~out] > 0).all()


def test_shared_prefix_fold_matches_autograd():
    """expand_shared / fold_shared: the dense-equivalent reference folds to the gradients of the shared semantics (prefix rows are
    one leaf per group, seen by all G rows; prefix dO given once per group)."""
    U, G, Lp, Ls, Hq, Hkv, D = 2, 3, 64, 20, 4, 2, 32
    R, L = U * G, Lp + Ls
    windows = [(ks, ke) for ks, kes in ((5, (84, 70, 66)), (0, (84, 84, 77))) for ke in kes]
    q, k, v, do = ar.make_inputs("random", R, L, Hq, Hkv, windows, D=D, seed=3, group=(G, Lp))
    do = do.clone()
    do[torch.arange(R) % G != 0, :Lp] = 0
    r = ar.attn_ref(q, k, v, do, windows)
    # shared semantics through autograd: leaves on the shared buffer
    leaves = [ar.fold_shared(t, U, G, Lp, Ls, prefix="first").to(torch.float64).requires_grad_(True) for t in (q, k, v)]
    qd, kd, vd = (ar.expand_shared(t, U, G, Lp, Ls) for t in leaves)
    o, _, _, _, _ = _autograd(qd.detach(), kd.detach(), vd.detach(), do, windows)
    GQ = Hq // Hkv
    vis = torch.stack([ar.visible(L, ks, ke, "cpu") for ks, ke in windows])[:, None]
    s = (qd.transpose(1, 2) @ kd.transpose(1, 2).repeat_interleave(GQ, 1).transpose(-1, -2) * D ** -0.5).masked_fill(~vis, -math.inf)
    out = (torch.softmax(s, -1).nan_to_num(0.0) @ vd.transpose(1, 2).repeat_interleave(GQ, 1)).transpose(1, 2)
    out.backward(do.to(torch.float64))
    _close(ar.fold_shared(r["o"], U, G, Lp, Ls, prefix="first"), ar.fold_shared(o, U, G, Lp, Ls, prefix="first"))
    for name, leaf in zip(("dq", "dk", "dv"), leaves):
        _close(ar.fold_shared(r[name], U, G, Lp, Ls), leaf.grad)


# windows with a left edge off the tile grid, a post-EOS tail, and a full row (GQA 4:1 over two KV heads, five key tiles)
MUT_B, MUT_L, MUT_HQ, MUT_HKV = 3, 300, 8, 2
MUT_WINDOWS = [(37, 250), (0, 300), (70, 131)]


@pytest.fixture(scope="module", params=["decoy", "first_key"])
def family_ref(request):
    q, k, v, do = ar.make_inputs(request.param, MUT_B, MUT_L, MUT_HQ, MUT_HKV, MUT_WINDOWS, D=128, seed=7)
    return request.param, (q, k, v, do), ar.attn_ref(q, k, v, do, MUT_WINDOWS)


def _worst(r, m):
    return {n: ar.worst_ratio(m[n], r[n], r["b_" + n]) for n in ("o", "lse", "dq", "dk", "dv")}


def test_reference_is_within_its_own_bound(family_ref):
    """Sanity: the correct tiled forward (the kernel's algorithm in fp64) stays far inside the bound."""
    family, (q, k, v, do), r = family_ref
    m = ar.attn_ref(q, k, v, do, MUT_WINDOWS, variant="online", bounds=False)
    worst = _worst(r, m)
    assert max(worst.values()) < 1e-6, worst


@pytest.mark.parametrize("variant", ar.VARIANTS)
def test_mutants_break_the_bound(family_ref, variant):
    """Each one-bug variant exceeds the bound by >= 10x in at least one output.  On first_key the running maximum never grows after
    the first tile, so a skipped online-softmax rescale is invisible there by construction; decoy catches it."""
    family, (q, k, v, do), r = family_ref
    m = ar.attn_ref(q, k, v, do, MUT_WINDOWS, variant=variant, bounds=False)
    worst = _worst(r, m)
    print(f"{family} {variant}: " + " ".join(f"{n} {x:.3g}" for n, x in worst.items()))
    if family == "first_key" and variant == "no_rescale":
        assert max(worst.values()) < 1e-6
        return
    assert max(worst.values()) >= 10, worst
