"""The sampler's token draw against the float64 reference of sampler_ref.py, draw by draw: every draw not at risk equals the
reference token, an at-risk draw is one of the tokens beside the boundary it is at risk on.  All four entry points (single / two
stage, with / without the log-prob output) make the same draw, including on rows with more ties of the k-th value than a chunk or the
1024-value collection can hold.  Also: the bookkeeping (tokens, next_ids, finished, pad, step >= max_steps) bit for bit, strided
logits, br_decode_advance, the argument refusals, and the one-bug variants disagreeing with the kernel."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sampler_ref as sr  # noqa: E402

pytestmark = pytest.mark.gpu
SENTINEL = -7


@pytest.fixture(scope="module")
def ops():
    from bioreason_b200.build import ensure_built
    ensure_built()
    from bioreason_b200 import ops as o
    return o


ENTRIES = ("single", "single_logp", "two_stage", "two_stage_logp")


def run_entry(ops, z, entry, T, k, p, U, do_sample=True, finished=None, eos_id=-1, pad_id=0, steps=None, max_steps=None):
    """Tokens [R, max_steps] (sentinel where unwritten) and next_ids of the last call, from one entry point over steps."""
    R, V = z.shape
    S = U.shape[0]
    max_steps = S if max_steps is None else max_steps
    two, lp = entry.startswith("two"), entry.endswith("logp")
    ws = ops.sample_workspace(R, V, "cuda", logp=lp) if two else None
    tok = torch.full((R, max_steps), SENTINEL, device="cuda", dtype=torch.int64)
    nxt = torch.full((R,), SENTINEL, device="cuda", dtype=torch.int64)
    logp = torch.zeros(R, max_steps, device="cuda") if lp else None
    step = torch.zeros(1, device="cuda", dtype=torch.int32)
    fin = torch.zeros(R, device="cuda", dtype=torch.int32) if finished is None else finished
    for s in (range(S) if steps is None else steps):
        step.fill_(s)
        ops.sample_next(z, workspace=ws, temperature=T, top_k=k, top_p=p, do_sample=do_sample, uniforms=U if do_sample else None,
                        step=step, max_steps=max_steps, eos_id=eos_id, pad_id=pad_id, finished=fin, tokens=tok, next_ids=nxt, logp=logp)
    return tok.cpu(), nxt.cpu(), fin.cpu()


# (family, V, R, T, top_k, top_p, steps): a covering set of V x R x T x top_k x top_p; uniform_grid uses 32 rows x 64 steps
CASES = [
    ("uniform_grid", 1, 32, 0.6, 20, 0.95, 64), ("uniform_grid", 19, 32, 1.0, 20, 1.0, 64), ("uniform_grid", 20, 32, 1.5, 20, 0.5, 64),
    ("uniform_grid", 21, 32, 0.3, 20, 1.0, 64), ("uniform_grid", 1000, 32, 1.0, 33, 0.95, 64),
    ("uniform_grid", 1000, 32, 1.5, 1024, 1.0, 64), ("uniform_grid", 4095, 32, 0.6, 2, 1.0, 64),
    ("uniform_grid", 4096, 32, 1.0, 32, 0.5, 64), ("uniform_grid", 4097, 32, 1.5, 50, 0.95, 64),
    ("uniform_grid", 3 * 4096 + 1, 32, 0.6, 20, 0.95, 64), ("uniform_grid", 151936, 32, 0.6, 20, 0.95, 64),
    ("uniform_grid", 151936, 32, 1.0, 32, 1.0, 64), ("uniform_grid", 151936, 32, 1.5, 50, 0.5, 64),
    ("uniform_grid", 152000, 32, 0.3, 33, 1.0, 64), ("uniform_grid", 152000, 32, 1.0, 20, 0.95, 64),
    ("uniform_grid", 262144, 32, 0.6, 20, 1.0, 64), ("uniform_grid", 262145, 32, 1.0, 20, 0.95, 64),
    ("uniform_grid", 262145, 32, 1.5, 50, 1.0, 64), ("uniform_grid", 4097, 32, 1.0, 1, 1.0, 64),
    ("uniform_grid", 151936, 32, 1.0, 20, 1e-3, 64), ("uniform_grid", 12289, 32, 1.5, 32, 0.5, 64),
    ("uniform_grid", 152000, 32, 0.6, 2, 0.95, 64), ("uniform_grid", 4096, 32, 0.3, 1024, 0.95, 64),
    ("uniform_grid", 1000, 32, 0.6, 20, 0.5, 64), ("uniform_grid", 262144, 32, 1.5, 33, 0.95, 64),
    ("randn1", 151936, 8, 0.6, 20, 0.95, 8), ("randn1", 1000, 32, 1.0, 50, 1.0, 8), ("randn1", 262145, 8, 1.5, 20, 0.5, 8),
    ("randn3", 151936, 32, 0.6, 20, 0.95, 8), ("randn3", 4097, 8, 1.0, 32, 1e-3, 8), ("randn3", 21, 8, 0.3, 33, 0.95, 8),
    ("randn10", 151936, 8, 1.0, 20, 0.95, 8), ("randn10", 262145, 8, 0.6, 50, 1.0, 8), ("randn10", 12289, 32, 1.5, 2, 0.5, 8),
    ("randn30", 151936, 8, 0.6, 20, 0.95, 8), ("randn30", 262144, 8, 1.0, 32, 1.0, 8), ("randn30", 4096, 8, 1.5, 1024, 0.95, 8),
    ("peaked", 151936, 8, 1.5, 20, 0.95, 8), ("peaked", 1000, 8, 0.6, 50, 0.5, 8),
    ("flat_top", 151936, 8, 1.0, 20, 0.5, 8), ("flat_top", 152000, 8, 0.6, 50, 0.95, 8), ("flat_top", 4097, 8, 1.5, 32, 1e-3, 8),
    ("chunk_local", 151936, 8, 1.0, 20, 0.95, 8), ("chunk_local", 152000, 8, 0.6, 32, 1.0, 8),
    ("chunk_local", 262145, 8, 1.0, 50, 0.95, 8),
    ("fewer_finite_than_k", 151936, 12, 1.0, 20, 0.95, 8), ("fewer_finite_than_k", 1000, 12, 0.6, 50, 1.0, 8),
    ("fewer_finite_than_k", 262145, 12, 1.5, 32, 0.5, 8),
    ("tie_overflow_chunk", 151936, 8, 1.0, 20, 1.0, 8), ("tie_overflow_chunk", 1000, 8, 0.6, 20, 0.95, 8),
    ("tie_overflow_chunk", 262145, 8, 1.0, 32, 0.95, 8), ("tie_overflow_chunk", 152000, 8, 1.5, 50, 1.0, 8),
    ("tie_overflow_1024", 151936, 8, 1.0, 20, 1.0, 8), ("tie_overflow_1024", 262145, 8, 0.6, 20, 0.95, 8),
    ("tie_overflow_1024", 81920, 8, 1.0, 33, 1.0, 8),
]
STATS = {}


def _case_id(c):
    return f"{c[0]}-V{c[1]}-R{c[2]}-T{c[3]}-k{c[4]}-p{c[5]}"


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_draws_vs_fp64(ops, case):
    fam, V, R, T, k, p, S = case
    z = sr.make_logits(fam, R, V, seed=V + 7 * R + k)
    U = sr.grid_uniforms(S, R) if fam == "uniform_grid" else sr.distinct_uniforms(S, R, seed=V + k)
    zc, Uc = z.cuda(), U.cuda()
    entries = ENTRIES if k <= 32 else ENTRIES[:2]
    toks = {e: run_entry(ops, zc, e, T, k, p, Uc)[0] for e in entries}
    again = run_entry(ops, zc, entries[-1], T, k, p, Uc)[0]
    for e in entries:
        assert torch.equal(toks[e], toks["single"]), (e, "differs from the single-stage draw")
    assert torch.equal(again, toks[entries[-1]]), "repeated launch differs"
    got = toks["single"].numpy()
    rows = [sr.Row(z[0].numpy(), T, k, p)] * R if fam == "uniform_grid" else [sr.Row(z[r].numpy(), T, k, p) for r in range(R)]
    st = STATS.setdefault(fam, {"draws": 0, "at_risk": 0, "min_ratio_exact": math.inf, "min_topp_ratio": math.inf})
    for r in range(R):
        ref = rows[r].draw(U[:, r].numpy())
        ok = ~ref["at_risk"]
        assert np.array_equal(got[r][ok], ref["token"][ok]), (r, np.nonzero(got[r] != ref["token"])[0])
        assert (ref["allowed"] == got[r][:, None]).any(1).all(), r
        st["draws"] += S
        st["at_risk"] += int(ref["at_risk"].sum())
        if ok.any():
            st["min_ratio_exact"] = min(st["min_ratio_exact"], float(ref["ratio"][ok].min()))
        st["min_topp_ratio"] = min(st["min_topp_ratio"], rows[r].m_topp)
    # greedy: the largest logit, the smallest id among equal maxima
    want = torch.tensor([sr.greedy_ref(z[r].numpy()) for r in range(R)])
    for e in ENTRIES:
        g = run_entry(ops, zc, e, T, k, p, Uc[:1], do_sample=False)[0][:, 0]
        assert torch.equal(g, want), e


def test_draw_totals():
    """Runs after the draw cases: the per-family table (draws, at-risk draws, smallest margin / delta among exact draws)."""
    if not STATS:
        pytest.skip("no draw case ran")
    total = sum(s["draws"] for s in STATS.values())
    for fam, s in sorted(STATS.items()):
        print(f"{fam:22s} draws {s['draws']:6d}  at risk {s['at_risk']:4d}  min margin/delta (exact) {s['min_ratio_exact']:.3g}"
              f"  min top-p margin/delta {s['min_topp_ratio']:.3g}")
    print(f"total draws {total}")
    if len(STATS) == len(sr.FAMILIES):
        assert total >= 50000


def test_variants_disagree_with_the_kernel(ops):
    """On the kernel's own draws, each one-bug variant differs on at least one draw that is not at risk."""
    for variant, fam in sr.EXPOSED_BY.items():
        V = 151936
        R, S = 4, 16
        z = sr.make_logits(fam, R, V, seed=3)
        U = sr.grid_uniforms(S, R)
        n = 0
        for T, k, p in [(0.6, 20, 0.95), (1.0, 20, 1.0), (1.0, 20, 0.5)]:
            got = run_entry(ops, z.cuda(), "two_stage", T, k, p, U.cuda())[0].numpy()
            Uf = U.numpy().reshape(-1)
            for r in range(R):
                ref = sr.Row(z[r].numpy(), T, k, p).draw(U[:, r].numpy())
                uv = Uf[[sr.uniform_index(s, r, S, R, variant) for s in range(S)]]
                wrong = sr.Row(z[r].numpy(), T, k, p, variant=None if variant == "uniforms_row_major" else variant).draw(uv)
                n += int((~ref["at_risk"] & (wrong["token"] != got[r])).sum())
        assert n > 0, variant


# ------------------------------------------------------------------------------------------------------------------- bookkeeping
@pytest.mark.parametrize("entry", ENTRIES)
def test_bookkeeping_bit_exact(ops, entry):
    R, V, S = 8, 4097, 5
    z = sr.make_logits("randn3", R, V, seed=1)
    z[2, 77] = 60.0                                                    # row 2 samples EOS = 77 at every step
    U = sr.distinct_uniforms(S, R, seed=2)
    ref = [sr.Row(z[r].numpy(), 0.6, 20, 0.95) for r in range(R)]
    fin0 = torch.zeros(R, dtype=torch.int32)
    fin0[[1, 6]] = 1                                                   # already finished
    eos, pad = 77, 12345
    steps = [0, 1, 2, S - 1]                                           # ... and step = max_steps - 1
    tok, nxt, fin = run_entry(ops, z.cuda(), entry, 0.6, 20, 0.95, U.cuda(), finished=fin0.cuda(), eos_id=eos, pad_id=pad, steps=steps,
                              max_steps=S)
    want = torch.full((R, S), SENTINEL, dtype=torch.int64)
    for r in range(R):
        d = ref[r].draw(U[:, r].numpy())
        assert not d["at_risk"][steps].any()
        done = bool(fin0[r])
        for s in steps:
            want[r, s] = pad if done else int(d["token"][s])
            done = done or want[r, s].item() == eos
    assert torch.equal(tok, want) and torch.all(want[2, 1:][want[2, 1:] != SENTINEL] == pad)
    assert torch.equal(nxt, want[:, S - 1])
    assert fin.tolist() == [int(bool(fin0[r]) or bool((want[r] == eos).any())) for r in range(R)] and fin[2] == 1
    # step = max_steps: tokens untouched, next_ids still written
    Ub = torch.cat([U, U[:1] * 0.5])                                   # uniforms[S] for the step past the end
    tok3, nxt3, _ = run_entry(ops, z.cuda(), entry, 0.6, 20, 0.95, Ub.cuda(), steps=[S], max_steps=S)
    assert torch.all(tok3 == SENTINEL) and torch.equal(nxt3, torch.tensor([int(ref[r].draw(Ub[S:, r].numpy())["token"][0]) for r in range(R)]))


@pytest.mark.parametrize("entry", ENTRIES)
def test_strided_logits(ops, entry):
    """ld > V with huge finite values in the gap columns: a single read past V would change the draw."""
    R, V, S, gap = 8, 12289, 4, 37
    z = sr.make_logits("randn3", R, V, seed=4)
    buf = torch.full((R, V + gap), 1e30)
    buf[:, :V] = z
    U = sr.distinct_uniforms(S, R, seed=5)
    view = buf.cuda()[:, :V]
    tok = run_entry(ops, view, entry, 1.0, 20, 0.95, U.cuda())[0]
    assert torch.equal(tok, run_entry(ops, z.cuda(), entry, 1.0, 20, 0.95, U.cuda())[0])
    for r in range(R):
        d = sr.Row(z[r].numpy(), 1.0, 20, 0.95).draw(U[:, r].numpy())
        assert np.array_equal(tok[r].numpy()[~d["at_risk"]], d["token"][~d["at_risk"]])
    g = run_entry(ops, view, entry, 1.0, 20, 0.95, U.cuda()[:1], do_sample=False)[0][:, 0]
    assert torch.equal(g, z.argmax(1))


@pytest.mark.parametrize("R", [1, 32, 1024])
def test_decode_advance(ops, R):
    cur = torch.arange(R + 8, dtype=torch.int32, device="cuda") * 3
    step = torch.tensor([5, 99], dtype=torch.int32, device="cuda")
    before = cur.clone()
    ops.decode_advance(step, cur[:R])
    torch.cuda.synchronize()
    assert torch.equal(cur[:R], before[:R] + 1) and torch.equal(cur[R:], before[R:])
    assert step.tolist() == [6, 99]


def test_refusals(ops):
    from bioreason_b200._lib import check, ffi, lib, ptr
    z = torch.randn(2, 5000, device="cuda")
    U = torch.rand(1, 2, device="cuda")
    tok = torch.zeros(2, 1, dtype=torch.int64, device="cuda")
    ws = ops.sample_workspace(2, 5000, "cuda")
    for kw, what in ((dict(top_k=0), "top_k"), (dict(temperature=0.0), "T > 0"), (dict(temperature=-1.0), "T > 0"),
                     (dict(top_p=0.0), "top_p"), (dict(top_p=-0.5), "top_p")):
        args = dict(temperature=1.0, top_k=20, top_p=0.9) | kw
        for w in (None, ws):
            with pytest.raises(RuntimeError, match=what):
                ops.sample_next(z, workspace=w, do_sample=True, uniforms=U, max_steps=1, tokens=tok, **args)
    stream = ffi.cast("void*", torch.cuda.current_stream().cuda_stream)
    with pytest.raises(RuntimeError, match="top_k"):                   # ops routes top_k > 32 to the single stage; the C ABI refuses it
        check(lib().br_sample_next_2stage(ptr(z, "float*"), 5000, 2, 5000, 1.0, 33, 0.9, 1, ptr(U, "float*"), ffi.NULL, 1, -1, 0, ffi.NULL,
                                          ptr(tok, "int64_t*"), ffi.NULL, ptr(ws), stream), "sample_next_2stage")
    cur = torch.zeros(1025, dtype=torch.int32, device="cuda")
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    for n in (0, 1025):
        with pytest.raises(RuntimeError, match="R in"):
            ops.decode_advance(step, cur[:n])
    torch.cuda.synchronize()
    assert torch.all(cur == 0) and step.item() == 0
