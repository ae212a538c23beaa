"""The processed sampler (br_sample_next_proc / br_sample_next_2stage_proc: repetition penalty, min_new_tokens, min-p) against the
float64 reference of sampler_proc_ref.py, draw by draw, with and without the log-prob output; the bitmap and the rest of the
bookkeeping bit for bit; neutral parameters equal the sampler without processors bit for bit; the one-bug variants disagree with the
kernel; and end to end on the tiny model: generate() against HF and the manual processed loop, graph against eager, the graph cache
key, num_return_sequences, and the trainer's sampling_from_config."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sampler_proc_ref as pr  # noqa: E402
import sampler_ref as sr  # noqa: E402

pytestmark = pytest.mark.gpu
SENTINEL = -7


@pytest.fixture(scope="module")
def ops():
    from bioreason_b200.build import ensure_built
    ensure_built()
    from bioreason_b200 import ops as o
    return o


def call_proc(z, *, two, logp, T, k, p, do_sample, U, step, max_steps, eos, pad, fin, tok, nxt, theta, min_p, m, presence, ws=None):
    """One call of a processed entry point through the C ABI (ops.sample_next routes neutral parameters to the plain sampler)."""
    from bioreason_b200._lib import check, ffi, lib, ptr
    R, V = z.shape
    proc = ffi.new("br_sample_proc*")
    proc.repetition_penalty, proc.min_p, proc.min_new_tokens = float(theta), float(min_p), int(m)
    proc.presence = ptr(presence, "uint32_t*")
    stream = ffi.cast("void*", torch.cuda.current_stream().cuda_stream)
    args = (ptr(z, "float*"), z.stride(0), R, V, float(T), int(k), float(p), 1 if do_sample else 0, ptr(U, "float*"), ptr(step, "int32_t*"),
            int(max_steps), int(eos), int(pad), ptr(fin, "int32_t*"), ptr(tok, "int64_t*"), ptr(nxt, "int64_t*"), ptr(logp, "float*"), proc)
    if two:
        check(lib().br_sample_next_2stage_proc(*args, ptr(ws), stream), "sample_next_2stage_proc")
    else:
        check(lib().br_sample_next_proc(*args, stream), "sample_next_proc")


def run_steps(ops, z, ids_per_row, *, two, logp, T, k, p, U, do_sample=True, eos=-1, m=0, theta=1.3, min_p=0.0, steps=(0,), fresh=True,
              fin0=None, pad=0, track_finished=True):
    """Tokens [R, S] and logp [R, S] over the given steps; fresh: the presence bitmap is reset to ids_per_row before each call;
    track_finished=False: no finished buffer (every step draws, whatever the row drew before)."""
    R, V = z.shape
    S = max(steps) + 1
    bm0 = torch.from_numpy(pr.bitmap(ids_per_row, V)).cuda()
    pres = bm0.clone()
    ws = ops.sample_workspace(R, V, "cuda", logp=True) if two else None
    tok = torch.full((R, S), SENTINEL, device="cuda", dtype=torch.int64)
    nxt = torch.full((R,), SENTINEL, device="cuda", dtype=torch.int64)
    lp = torch.zeros(R, S, device="cuda") if logp else None
    fin = torch.zeros(R, device="cuda", dtype=torch.int32) if fin0 is None else fin0.clone().cuda()
    step = torch.zeros(1, device="cuda", dtype=torch.int32)
    for s in steps:
        if fresh:
            pres.copy_(bm0)
        step.fill_(s)
        call_proc(z, two=two, logp=lp, T=T, k=k, p=p, do_sample=do_sample, U=U, step=step, max_steps=S, eos=eos, pad=pad,
                  fin=fin if track_finished else None, tok=tok,
                  nxt=nxt, theta=theta, min_p=min_p, m=m, presence=pres, ws=ws)
    torch.cuda.synchronize()
    return tok.cpu(), (lp.cpu() if logp else None), nxt.cpu(), fin.cpu(), pres.cpu()


ENTRIES = [(False, False), (False, True), (True, False), (True, True)]        # (two-stage, logp)

# (family, V, R, theta, top_k, T, top_p, min_p, m)
CASES = [
    ("max_demoted", 151936, 8, 1.3, 20, 0.6, 0.95, 0.05, 0), ("max_demoted", 1000, 3, 2.0, 64, 1.0, 1.0, 0.1, 0),
    ("negatives_in_set", 151936, 8, 1.3, 20, 1.0, 0.95, 0.0, 0), ("negatives_in_set", 12289, 3, 0.7, 32, 0.6, 1.0, 0.02, 0),
    ("negatives_in_set", 1000, 1, 0.7, 64, 1.0, 0.95, 0.0, 0),
    ("penalty_tie", 151936, 8, 1.3, 20, 0.6, 1.0, 0.0, 0), ("penalty_tie", 12289, 8, 1.1, 32, 0.6, 1.0, 0.0, 0),
    ("penalty_tie", 1000, 3, 0.7, 64, 0.6, 1.0, 0.0, 0),
    ("tie_overflow_chunk", 151936, 8, 1.3, 20, 1.0, 1.0, 0.0, 0), ("tie_overflow_chunk", 12289, 8, 0.7, 20, 0.6, 0.95, 0.0, 0),
    ("tie_overflow_chunk", 1000, 3, 1.1, 64, 1.0, 1.0, 0.0, 0),
    ("chunk_in_set", 151936, 8, 1.3, 20, 1.0, 0.95, 0.0, 0), ("chunk_in_set", 12289, 3, 0.7, 32, 0.6, 0.95, 0.05, 0),
    ("chunk_in_set", 1000, 8, 2.0, 64, 1.0, 1.0, 0.0, 0),
    ("eos_argmax", 151936, 8, 1.3, 20, 0.6, 0.95, 0.0, 3), ("eos_argmax", 12289, 32, 0.7, 32, 1.0, 1.0, 0.0, 2),
    ("eos_argmax", 1000, 3, 1.1, 64, 1.0, 0.95, 0.0, 5),
    ("minp_only_max", 151936, 8, 1.3, 20, 1.0, 1.0, 0.1, 0), ("minp_only_max", 1000, 3, 0.7, 64, 0.6, 0.95, 0.2, 0),
    ("minp_boundary", 151936, 8, 1.1, 20, 1.0, 1.0, 0.1, 0), ("minp_boundary", 12289, 32, 1.3, 32, 1.0, 0.95, 0.1, 0),
    ("minp_boundary", 1000, 8, 0.7, 64, 1.0, 1.0, 0.1, 0),
    ("history_dups", 151936, 32, 1.3, 20, 0.6, 0.95, 0.0, 0), ("history_dups", 1000, 8, 2.0, 32, 1.0, 1.0, 0.0, 0),
    ("randn3", 151936, 32, 1.1, 20, 0.6, 0.95, 0.02, 2), ("randn3", 12289, 8, 0.7, 64, 1.0, 0.95, 0.0, 0),
    ("randn3", 1000, 1, 1.3, 32, 1.5, 0.5, 0.05, 1),
]
STATS = {}


def _case_id(c):
    return f"{c[0]}-V{c[1]}-R{c[2]}-th{c[3]}-k{c[4]}-T{c[5]}-p{c[6]}-mp{c[7]}-m{c[8]}"


def _rows(fam, V, R, theta, k, T, seed):
    cases = [pr.make_case(fam, V, seed + r, top_k=k, theta=theta, T=T) for r in range(R)]
    z = torch.from_numpy(np.stack([c[0] for c in cases]))
    return z, [c[1] for c in cases], [c[2] for c in cases], cases


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_draws_vs_fp64(ops, case):
    fam, V, R, theta, k, T, p, mp, m = case
    S = 8
    z, ids, eos_rows, _ = _rows(fam, V, R, theta, k, T, seed=V + R)
    eos = eos_rows[0]
    if fam == "eos_argmax":                                            # one EOS id for the call: put it on every row's argmax
        for r in range(R):
            z[r, eos] = z[r].max() + 20.0
    U = sr.distinct_uniforms(S, R, seed=V + k)
    zc, Uc = z.cuda(), U.cuda()
    steps = tuple(range(S))
    entries = ENTRIES if k <= 32 else ENTRIES[:2]
    res = {e: run_steps(ops, zc, ids, two=e[0], logp=e[1], T=T, k=k, p=p, U=Uc, eos=eos, m=m, theta=theta, min_p=mp, steps=steps,
                        track_finished=False) for e in entries}
    tok = res[entries[0]][0]
    for e in entries:
        assert torch.equal(res[e][0], tok), (e, "differs from the single-stage draw")
    st = STATS.setdefault(fam, {"draws": 0, "at_risk": 0, "min_cut_ratio": math.inf})
    for r in range(R):
        for s in steps:
            d = pr.draw_proc_ref(z[r].numpy(), ids[r], theta, s, m, eos, T, k, p, mp, U[s, r].item())
            y = int(tok[r, s])
            if not d["at_risk"][0]:
                assert y == int(d["token"][0]), (r, s, y, int(d["token"][0]))
            assert (d["allowed"][0] == y).any(), (r, s)
            if fam == "eos_argmax" and s < m:
                assert y != eos
            st["draws"] += 1
            st["at_risk"] += int(d["at_risk"][0])
            st["min_cut_ratio"] = min(st["min_cut_ratio"], d["row"].m_minp)
            for e in entries:
                if e[1]:                                               # log-prob of the raw row at the chosen token
                    lp = float(res[e][1][r, s])
                    want = pr.logp_raw(z[r].numpy(), y)
                    assert abs(lp - want) <= 1e-5 * (1 + abs(want)), (e, r, s, lp, want)
    # greedy: argmax of the processed row, EOS masked while step < m
    for e in ENTRIES:
        for s in (0, m):
            g = run_steps(ops, zc, ids, two=e[0], logp=e[1], T=T, k=k, p=p, U=Uc[:1], do_sample=False, eos=eos, m=m, theta=theta,
                          min_p=mp, steps=(s,))[0][:, s]
            want = torch.tensor([pr.greedy_proc_ref(z[r].numpy(), ids[r], theta, s, m, eos) for r in range(R)])
            assert torch.equal(g, want), (e, s)


def test_draw_totals():
    if not STATS:
        pytest.skip("no draw case ran")
    for fam, s in sorted(STATS.items()):
        print(f"{fam:20s} draws {s['draws']:5d}  at risk {s['at_risk']:3d}  min min-p cut margin/delta {s['min_cut_ratio']:.3g}")


VARIANT_SETTINGS = {                                                   # (theta, T, top_k, top_p, min_p, m, greedy)
    "dup_twice": (1.3, 1.0, 20, 1.0, 0.0, 0, True), "penalty_after_T": (1.3, 0.6, 20, 1.0, 0.0, 0, False),
    "neg_divided": (1.3, 1.0, 20, 1.0, 0.0, 0, True), "min_new_le": (1.3, 1.0, 20, 1.0, 0.0, 2, True),
    "minp_raw_max": (1.3, 1.0, 20, 1.0, 0.1, 0, False), "minp_T1": (1.1, 0.6, 20, 1.0, 0.1, 0, False),
}


def test_variants_disagree_with_the_kernel(ops):
    """On the kernel's own draws, each kernel-level one-bug variant differs on a draw that is not at risk (prompt_in_set is a rollout
    variant: test_generate_matches_manual_loop and the CPU test against HF generate cover it)."""
    V, R, S = 151936, 4, 16
    for variant, (theta, T, k, p, mp, m, greedy) in VARIANT_SETTINGS.items():
        fam = pr.EXPOSED_BY[variant]
        z, ids, eos_rows, _ = _rows(fam, V, R, theta, k, T, seed=3)
        eos = eos_rows[0]
        if fam == "eos_argmax":
            for r in range(R):
                z[r, eos] = z[r].max() + 20.0
        U = sr.grid_uniforms(S, R)
        n = 0
        if greedy:
            for s in range(S):
                got = run_steps(ops, z.cuda(), ids, two=True, logp=False, T=T, k=k, p=p, U=U.cuda()[:1], do_sample=False, eos=eos, m=m,
                                theta=theta, steps=(s,), track_finished=False)[0][:, s]
                for r in range(R):
                    n += int(pr.greedy_proc_ref(z[r].numpy(), ids[r], theta, s, m, eos, variant=variant) != int(got[r]))
        else:
            got = run_steps(ops, z.cuda(), ids, two=True, logp=False, T=T, k=k, p=p, U=U.cuda(), eos=eos, m=m, theta=theta, min_p=mp,
                            steps=tuple(range(S)), track_finished=False)[0].numpy()
            for r in range(R):
                for s in range(S):
                    ref = pr.draw_proc_ref(z[r].numpy(), ids[r], theta, s, m, eos, T, k, p, mp, U[s, r].item())
                    wrong = pr.draw_proc_ref(z[r].numpy(), ids[r], theta, s, m, eos, T, k, p, mp, U[s, r].item(), variant=variant)
                    n += int(not ref["at_risk"][0] and int(wrong["token"][0]) != got[r, s])
        assert n > 0, variant


@pytest.mark.parametrize("two,logp", ENTRIES)
def test_bookkeeping_bitmap_exact(ops, two, logp):
    """A sequence of calls without resetting the bitmap: each draw sees the tokens emitted before it, the bitmap ends as the initial
    set plus every emitted token (pad for finished rows), tokens / next_ids / finished / logp exact."""
    R, V, S = 8, 4097, 6
    z = sr.make_logits("randn3", R, V, seed=1)
    z[2, 77] = 60.0                                                    # row 2 draws EOS = 77 once step >= m
    eos, pad, m, theta = 77, 4000, 2, 1.3
    init = [np.random.default_rng(r).integers(0, V, 5) for r in range(R)]
    U = sr.distinct_uniforms(S, R, seed=2)
    fin0 = torch.zeros(R, dtype=torch.int32)
    fin0[6] = 1
    tok, lp, nxt, fin, pres = run_steps(ops, z.cuda(), init, two=two, logp=logp, T=0.6, k=20, p=0.95, U=U.cuda(), eos=eos, m=m, theta=theta,
                                        steps=tuple(range(S)), fresh=False, fin0=fin0, pad=pad)
    for r in range(R):
        seen = list(init[r])
        done = bool(fin0[r])
        for s in range(S):
            y = int(tok[r, s])
            if done:
                assert y == pad
            else:
                d = pr.draw_proc_ref(z[r].numpy(), seen, theta, s, m, eos, 0.6, 20, 0.95, 0.0, U[s, r].item())
                assert d["at_risk"][0] or y == int(d["token"][0]), (r, s)
                assert (d["allowed"][0] == y).any()
                if logp:
                    assert abs(float(lp[r, s]) - pr.logp_raw(z[r].numpy(), y)) <= 1e-5 * (1 + abs(float(lp[r, s])))
            if logp and done:
                assert float(lp[r, s]) == 0.0
            seen.append(y)
            done = done or y == eos
        assert bool(fin[r]) == done and int(nxt[r]) == int(tok[r, S - 1])
        assert np.array_equal(pr.ids_of_bitmap(pres[r:r + 1].numpy(), V)[0], np.unique(seen)), r
    assert int(tok[2, 0]) != eos and int(tok[2, 1]) != eos and int(tok[2, 2]) == eos and bool(fin[2])


@pytest.mark.parametrize("fam", sr.FAMILIES)
def test_neutral_parameters_equal_the_plain_sampler(ops, fam):
    """theta = 1, min_p = 0, m = 0 through the processed entry points: the tokens and log-probs of the plain sampler, bit for bit."""
    R, S = 8, 8
    V = 151936
    z = sr.make_logits(fam, R, V, seed=11)
    U = (sr.grid_uniforms(S, R) if fam == "uniform_grid" else sr.distinct_uniforms(S, R, seed=12)).cuda()
    zc = z.cuda()
    for two, logp in ENTRIES:
        for do_sample in (True, False):
            ws = ops.sample_workspace(R, V, "cuda", logp=True) if two else None
            t0 = torch.full((R, S), SENTINEL, device="cuda", dtype=torch.int64)
            l0 = torch.zeros(R, S, device="cuda") if logp else None
            step = torch.zeros(1, device="cuda", dtype=torch.int32)
            for s in range(S):
                step.fill_(s)
                ops.sample_next(zc, workspace=ws, temperature=0.6, top_k=20, top_p=0.95, do_sample=do_sample, uniforms=U, step=step,
                                max_steps=S, tokens=t0, logp=l0)
            tok, lp, *_ = run_steps(ops, zc, [[]] * R, two=two, logp=logp, T=0.6, k=20, p=0.95, U=U, do_sample=do_sample, theta=1.0,
                                    steps=tuple(range(S)))
            assert torch.equal(tok, t0.cpu()), (two, logp, do_sample)
            if logp:
                assert torch.equal(lp.view(torch.int32), l0.cpu().view(torch.int32))


def test_refusals(ops):
    z = torch.randn(2, 5000, device="cuda")
    U = torch.rand(1, 2, device="cuda")
    tok = torch.zeros(2, 1, dtype=torch.int64, device="cuda")
    pres = ops.presence_bitmap(2, 5000, "cuda")
    for kw, what in ((dict(repetition_penalty=0.0), "repetition_penalty"), (dict(repetition_penalty=-1.0), "repetition_penalty"),
                     (dict(min_p=1.5), "min_p"), (dict(min_p=-0.1), "min_p"), (dict(min_new_tokens=-1), "min_new_tokens"),
                     (dict(repetition_penalty=1.2, presence=None), "presence")):
        args = dict(presence=pres) | kw
        for w in (None, ops.sample_workspace(2, 5000, "cuda")):
            with pytest.raises(RuntimeError, match=what):
                ops.sample_next(z, workspace=w, do_sample=True, temperature=1.0, top_k=20, top_p=0.9, uniforms=U, max_steps=1, tokens=tok,
                                **args)
    torch.cuda.synchronize()
    assert torch.all(pres == 0)


# ------------------------------------------------------------------------------------------------------------------- end to end
def _model(seed=5, size="tiny"):
    from bioreason_b200.configs import dna_config, text_config
    from bioreason_b200.models import DNALLMModel
    from oracle.models import build_oracle
    tc, dc = text_config(size), dna_config(size)
    oracle = build_oracle(tc, dc, seed=seed)
    return DNALLMModel.from_oracle(oracle), oracle, tc, dc


def test_greedy_matches_hf_generate():
    """Greedy generate(repetition_penalty, min_new_tokens / min_length) against HF generate on the fp32 oracle, under the project's
    greedy rule: identical up to the first step whose fp32 top-2 margin is below 1e-2 (a bf16 rollout may flip such a near tie)."""
    from oracle.models import synth_batch
    from sampler_proc_ref import manual_processed_generate
    m, oracle, tc, dc = _model()
    batch = synth_batch(tc, dc, batch=4, n_seq=2, dna_len=10, text_len=18, seed=14)
    P = batch["input_ids"].shape[1]
    eos = tc.eos_token_id
    for kw in (dict(repetition_penalty=1.3, min_new_tokens=4), dict(repetition_penalty=0.8, min_length=P + 3)):
        ids = m.generate(**batch, max_new_tokens=10, do_sample=False, eos_token_id=eos, pad_token_id=0, **kw).cpu()
        want = oracle.generate(**batch, max_new_tokens=10, do_sample=False, eos_token_id=eos, pad_token_id=0, **kw)
        _, margins = manual_processed_generate(oracle, batch, max_new_tokens=10, eos_token_id=eos, pad_token_id=0, return_margins=True,
                                               repetition_penalty=kw["repetition_penalty"], min_new_tokens=kw.get("min_new_tokens", 3))
        for r in range(ids.shape[0]):
            n = min(ids.shape[1], want.shape[1])
            close = (margins[r, :n] < 1e-2).nonzero()
            upto = int(close[0]) if len(close) else n
            assert torch.equal(ids[r, :upto], want[r, :upto].cpu()), (kw, r, ids[r], want[r])


def test_generate_matches_manual_loop_graph_and_cache():
    """Sampled generate with supplied uniforms equals the manual processed loop on the same (bf16-rounded) weights at every step the
    oracle's margin leaves exact; graph equals eager bit for bit; back-to-back rollouts with different theta each equal a fresh engine's."""
    from oracle.models import synth_batch
    from bioreason_b200.generation import RolloutEngine
    m, oracle, tc, dc = _model(seed=6)
    batch = synth_batch(tc, dc, batch=4, n_seq=2, dna_len=10, text_len=18, seed=15, same_prompt=True)
    C = 12
    U = torch.rand(C, 4, generator=torch.Generator().manual_seed(3))
    kw = dict(max_new_tokens=C, do_sample=True, temperature=0.7, top_k=20, top_p=0.95, min_p=0.05, uniforms=U, eos_token_id=tc.eos_token_id,
              pad_token_id=0)
    res = {}
    for th in (1.3, 0.8, 1.3):
        for use_graph in (True, False):
            res[(th, use_graph)] = m.generate(**batch, repetition_penalty=th, min_new_tokens=3, use_graph=use_graph, return_logprobs=True,
                                              **kw)
        a, b = res[(th, True)], res[(th, False)]
        assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32)), th
        m._rollout = RolloutEngine(m)                                  # a fresh engine for the next theta's reference below
        fresh = m.generate(**batch, repetition_penalty=th, min_new_tokens=3, use_graph=True, return_logprobs=True, **kw)
        assert torch.equal(fresh[0], a[0]), th
    # the cached engine, alternating theta (no engine reset): each equals the fresh result
    m._rollout = RolloutEngine(m)
    for th in (1.3, 0.8, 1.3, 0.8):
        ids = m.generate(**batch, repetition_penalty=th, min_new_tokens=3, **kw)
        assert torch.equal(ids, res[(th, True)][0]), th
    assert not torch.equal(res[(1.3, True)][0], res[(0.8, True)][0])
    # against the manual processed loop (HF's processor classes in HF's order, draw from the uniforms)
    from sampler_proc_ref import manual_processed_generate
    for th in (1.3, 0.8):
        want, margins = manual_processed_generate(oracle, batch, max_new_tokens=C, do_sample=True, temperature=0.7, top_k=20, top_p=0.95,
                                                  min_p=0.05, uniforms=U, eos_token_id=tc.eos_token_id, pad_token_id=0,
                                                  repetition_penalty=th, min_new_tokens=3, return_margins=True)
        got = res[(th, True)][0].cpu()
        for r in range(4):
            n = min(got.shape[1], want.shape[1])
            close = (margins[r, :n] < 3e-2).nonzero()                  # bf16 rollout vs fp32 loop: a draw this near an edge may flip
            upto = int(close[0]) if len(close) else n
            assert torch.equal(got[r, :upto], want[r, :upto]), (th, r, got[r], want[r])


def test_eos_terminated_rollout_respects_min_new_tokens():
    from oracle.models import synth_batch
    m, oracle, tc, dc = _model(seed=7)
    batch = synth_batch(tc, dc, batch=3, n_seq=1, dna_len=[9, 7, 9], text_len=[20, 15, 18], seed=9)
    ids = m.generate(**batch, max_new_tokens=8, do_sample=False).cpu()
    eos = int(ids[0, 1])                                               # row 0 emits this at step 1 without processors
    for use_graph in (False, True):
        out = m.generate(**batch, max_new_tokens=8, do_sample=False, eos_token_id=eos, pad_token_id=0, min_new_tokens=4,
                         use_graph=use_graph).cpu()
        for r in range(out.shape[0]):
            hit = (out[r] == eos).nonzero()
            assert len(hit) == 0 or int(hit[0]) >= 4, (r, out[r])
        keep = ids[:, 0] != eos                                        # rows whose first token was not EOS draw the same first token
        assert torch.equal(out[keep, :1], ids[keep, :1])


def test_num_return_sequences_equals_repeated_rows():
    from oracle.models import synth_batch
    from bioreason_b200.generation import expand_return_sequences
    m, oracle, tc, dc = _model(seed=8)
    batch = synth_batch(tc, dc, batch=2, n_seq=2, dna_len=10, text_len=18, seed=16)
    n, C = 4, 8
    U = torch.rand(C, 2 * n, generator=torch.Generator().manual_seed(4))
    kw = dict(max_new_tokens=C, do_sample=True, temperature=0.8, top_k=20, top_p=0.95, uniforms=U, repetition_penalty=1.2)
    ids, st = m.generate(**batch, num_return_sequences=n, return_stats=True, **kw)
    ii, am, dna, bim = expand_return_sequences(batch["input_ids"], batch["attention_mask"], batch["dna_tokenized"], batch["batch_idx_map"], n)
    ids2 = m.generate(input_ids=ii, attention_mask=am, dna_tokenized=dna, batch_idx_map=bim, **kw)
    assert torch.equal(ids, ids2) and ids.shape[0] == 2 * n
    assert st["G"] == n and st["unique_prompts"] == 2


def _trainer(sampling_from_config, **cfg_kw):
    from bioreason_b200.trainer import DNALLMGRPOConfig, DNALLMGRPOTrainer
    from oracle.models import synth_batch
    m, oracle, tc, dc = _model(seed=21)
    batch = synth_batch(tc, dc, batch=4, n_seq=2, dna_len=10, text_len=18, seed=14, same_prompt=True)
    cfg = DNALLMGRPOConfig(num_generations=4, max_completion_length=6, per_device_train_batch_size=4, learning_rate=1e-2, lora_r=16,
                           lora_alpha=32.0, micro_rows=4, sampling_from_config=sampling_from_config, **cfg_kw)
    reward = lambda completion_ids, **kw: (completion_ids % 7 == 0).float().sum(1)
    return DNALLMGRPOTrainer(m, [reward], cfg), m, batch


def test_trainer_sampling_from_config():
    """The reference's values with theta = 1 and min_p None: the same rollout ids as the flag off; theta = 1.2: the rollout equals
    model.generate with the config's kwargs."""
    tr0, m0, batch = _trainer(False)
    tr1, m1, _ = _trainer(True, temperature=0.6, top_p=0.95, top_k=20, min_p=None, repetition_penalty=1.0)
    assert tr0.generation_kwargs == {k: v for k, v in tr1.generation_kwargs.items() if k not in ("min_p", "repetition_penalty")}
    U = torch.rand(6, 4, generator=torch.Generator().manual_seed(9))
    mm = (batch["input_ids"], batch["attention_mask"], batch["dna_tokenized"], batch["batch_idx_map"])
    a = m0.generate(*mm, uniforms=U, **tr0.generation_kwargs)
    b = m1.generate(*mm, uniforms=U, **tr1.generation_kwargs)
    assert torch.equal(a, b)
    tr2, m2, _ = _trainer(True, repetition_penalty=1.2, temperature=0.9, top_k=30, top_p=0.9, min_p=0.02)
    kw = tr2.generation_kwargs
    assert (kw["repetition_penalty"], kw["temperature"], kw["top_k"], kw["top_p"], kw["min_p"]) == (1.2, 0.9, 30, 0.9, 0.02)
    c = m2.generate(*mm, uniforms=U, **kw)
    d = m2.generate(*mm, uniforms=U, max_new_tokens=6, do_sample=True, temperature=0.9, top_p=0.9, top_k=30, min_p=0.02,
                    repetition_penalty=1.2, pad_token_id=kw["pad_token_id"], eos_token_id=kw["eos_token_id"])
    assert torch.equal(c, d)
    assert not torch.equal(c, m2.generate(*mm, uniforms=U, **tr0.generation_kwargs))
