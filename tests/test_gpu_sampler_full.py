"""The full-vocabulary sampler (br_sample_next_full) against the float64 reference of sampler_full_ref.py, draw by draw: every draw not
at risk equals the reference token, an at-risk draw is one of the tokens beside the boundary it is at risk on.  Also the bookkeeping and
the presence bitmap bit for bit, repeated launches bit-identical, agreement with the two-stage sampler at top_k <= 32 (tokens off risk,
logp bit-equal), the one-bug variants disagreeing with the kernel, and generate() / the trainer with top_k = 0 end to end."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sampler_full_ref as fr  # noqa: E402
import sampler_proc_ref as spr  # noqa: E402
import sampler_ref as sr  # noqa: E402

pytestmark = pytest.mark.gpu
SENTINEL = -7


@pytest.fixture(scope="module")
def ops():
    from bioreason_b200.build import ensure_built
    ensure_built()
    from bioreason_b200 import ops as o
    return o


def run_full(ops, z, T, k, p, U, *, logp=False, proc=None, presence=None, finished=None, eos_id=-1, pad_id=0, steps=None, ws=None):
    R, V = z.shape
    S = U.shape[0]
    ws = ops.sample_full_workspace(R, V, "cuda") if ws is None else ws
    tok = torch.full((R, S), SENTINEL, device="cuda", dtype=torch.int64)
    nxt = torch.full((R,), SENTINEL, device="cuda", dtype=torch.int64)
    lp = torch.zeros(R, S, device="cuda") if logp else None
    step = torch.zeros(1, device="cuda", dtype=torch.int32)
    fin = torch.zeros(R, device="cuda", dtype=torch.int32) if finished is None else finished
    for s in (range(S) if steps is None else steps):
        step.fill_(s)
        ops.sample_next_full(z, workspace=ws, temperature=T, top_k=k, top_p=p, uniforms=U, step=step, max_steps=S, eos_id=eos_id,
                             pad_id=pad_id, finished=fin, tokens=tok, next_ids=nxt, logp=lp, presence=presence, **(proc or {}))
    torch.cuda.synchronize()
    return tok.cpu(), nxt.cpu(), fin.cpu(), (lp.cpu() if logp else None)


def check_draws(z, T, k, p, U, tok, min_p=0.0):
    """Every draw off risk equals the reference; at-risk draws are allowed tokens.  Returns (n_draws, n_at_risk)."""
    n = risk = 0
    for r in range(z.shape[0]):
        out = fr.draw_full_ref(z[r].numpy(), T, k, p, U[:, r].numpy(), min_p)
        got = tok[r].numpy()
        for s in range(U.shape[0]):
            n += 1
            if out["at_risk"][s]:
                risk += 1
                assert got[s] in out["allowed"][s], (r, s, got[s], out["allowed"][s])
            else:
                assert got[s] == out["token"][s], (r, s, got[s], out["token"][s], T, k, p)
    return n, risk


SIZES = [(1, 151936), (3, 152000), (8, 12289), (32, 1000)]
SETTINGS = [(0.6, 0, 0.95), (1.0, 0, 1.0), (1.5, 0, 0.5), (1.0, 1025, 0.95), (0.6, 5000, 1.0), (1.5, "V", 0.95), (1.0, "V+7", 0.5)]


@pytest.mark.parametrize("R,V", SIZES)
@pytest.mark.parametrize("family", ["flat", "randn1", "randn3", "randn10", "randn30", "peaked", "ties_spread", "last_chunk_mass",
                                    "neg_inf_chunks", "zero_mass"])
def test_draws_against_reference(ops, R, V, family):
    z = fr.make_logits(family, R, V, seed=V + R)
    zc = z.cuda()
    S = 6
    n = risk = 0
    for i, (T, k, p) in enumerate(SETTINGS):
        k = V if k == "V" else (V + 7 if k == "V+7" else k)
        U = sr.distinct_uniforms(S, R, seed=100 * i + R)
        tok, nxt, _, lp = run_full(ops, zc, T, k, p, U.cuda(), logp=(i % 2 == 0))
        a, b = check_draws(z, T, k, p, U, tok)
        n += a; risk += b
        assert torch.equal(nxt, tok[:, -1])
        if lp is not None:
            for r in range(R):
                for s in range(S):
                    y = int(tok[r, s])
                    assert abs(float(lp[r, s]) - spr.logp_raw(z[r].numpy(), y)) <= 1e-4 * (1 + abs(spr.logp_raw(z[r].numpy(), y)))
    if family in fr.RANDOM_FAMILIES:
        assert risk <= 0.01 * n + 1, (risk, n)


@pytest.mark.parametrize("V", [151936, 12289])
def test_processors_against_reference(ops, V):
    R, S = 4, 5
    z = fr.make_logits("randn3", R, V, seed=7)
    ids = [np.random.default_rng(r).integers(0, V, 40) for r in range(R)]
    eos, theta, m, min_p = 11, 1.3, 3, 0.05
    for T, k, p in [(1.0, 0, 0.95), (0.6, 2000, 1.0), (1.5, 0, 0.5)]:
        U = sr.distinct_uniforms(S, R, seed=int(T * 10) + k)
        pres = torch.from_numpy(spr.bitmap(ids, V)).cuda()
        tok, _, _, lp = run_full(ops, z.cuda(), T, k, p, U.cuda(), logp=True, presence=pres, eos_id=eos,
                                 proc=dict(repetition_penalty=theta, min_p=min_p, min_new_tokens=m))
        for r in range(R):
            seen = list(ids[r])
            for s in range(S):
                zp = spr.penalize(z[r].numpy(), seen, theta, eos=eos, blocked=spr.eos_blocked(s, m))
                out = fr.draw_full_ref(zp, T, k, p, U[s:s + 1, r].numpy(), min_p)
                got = int(tok[r, s])
                if out["at_risk"][0]:
                    assert got in out["allowed"][0]
                else:
                    assert got == out["token"][0], (r, s, got, out["token"][0])
                assert abs(float(lp[r, s]) - spr.logp_raw(z[r].numpy(), got)) <= 1e-4 * (1 + abs(spr.logp_raw(z[r].numpy(), got)))
                seen.append(got)
        got_ids = spr.ids_of_bitmap(pres.cpu().numpy(), V)
        for r in range(R):
            assert np.array_equal(got_ids[r], np.unique(np.concatenate([ids[r], tok[r].numpy()])))


def test_bookkeeping_and_repeat(ops):
    R, V, S = 5, 151936, 8
    z = fr.make_logits("randn3", R, V, seed=3)
    z[2, 77] = 60.0                                                    # row 2 draws EOS = 77 at every step
    U = sr.distinct_uniforms(S, R, seed=5).cuda()
    fin = torch.zeros(R, device="cuda", dtype=torch.int32)
    fin[4] = 1                                                         # already finished: pad
    tok, nxt, f, _ = run_full(ops, z.cuda(), 1.0, 0, 0.95, U, finished=fin, eos_id=77, pad_id=5)
    assert tok[2, 0] == 77 and (tok[2, 1:] == 5).all() and f[2] == 1
    assert (tok[4] == 5).all() and f[4] == 1
    assert torch.equal(nxt, tok[:, -1])
    ws = ops.sample_full_workspace(R, V, "cuda")
    ws.fill_(0xAB)                                                     # no initialisation needed
    a = run_full(ops, z.cuda(), 0.6, 0, 0.95, U, logp=True, ws=ws)
    for _ in range(3):
        b = run_full(ops, z.cuda(), 0.6, 0, 0.95, U, logp=True, ws=ws)
        assert torch.equal(a[0], b[0]) and torch.equal(a[3], b[3])
    # step >= max_steps writes no token
    tok2, nxt2, _, _ = run_full(ops, z.cuda(), 1.0, 0, 1.0, U[:2], steps=[5])
    assert (tok2 == SENTINEL).all() and (nxt2 != SENTINEL).all()


def test_empty_row_draws_pad(ops):
    R, V = 3, 12289
    z = torch.randn(R, V)
    z[1] = -math.inf
    U = sr.distinct_uniforms(2, R, seed=1)
    for k, p in [(0, 1.0), (0, 0.9), (2000, 0.9)]:
        tok, _, _, _ = run_full(ops, z.cuda(), 1.0, k, p, U.cuda(), pad_id=9)
        assert (tok[1] == 9).all()


@pytest.mark.parametrize("k", [1, 20, 32])
def test_matches_two_stage(ops, k):
    R, V, S = 8, 151936, 8
    z = fr.make_logits("randn3", R, V, seed=k)
    U = sr.distinct_uniforms(S, R, seed=k)
    for T, p in [(1.0, 0.95), (0.6, 1.0)]:
        full = run_full(ops, z.cuda(), T, k, p, U.cuda(), logp=True)
        ws = ops.sample_workspace(R, V, "cuda", logp=True)
        tok = torch.full((R, S), SENTINEL, device="cuda", dtype=torch.int64)
        lp = torch.zeros(R, S, device="cuda")
        step = torch.zeros(1, device="cuda", dtype=torch.int32)
        for s in range(S):
            step.fill_(s)
            ops.sample_next(z.cuda(), workspace=ws, temperature=T, top_k=k, top_p=p, uniforms=U.cuda(), step=step, max_steps=S,
                            tokens=tok, logp=lp)
        tok, lp = tok.cpu(), lp.cpu()
        for r in range(R):
            ref = fr.draw_full_ref(z[r].numpy(), T, k, p, U[:, r].numpy())
            for s in range(S):
                if not ref["at_risk"][s]:
                    assert full[0][r, s] == tok[r, s]
                if full[0][r, s] == tok[r, s]:
                    assert full[3][r, s].item() == lp[r, s].item()           # bit-equal log-prob


def test_refusals(ops):
    z = torch.randn(2, 1000, device="cuda")
    ws = ops.sample_full_workspace(2, 1000, "cuda")
    U = torch.rand(1, 2, device="cuda")
    for kw in (dict(temperature=0.0), dict(top_p=0.0), dict(top_k=-1), dict(uniforms=None), dict(min_p=1.5)):
        args = dict(workspace=ws, uniforms=U, max_steps=1)
        args.update(kw)
        with pytest.raises(RuntimeError):
            ops.sample_next_full(z, **args)
    with pytest.raises(RuntimeError):
        ops.sample_next(z, top_k=0, do_sample=True, uniforms=U)          # the top-k samplers still refuse top_k = 0


@pytest.mark.parametrize("variant", fr.VARIANTS)
def test_variants_disagree_with_kernel(ops, variant):
    fam = fr.EXPOSED_BY[variant]
    R, V, S = 8, 151936 if fam != "last_chunk_mass" else 152000, 16
    z = fr.make_logits(fam, R, V, seed=11)
    T, k, p = (1.0, 0, 0.5) if variant != "cut_at_T1" else (0.6, 0, 0.5)
    U = sr.grid_uniforms(S, R)
    tok = run_full(ops, z.cuda(), T, k, p, U.cuda())[0]
    diff = 0
    for r in range(R):
        ref = fr.draw_full_ref(z[r].numpy(), T, k, p, U[:, r].numpy(), variant=variant)
        diff += int((ref["token"] != tok[r].numpy()).sum())
    assert diff > 0, variant


# ------------------------------------------------------------------------------------------------------------------- end to end
def _model(seed=5):
    from bioreason_b200.configs import dna_config, text_config
    from bioreason_b200.models import DNALLMModel
    from oracle.models import build_oracle
    tc, dc = text_config("tiny"), dna_config("tiny")
    oracle = build_oracle(tc, dc, seed=seed)
    return DNALLMModel.from_oracle(oracle), oracle, tc, dc


def test_generate_top_k_0_against_manual_loop_graph_and_fp8():
    """generate(do_sample=True, top_k=0) with supplied uniforms equals the manual loop (HF's warpers without top-k) at every step the
    oracle's margin leaves exact; graph equals eager bit for bit; top_k > 1024 takes the same path; FP8 rollout returns log-probs."""
    from oracle.models import synth_batch
    m, oracle, tc, dc = _model(seed=6)
    batch = synth_batch(tc, dc, batch=4, n_seq=2, dna_len=10, text_len=18, seed=15, same_prompt=True)
    C = 12
    U = torch.rand(C, 4, generator=torch.Generator().manual_seed(3))
    for T, p in [(1.0, 1.0), (0.7, 0.9)]:
        kw = dict(max_new_tokens=C, do_sample=True, temperature=T, top_k=0, top_p=p, uniforms=U, eos_token_id=tc.eos_token_id, pad_token_id=0)
        a = m.generate(**batch, use_graph=True, return_logprobs=True, **kw)
        b = m.generate(**batch, use_graph=False, return_logprobs=True, **kw)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))
        assert torch.all(torch.isfinite(a[1])) and torch.all(a[1] <= 0)
        want, margins = spr.manual_processed_generate(oracle, batch, max_new_tokens=C, do_sample=True, temperature=T, top_k=0, top_p=p,
                                                      uniforms=U, eos_token_id=tc.eos_token_id, pad_token_id=0, return_margins=True)
        got = a[0].cpu()
        for r in range(4):
            n = min(got.shape[1], want.shape[1])
            close = (margins[r, :n] < 3e-2).nonzero()
            upto = int(close[0]) if len(close) else n
            assert torch.equal(got[r, :upto], want[r, :upto]), (T, p, r, got[r], want[r])
        big = m.generate(**batch, **{**kw, "top_k": tc.vocab_size + 5})
        assert torch.equal(big, a[0])                                    # top_k >= V keeps every finite value: same as top_k = 0
    m.set_fp8_rollout(True)
    ids, lp = m.generate(**batch, return_logprobs=True, max_new_tokens=C, do_sample=True, top_k=0, top_p=0.95, uniforms=U)
    m.set_fp8_rollout(False)
    assert lp.shape == ids.shape and torch.all(torch.isfinite(lp)) and torch.all(lp <= 0)


def test_training_step_top_k_0_with_is_correction():
    from bioreason_b200.trainer import DNALLMGRPOConfig, DNALLMGRPOTrainer
    from oracle.models import synth_batch
    m, oracle, tc, dc = _model(seed=21)
    batch = synth_batch(tc, dc, batch=4, n_seq=2, dna_len=10, text_len=18, seed=14, same_prompt=True)
    cfg = DNALLMGRPOConfig(num_generations=4, max_completion_length=6, per_device_train_batch_size=4, learning_rate=1e-2, lora_r=16,
                           lora_alpha=32.0, micro_rows=4, sampling_from_config=True, temperature=1.0, top_k=0, top_p=1.0,
                           rollout_is_correction=True)
    reward = lambda completion_ids, **kw: (completion_ids % 7 == 0).float().sum(1)
    tr = DNALLMGRPOTrainer(m, [reward], cfg)
    assert tr.generation_kwargs["top_k"] == 0
    for _ in range(2):
        assert torch.isfinite(tr.training_step(batch))
    met = tr.log_metrics()
    assert 0 < met["rollout_is/ratio_mean"] and math.isfinite(met["rollout_is/logp_diff"])
