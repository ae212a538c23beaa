"""The float64 draw reference of tests/sampler_ref.py, without a GPU: it equals transformers' own warpers run in float64 where the tie
order is unambiguous, an fp32 emulation of the kernel's arithmetic with every __expf perturbed by its full error agrees with it on every
draw that is not at risk, each one-bug variant differs from it on its own family, and at-risk draws are rare."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sampler_ref as sr  # noqa: E402

V_CPU = 5000                     # two chunks: the tail chunk is short
SETTINGS = [(0.6, 20, 0.95), (1.0, 50, 1.0), (0.3, 2, 0.5), (1.5, 33, 1e-3), (1.0, 1, 1.0), (0.6, 1024, 0.95)]


def hf_draw(z, T, k, p, u):
    """transformers' TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper in float64, then the id-ordered inverse CDF."""
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    s = torch.from_numpy(np.asarray(z, dtype=np.float32).astype(np.float64))[None]
    for w in (TemperatureLogitsWarper(sr.f32(T)), TopKLogitsWarper(top_k=k), TopPLogitsWarper(top_p=sr.f32(p))):
        s = w(None, s)
    probs = torch.softmax(s, -1)[0]
    cdf = probs.cumsum(0)
    u = torch.from_numpy(np.asarray(u, dtype=np.float32).astype(np.float64))
    tok = torch.searchsorted(cdf, u * cdf[-1], right=True).clamp(max=len(cdf) - 1)
    return tok.numpy(), np.nonzero(probs.numpy() > 0)[0]


@pytest.mark.parametrize("family", ["randn1", "randn3", "randn10", "randn30", "peaked", "flat_top", "chunk_local", "fewer_finite_than_k"])
def test_draw_ref_equals_hf_warpers(family):
    z = sr.make_logits(family, 6, V_CPU, seed=3).numpy()
    u = sr.distinct_uniforms(64, 1, seed=4).numpy()[:, 0]
    n = 0
    for r in range(z.shape[0]):
        for T, k, p in SETTINGS:
            ref = sr.draw_ref(z[r], T, k, p, u, maxc=None)
            if len(np.unique(z[r][ref["kept_topk"]])) != len(ref["kept_topk"]):
                continue                                               # tie order at the cut unspecified in HF
            tok, support = hf_draw(z[r], T, k, p, u)
            assert np.array_equal(support, ref["kept"]), (family, r, T, k, p)
            ok = ~ref["at_risk"]
            assert np.array_equal(tok[ok], ref["token"][ok]), (family, r, T, k, p)
            n += int(ok.sum())
    assert n > 0


def test_draw_ref_keeps_every_tie_like_hf():
    """tie_overflow_chunk: HF keeps the 10 distinct values and all 100 ties of the k-th (110 tokens, the ties hold
    100 / (10 e + 100) ~ 0.79 at T = 1 for exact 1.0 values); so does the reference, and cap64_per_chunk keeps 64."""
    z = sr.make_logits("tie_overflow_chunk", 2, V_CPU, seed=1).numpy()
    for r in range(2):
        ref = sr.draw_ref(z[r], 1.0, 20, 1.0, np.array([0.5], np.float32))
        hf_support = hf_draw(z[r], 1.0, 20, 1.0, [0.5])[1]
        assert len(ref["kept"]) == 110 and np.array_equal(hf_support, ref["kept"])
        assert len(sr.draw_ref(z[r], 1.0, 20, 1.0, [0.5], variant="cap64_per_chunk")["kept"]) == 64
    z = sr.make_logits("tie_overflow_1024", 1, 20 * sr.CHUNK, seed=1).numpy()[0]
    ref = sr.draw_ref(z, 1.0, 20, 1.0, [0.5])
    kth_ties = np.nonzero(z == 0.0)[0]
    assert len(kth_ties) == 1200 and len(ref["kept"]) == sr.MAXC
    assert np.array_equal(np.setdiff1d(ref["kept"], kth_ties), np.arange(19) * sr.CHUNK)   # every value above the k-th stays
    assert np.array_equal(np.intersect1d(ref["kept"], kth_ties), kth_ties[:sr.MAXC - 19])   # then the lowest-id ties
    assert len(sr.draw_ref(z, 1.0, 20, 1.0, [0.5], maxc=None)["kept"]) == 1219


def test_top_k_clamped_to_v():
    z = sr.make_logits("randn3", 1, 19, seed=2).numpy()[0]
    ref = sr.draw_ref(z, 1.0, 50, 1.0, np.linspace(0, 0.99, 9, dtype=np.float32))
    assert np.array_equal(ref["kept"], np.arange(19))


@pytest.mark.parametrize("family", ["randn1", "randn3", "randn10", "randn30", "flat_top", "peaked", "tie_overflow_chunk",
                                    "fewer_finite_than_k"])
def test_fp32_emulation_agrees_off_risk(family):
    z = sr.make_logits(family, 4, V_CPU, seed=7).numpy()
    u = sr.grid_uniforms(256, 1).numpy()[:, 0]
    rng = np.random.default_rng(0)
    n_risk = n = 0
    for r in range(z.shape[0]):
        for T, k, p in SETTINGS:
            ref = sr.draw_ref(z[r], T, k, p, u)
            c = len(ref["kept_topk"])
            for signs in (np.ones(c), -np.ones(c), np.where(np.arange(c) % 2 == 0, 1.0, -1.0), rng.uniform(-1, 1, c)):
                tok = sr.emulate_fp32(z[r], T, k, p, u, signs)
                ok = ~ref["at_risk"]
                assert np.array_equal(tok[ok], ref["token"][ok]), (family, r, T, k, p)
                bad = ref["at_risk"] & ~(ref["allowed"] == tok[:, None]).any(1)
                assert not bad.any(), (family, r, T, k, p)
            n += len(u)
            n_risk += int(ref["at_risk"].sum())
    print(f"{family}: {n_risk} of {n} draws at risk")


def _variant_draws(variant, family):
    V = 20 * sr.CHUNK if family == "tie_overflow_1024" else V_CPU
    z = sr.make_logits(family, 3, V, seed=5).numpy()
    S, R = 32, 3
    U = sr.grid_uniforms(S, R).numpy().reshape(-1)
    for r in range(R):
        for T, k, p in [(0.6, 20, 0.95), (1.0, 20, 1.0), (1.0, 20, 0.5)]:
            u = U[[sr.uniform_index(s, r, S, R) for s in range(S)]]
            ref = sr.draw_ref(z[r], T, k, p, u)
            uv = U[[sr.uniform_index(s, r, S, R, variant) for s in range(S)]]
            yield ref, sr.draw_ref(z[r], T, k, p, uv, variant=None if variant == "uniforms_row_major" else variant)


@pytest.mark.parametrize("variant", sr.VARIANTS)
def test_variants_differ_off_risk(variant):
    n = 0
    for ref, wrong in _variant_draws(variant, sr.EXPOSED_BY[variant]):
        n += int((~ref["at_risk"] & (wrong["token"] != ref["token"])).sum())
    assert n > 0, variant


def test_at_risk_draws_are_rare():
    n = n_risk = 0
    for family in sr.RANDOM_FAMILIES:
        z = sr.make_logits(family, 4, V_CPU, seed=9).numpy()
        u = sr.distinct_uniforms(128, 1, seed=1).numpy()[:, 0]
        for r in range(4):
            for T, k, p in SETTINGS:
                ref = sr.draw_ref(z[r], T, k, p, u)
                n += len(u)
                n_risk += int(ref["at_risk"].sum())
    print(f"random families: {n_risk} of {n} draws at risk ({100 * n_risk / n:.3f} %)")
    assert n_risk < 0.01 * n
