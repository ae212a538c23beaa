"""CPU checks of the full-vocabulary sampler's reference (sampler_full_ref.py): it equals HF's float64 warpers (temperature -> top-p ->
min-p with top-k off, and TopKLogitsWarper for k > 1024) on off-risk draws; an emulation of the kernel's integer arithmetic with
adversarial exp errors agrees with it off risk; each one-bug variant differs; the at-risk fraction of the random families is below 1 %;
SamplingParams routes top_k = 0 and refuses top_k < 0."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sampler_full_ref as fr  # noqa: E402
import sampler_ref as sr  # noqa: E402

V = 12289


def hf_draw(z, T, top_k, top_p, min_p, u):
    """HF's warpers in float64, then the inverse CDF in id order with the uniforms u."""
    from transformers.generation.logits_process import MinPLogitsWarper, TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    s = torch.from_numpy(np.asarray(z, dtype=np.float32).astype(np.float64))[None]
    ids = torch.zeros(1, 0, dtype=torch.long)
    s = TemperatureLogitsWarper(float(np.float32(T)))(ids, s)
    if top_k:
        s = TopKLogitsWarper(top_k)(ids, s)
    if top_p < 1:
        s = TopPLogitsWarper(float(np.float32(top_p)))(ids, s)
    if min_p > 0:
        s = MinPLogitsWarper(float(np.float32(min_p)))(ids, s)
    cdf = torch.softmax(s, -1).cumsum(-1)[0].numpy()
    t = np.asarray(u, dtype=np.float32).astype(np.float64) * cdf[-1]
    return np.searchsorted(cdf, t, side="right")


@pytest.mark.parametrize("family", ["flat", "randn1", "randn3", "randn10", "peaked"])
@pytest.mark.parametrize("T,k,p,mp", [(1.0, 0, 0.95, 0.0), (0.6, 0, 0.5, 0.0), (1.5, 0, 0.9, 0.05), (1.0, 2000, 1.0, 0.0),
                                      (1.0, 1500, 0.9, 0.0)])
def test_reference_equals_hf(family, T, k, p, mp):
    z = fr.make_logits(family, 2, V, seed=3)
    U = sr.distinct_uniforms(40, 2, seed=4)
    for r in range(2):
        ref = fr.draw_full_ref(z[r].numpy(), T, k, p, U[:, r].numpy(), mp)
        hf = hf_draw(z[r].numpy(), T, k, p, mp, U[:, r].numpy())
        ok = ~ref["at_risk"]
        assert ok.sum() >= 30
        assert np.array_equal(ref["token"][ok], hf[ok]), (family, r)


@pytest.mark.parametrize("family", ["flat", "randn3", "randn30", "ties_spread", "last_chunk_mass", "neg_inf_chunks", "zero_mass"])
def test_kernel_emulation_agrees_off_risk(family):
    z = fr.make_logits(family, 3, V, seed=5)
    U = sr.distinct_uniforms(12, 3, seed=6)
    rng = np.random.default_rng(0)
    for T, k, p, mp in [(1.0, 0, 0.95, 0.0), (0.6, 5000, 0.5, 0.0), (1.5, 0, 1.0, 0.02)]:
        for r in range(3):
            ref = fr.draw_full_ref(z[r].numpy(), T, k, p, U[:, r].numpy(), mp)
            for signs in (None, rng.uniform(-1, 1, V), np.ones(V), -np.ones(V)):
                got = fr.emulate_kernel(z[r].numpy(), T, k, p, U[:, r].numpy(), mp, signs=signs)
                for s in range(len(got)):
                    if ref["at_risk"][s]:
                        assert got[s] in ref["allowed"][s]
                    else:
                        assert got[s] == ref["token"][s], (family, T, k, p, r, s)


@pytest.mark.parametrize("variant", fr.VARIANTS)
def test_variants_differ(variant):
    fam = fr.EXPOSED_BY[variant]
    Vv = 151936 if fam != "last_chunk_mass" else 152000
    z = fr.make_logits(fam, 2, Vv, seed=11)
    T, k, p = (1.0, 0, 0.5) if variant != "cut_at_T1" else (0.6, 0, 0.5)
    U = sr.grid_uniforms(16, 2)
    diff = 0
    for r in range(2):
        a = fr.draw_full_ref(z[r].numpy(), T, k, p, U[:, r].numpy())["token"]
        b = fr.draw_full_ref(z[r].numpy(), T, k, p, U[:, r].numpy(), variant=variant)["token"]
        diff += int((a != b).sum())
    assert diff > 0, variant


def test_at_risk_fraction_below_one_percent():
    n = risk = 0
    for fam in fr.RANDOM_FAMILIES + ("flat",):
        z = fr.make_logits(fam, 2, 151936, seed=1)
        U = sr.distinct_uniforms(50, 2, seed=2)
        for T, k, p in [(1.0, 0, 0.95), (0.6, 0, 0.5), (1.0, 0, 1.0)]:
            for r in range(2):
                out = fr.draw_full_ref(z[r].numpy(), T, k, p, U[:, r].numpy())
                n += len(out["token"]); risk += int(out["at_risk"].sum())
    assert risk < 0.01 * n, (risk, n)


def test_sampling_params_routing_and_refusals():
    from types import SimpleNamespace
    from bioreason_b200.generation import FULL_VOCAB_TOP_K, SamplingParams
    cfg = SimpleNamespace(eos_token_id=2, pad_token_id=0)
    assert SamplingParams.from_hf_kwargs(cfg, dict(do_sample=True, top_k=0)).top_k == 0
    assert SamplingParams.from_hf_kwargs(cfg, dict(do_sample=True)).top_k == 50           # None: HF's default
    assert SamplingParams.from_hf_kwargs(cfg, dict(do_sample=True, top_k=5000)).top_k == 5000 > FULL_VOCAB_TOP_K
    with pytest.raises(ValueError):
        SamplingParams.from_hf_kwargs(cfg, dict(do_sample=True, top_k=-1))
