"""CPU checks of the processed sampler's reference (sampler_proc_ref.py) against transformers' own logits processors, its min-p error
model, the one-bug variants, the manual processed generation loop against HF generate() on the tiny oracle, and the host-side argument
handling (SamplingParams, num_return_sequences expansion, the trainer's sampling_from_config)."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sampler_proc_ref as pr  # noqa: E402
import sampler_ref as sr  # noqa: E402
from attn_ref import SAFETY  # noqa: E402
from transformers.generation.logits_process import (MinLengthLogitsProcessor, MinNewTokensLengthLogitsProcessor,  # noqa: E402
                                                    MinPLogitsWarper, RepetitionPenaltyLogitsProcessor, TemperatureLogitsWarper,
                                                    TopKLogitsWarper, TopPLogitsWarper)


def _special_row(V, seed):
    g = np.random.default_rng(seed)
    z = (g.standard_normal(V) * 3).astype(np.float32)
    z[:8] = [0.0, -0.0, -np.inf, -3.5, 2.25, 1e-30, -1e-30, 7.0]
    return z


@pytest.mark.parametrize("theta", [0.7, 1.1, 1.3, 2.0])
def test_penalty_equals_hf_bit_for_bit(theta):
    V, eos = 3000, 5
    for seed in range(4):
        z = _special_row(V, seed)
        g = np.random.default_rng(100 + seed)
        hist = np.concatenate([np.arange(8), [eos, eos], g.integers(0, V, 40), g.integers(0, 8, 10)])     # duplicates, EOS in the set
        for step, m in ((0, 3), (2, 3), (3, 3), (5, 0)):
            ids_t = torch.from_numpy(hist[None, :step + 50])               # any history length: HF sees the generated ids only
            s = RepetitionPenaltyLogitsProcessor(theta)(ids_t, torch.from_numpy(z[None].copy()))
            if m > 0:
                s = MinNewTokensLengthLogitsProcessor(0, m, eos)(torch.zeros(1, step, dtype=torch.long), s)
                s2 = MinLengthLogitsProcessor(m, eos)(torch.zeros(1, step, dtype=torch.long),
                                                      RepetitionPenaltyLogitsProcessor(theta)(ids_t, torch.from_numpy(z[None].copy())))
                assert torch.equal(s.view(torch.int32), s2.view(torch.int32))
            mine = pr.penalize(z, hist[:step + 50], theta, eos=eos, blocked=pr.eos_blocked(step, m))
            assert np.array_equal(s[0].numpy().view(np.int32), mine.view(np.int32)), (theta, seed, step, m)


@pytest.mark.parametrize("T,top_k,top_p,min_p", [(1.0, 50, 1.0, 0.1), (0.6, 20, 0.95, 0.05), (1.5, 64, 0.9, 0.2), (0.7, 1000, 1.0, 0.02)])
def test_min_p_kept_set_equals_hf(T, top_k, top_p, min_p):
    """After Temperature -> TopK -> TopP, HF's MinPLogitsWarper keeps the reference's set, except where the reference marks the cut at
    risk (then by one token)."""
    V, n_risk = 4000, 0
    for seed in range(30):
        z = pr.penalize(_special_row(V, seed)[::-1].copy(), np.arange(0, V, 7), 1.3)
        s = torch.from_numpy(z[None].astype(np.float64))
        for w in (TemperatureLogitsWarper(T), TopKLogitsWarper(top_k), TopPLogitsWarper(top_p), MinPLogitsWarper(min_p)):
            s = w(None, s)
        hf = np.sort(np.nonzero(np.isfinite(s[0].numpy()))[0])
        row = pr.ProcRow(z, T, top_k, top_p, min_p)
        if row.m_topp <= SAFETY:
            n_risk += 1
            assert abs(len(hf) - len(row.kept)) <= 1
        else:
            assert np.array_equal(hf, row.kept), (seed, len(hf), len(row.kept))
    assert n_risk <= 3


def test_min_p_error_model_covers_fp32():
    """An fp32 emulation of stage 2's weights (each __expf off by up to E(a) relative, flushed below 2^-126) makes the reference's min-p
    cut wherever the reference does not mark it at risk."""
    rng = np.random.default_rng(0)
    checked = 0
    for seed in range(200):
        z = pr.make_case("minp_boundary", 1000, seed)[0]
        row = pr.ProcRow(z, 1.0, 20, 1.0, 0.1)
        zs = row.zs.astype(np.float32)
        a = (zs.astype(np.float64) - np.float64(zs[0])).astype(np.float32)
        for _ in range(4):
            w = (np.exp(a.astype(np.float64)) * (1 + rng.uniform(-1, 1, len(a)) * sr._E(a))).astype(np.float32)
            w = np.where(w < np.float32(sr.FTZ), np.float32(0), w)
            drop = np.nonzero(w[1:row.c] < np.float32(0.1))[0]
            cut = 1 + int(drop[0]) if len(drop) else row.c
            if row.m_minp > SAFETY:
                assert cut == row.keep, seed
                checked += 1
    assert checked > 600


def test_variants_differ_on_their_family():
    """Each kernel-level variant changes a draw or the argmax, off risk, on its named family (prompt_in_set: see the HF loop test)."""
    settings = {"dup_twice": (1.3, 1.0, 20, 1.0, 0.0, 0, True), "penalty_after_T": (1.3, 0.6, 20, 1.0, 0.0, 0, False),
                "neg_divided": (1.3, 1.0, 20, 1.0, 0.0, 0, True), "min_new_le": (1.3, 1.0, 20, 1.0, 0.0, 2, True),
                "minp_raw_max": (1.3, 1.0, 20, 1.0, 0.1, 0, False), "minp_T1": (1.1, 0.6, 20, 1.0, 0.1, 0, False)}
    U = sr.grid_uniforms(64, 1)[:, 0].numpy()
    for variant, (theta, T, k, p, mp, m, greedy) in settings.items():
        n = 0
        for seed in range(4):
            z, ids, eos, _ = pr.make_case(pr.EXPOSED_BY[variant], 151936 if variant != "penalty_after_T" else 5000, seed, top_k=k,
                                          theta=theta, T=T)
            if greedy:
                for s in range(4):
                    n += pr.greedy_proc_ref(z, ids, theta, s, m, eos) != pr.greedy_proc_ref(z, ids, theta, s, m, eos, variant=variant)
            else:
                ref = pr.draw_proc_ref(z, ids, theta, 0, m, eos, T, k, p, mp, U)
                wrong = pr.draw_proc_ref(z, ids, theta, 0, m, eos, T, k, p, mp, U, variant=variant)
                n += int((~ref["at_risk"] & (ref["token"] != wrong["token"])).sum())
        assert n > 0, variant


def test_processed_families_are_mostly_off_risk():
    n = risk = 0
    for fam in pr.FAMILIES:
        for seed in range(3):
            z, ids, eos, _ = pr.make_case(fam, 12289, seed)
            d = pr.draw_proc_ref(z, ids, 1.3, 0, 0, eos, 0.6, 20, 0.95, 0.05, sr.grid_uniforms(32, 1)[:, 0].numpy())
            n += 32
            risk += int(d["at_risk"].sum())
    assert risk / n < 0.02, (risk, n)


# ------------------------------------------------------------------------------------------------------------------- against HF generate
def test_manual_loop_equals_hf_generate_greedy(tiny_oracle, golden):
    """The manual processed loop (HF's processor classes, embeds-only presence set) equals text_model.generate(inputs_embeds=...) with
    repetition_penalty and min_new_tokens, and with min_length (lowered by the embeds width); prompt_in_set does not."""
    D = golden["D"]
    cfg = tiny_oracle.text_config
    batch = D["batch"]
    P = batch["input_ids"].shape[1]
    eos = cfg.eos_token_id
    for theta, m in ((1.3, 4), (0.7, 2), (2.0, 6)):
        mine = pr.manual_processed_generate(tiny_oracle, batch, max_new_tokens=10, repetition_penalty=theta, min_new_tokens=m,
                                            eos_token_id=eos, pad_token_id=cfg.pad_token_id)
        hf = tiny_oracle.generate(**batch, max_new_tokens=10, do_sample=False, repetition_penalty=theta, min_new_tokens=m, eos_token_id=eos,
                                  pad_token_id=cfg.pad_token_id)
        assert torch.equal(mine, hf), (theta, m)
        hf_len = tiny_oracle.generate(**batch, max_new_tokens=10, do_sample=False, repetition_penalty=theta, min_length=P + m,
                                      eos_token_id=eos, pad_token_id=cfg.pad_token_id)
        assert torch.equal(mine, hf_len), (theta, m)
    wrong = pr.manual_processed_generate(tiny_oracle, batch, max_new_tokens=10, repetition_penalty=2.0, eos_token_id=eos,
                                         pad_token_id=cfg.pad_token_id, variant="prompt_in_set")
    hf = tiny_oracle.generate(**batch, max_new_tokens=10, do_sample=False, repetition_penalty=2.0, eos_token_id=eos,
                              pad_token_id=cfg.pad_token_id)
    assert not torch.equal(wrong[:, :hf.shape[1]], hf[:, :wrong.shape[1]])


# ------------------------------------------------------------------------------------------------------------------- arguments
def _cfg():
    from types import SimpleNamespace
    return SimpleNamespace(eos_token_id=7, pad_token_id=None)


def test_sampling_params_processors():
    from transformers import GenerationConfig
    from bioreason_b200.generation import SamplingParams
    p = SamplingParams.from_hf_kwargs(_cfg(), dict(max_new_tokens=5, do_sample=True, repetition_penalty=1.2, min_p=0.05, min_new_tokens=3))
    assert (p.repetition_penalty, p.min_p, p.min_new_tokens, p.num_return_sequences) == (1.2, 0.05, 3, 1)
    gc = GenerationConfig(max_new_tokens=9, do_sample=True, repetition_penalty=1.1, min_p=0.1, min_new_tokens=2, num_return_sequences=4)
    p = SamplingParams.from_hf_kwargs(_cfg(), dict(generation_config=gc))
    assert (p.repetition_penalty, p.min_p, p.min_new_tokens, p.num_return_sequences) == (1.1, 0.1, 2, 4)
    p = SamplingParams.from_hf_kwargs(_cfg(), dict(generation_config=gc, repetition_penalty=1.5, min_new_tokens=0))   # loose kwargs win
    assert (p.repetition_penalty, p.min_new_tokens) == (1.5, 0)
    # min_length: lowered by the prompt width P; min_new_tokens wins over it
    p = SamplingParams.from_hf_kwargs(_cfg(), dict(max_new_tokens=5, min_length=30), prompt_width=24)
    assert p.min_new_tokens == 6
    p = SamplingParams.from_hf_kwargs(_cfg(), dict(max_new_tokens=5, min_length=10), prompt_width=24)
    assert p.min_new_tokens == 0
    p = SamplingParams.from_hf_kwargs(_cfg(), dict(max_new_tokens=5, min_length=30, min_new_tokens=2), prompt_width=24)
    assert p.min_new_tokens == 2
    with pytest.raises(ValueError, match="num_return_sequences"):                                     # HF refuses n > 1 when greedy
        SamplingParams.from_hf_kwargs(_cfg(), dict(max_new_tokens=5, num_return_sequences=2))
    d = SamplingParams.from_hf_kwargs(_cfg(), {})
    assert (d.repetition_penalty, d.min_p, d.min_new_tokens, d.num_return_sequences, d.max_new_tokens) == (1.0, 0.0, 0, 1, 20)


@pytest.mark.parametrize("kw,what", [(dict(repetition_penalty=0.0), "repetition_penalty"), (dict(repetition_penalty=-1.0), "repetition_penalty"),
                                     (dict(min_p=1.5), "min_p"), (dict(min_p=-0.1), "min_p"), (dict(min_new_tokens=-1), "min_new_tokens"),
                                     (dict(min_length=-2), "min_length"), (dict(num_return_sequences=0), "num_return_sequences")])
def test_sampling_params_validation(kw, what):
    from bioreason_b200.generation import SamplingParams
    with pytest.raises(ValueError, match=what):
        SamplingParams.from_hf_kwargs(_cfg(), dict(max_new_tokens=4, **kw), prompt_width=8)


REFUSED = [("no_repeat_ngram_size", 3), ("bad_words_ids", [[5]]), ("suppress_tokens", [3]), ("begin_suppress_tokens", [3]),
           ("sequence_bias", {(5,): -1.0}), ("typical_p", 0.9), ("epsilon_cutoff", 1e-4), ("eta_cutoff", 1e-4), ("top_h", 0.5),
           ("num_beams", 2), ("penalty_alpha", 0.6), ("encoder_repetition_penalty", 1.2), ("forced_bos_token_id", 1),
           ("forced_eos_token_id", 2), ("guidance_scale", 1.5), ("stop_strings", ["x"]), ("output_scores", True), ("output_logits", True),
           ("return_dict_in_generate", True), ("max_time", 1.0), ("renormalize_logits", True)]


@pytest.mark.parametrize("name,value", REFUSED, ids=[n for n, _ in REFUSED])
def test_unbuilt_arguments_are_refused(name, value):
    from transformers import GenerationConfig
    from bioreason_b200.generation import SamplingParams
    with pytest.raises(NotImplementedError, match=name):
        SamplingParams.from_hf_kwargs(_cfg(), {"max_new_tokens": 4, name: value})
    with pytest.raises(NotImplementedError, match=name):
        SamplingParams.from_hf_kwargs(_cfg(), dict(max_new_tokens=4, generation_config=GenerationConfig(**{name: value})))


def test_call_arguments_and_max_length_are_refused():
    from transformers import LogitsProcessorList, StoppingCriteriaList
    from bioreason_b200.generation import SamplingParams
    for name in ("logits_processor", "stopping_criteria"):
        with pytest.raises(NotImplementedError, match=name):
            SamplingParams.from_hf_kwargs(_cfg(), {"max_new_tokens": 4, name: [object()]})
    SamplingParams.from_hf_kwargs(_cfg(), dict(max_new_tokens=4, logits_processor=LogitsProcessorList(), stopping_criteria=StoppingCriteriaList()))
    with pytest.raises(NotImplementedError, match="max_length"):
        SamplingParams.from_hf_kwargs(_cfg(), dict(max_length=40))
    SamplingParams.from_hf_kwargs(_cfg(), dict(max_length=40, max_new_tokens=4))                   # max_new_tokens wins, as in HF


def test_neutral_and_no_effect_arguments_pass():
    from transformers import GenerationConfig
    from bioreason_b200.generation import SamplingParams
    SamplingParams.from_hf_kwargs(_cfg(), dict(generation_config=GenerationConfig()))
    neutral = GenerationConfig._get_default_generation_params()
    neutral.pop("max_length")
    SamplingParams.from_hf_kwargs(_cfg(), dict(max_new_tokens=4, generation_config=GenerationConfig(**neutral), **neutral))
    p = SamplingParams.from_hf_kwargs(_cfg(), dict(max_new_tokens=4, use_cache=True, cache_implementation="static", bos_token_id=1,
                                                   num_beams=1, typical_p=1.0, output_attentions=False))
    assert p.max_new_tokens == 4
    # the trainer's kwargs, unchanged
    kw = dict(max_new_tokens=6, do_sample=True, temperature=0.6, top_p=0.95, top_k=20, pad_token_id=0, eos_token_id=7)
    p = SamplingParams.from_hf_kwargs(_cfg(), kw)
    assert (p.temperature, p.top_p, p.top_k, p.repetition_penalty, p.min_p, p.min_new_tokens) == (0.6, 0.95, 20, 1.0, 0.0, 0)


def test_num_return_sequences_expansion():
    from bioreason_b200.generation import detect_group_size, expand_return_sequences
    ids = torch.tensor([[1, 2, 3], [4, 5, 6]])
    am = torch.ones(2, 3, dtype=torch.long)
    dna = dict(input_ids=torch.tensor([[10, 11], [20, 21], [30, 31], [40, 41]]), attention_mask=torch.ones(4, 2, dtype=torch.long))
    bim = [0, 0, 1, 1]                                                  # two DNA sequences per row
    i2, a2, d2, b2 = expand_return_sequences(ids, am, dna, bim, 3)
    assert i2.tolist() == [[1, 2, 3]] * 3 + [[4, 5, 6]] * 3 and a2.shape == (6, 3)
    assert b2 == [0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5]
    assert d2["input_ids"][:, 0].tolist() == [10, 20] * 3 + [30, 40] * 3
    assert detect_group_size(i2, d2, b2).tolist() == [False, True, True, False, True, True]
    assert expand_return_sequences(ids, am, dna, bim, 1) == (ids, am, dna, bim)


def test_trainer_generation_kwargs():
    from bioreason_b200.trainer import DNALLMGRPOConfig
    assert DNALLMGRPOConfig().sampling_from_config is False
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "bioreason_b200", "trainer", "grpo_trainer.py")).read()
    assert "temperature=0.6, top_p=0.95, top_k=20" in src                # the flag off keeps the reference's hard-coded values
