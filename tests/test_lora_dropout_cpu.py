"""LoRA dropout on the CPU: the NumPy Philox against the Random123 known answers, the statistics of the mask, its independence of
row chunking, and the opt-in switches."""
import numpy as np
import pytest

from lora_dropout_ref import keep_mask, philox4x32_10, threshold


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(ctr, key, want):
    got = philox4x32_10(*[np.array([c], dtype=np.uint64) for c in ctr], *key)
    assert tuple(int(x[0]) for x in got) == want


@pytest.mark.parametrize("p", [0.05, 0.5])
def test_keep_fraction(p):
    T = threshold(p)
    m = keep_mask(1234, 7, 3, 2, np.arange(1000), 1280, T)                  # 1.28e6 elements
    n = m.size
    q = 1 - T / 65536
    sigma = np.sqrt(q * (1 - q) / n)
    assert abs(m.mean() - q) < 5 * sigma


def test_masks_of_different_streams_are_uncorrelated():
    T = threshold(0.5)
    base = keep_mask(99, 0, 0, 0, np.arange(400), 1024, T).ravel().astype(np.float64)
    for layer, proj, pass_id in ((1, 0, 0), (0, 1, 0), (0, 0, 1), (5, 6, 3)):
        other = keep_mask(99, pass_id, layer, proj, np.arange(400), 1024, T).ravel().astype(np.float64)
        r = np.corrcoef(base, other)[0, 1]
        assert abs(r) < 5 / np.sqrt(base.size), (layer, proj, pass_id, r)
        assert (base != other).mean() > 0.45
    assert (base != keep_mask(100, 0, 0, 0, np.arange(400), 1024, T).ravel()).mean() > 0.45        # the seed is the key


def test_row_slice_equals_the_full_pass_mask():
    T = threshold(0.05)
    full = keep_mask(5, 2, 4, 6, np.arange(3 * 77), 200, T)
    for lo, hi in ((0, 77), (77, 154), (100, 231), (230, 231)):
        assert np.array_equal(keep_mask(5, 2, 4, 6, np.arange(lo, hi), 200, T), full[lo:hi])


def test_set_dropout_range_and_threshold():
    from bioreason_b200.lora import LoraState
    st = object.__new__(LoraState)
    st.r = 32
    for bad in (-0.1, 1.0, 1.5, 0.99999999):
        with pytest.raises(ValueError):
            st.set_dropout(bad, seed=1)
    st.set_dropout(0.05, seed=3)
    assert st.dropout == (0.05, 3277, 3)
    st.set_dropout(0.0)
    assert st.dropout is None
    st.r = 8
    with pytest.raises(NotImplementedError):
        st.set_dropout(0.1)


def test_set_lora_dropout_needs_adapters():
    from bioreason_b200.models.dna_llm import DNALLMModel
    m = object.__new__(DNALLMModel)
    m._lora = None
    with pytest.raises(RuntimeError, match="enable_lora"):
        m.set_lora_dropout(0.05)
    assert m.new_lora_dropout_pass() is None


def test_config_default_is_off():
    from bioreason_b200.trainer import DNALLMGRPOConfig
    cfg = DNALLMGRPOConfig()
    assert cfg.apply_lora_dropout is False and cfg.lora_dropout == 0.05
