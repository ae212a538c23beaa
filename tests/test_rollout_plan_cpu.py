"""Host-side rollout logic that needs no GPU: grouping detection, KV page plan, HF generation-kwargs parsing."""
import math

import pytest
import torch

from bioreason_b200.generation import PAGE, SamplingParams, detect_group_size, group_size_from_flags, plan_pages


@pytest.mark.parametrize("plen,G,C", [([1848], 8, 512), ([40], 4, 12), ([100, 230, 64], 1, 8), ([200, 330], 4, 70), ([63], 8, 1), ([64], 8, 1)])
def test_page_plan_invariants(plen, G, C):
    p = plan_pages(plen, G, C)
    U = len(plen)
    tab = p["table"]
    assert len(tab) == U * G and all(len(r) == p["max_pages"] for r in tab)
    assert p["n_shared"] == (min(l // PAGE for l in plen) if G > 1 else 0)
    used = set()
    for u in range(U):
        need = math.ceil((plen[u] + C) / PAGE)                     # pages a row needs for prompt + C generated tokens
        rows = [tab[u * G + g] for g in range(G)]
        for r in rows:
            assert r[:p["n_shared"]] == rows[0][:p["n_shared"]]    # shared prefix identical inside the group
            assert len(set(r[:need])) == need and max(r[:need]) < p["n_pages"]
        priv = [tuple(r[p["n_shared"]:need]) for r in rows]
        flat = [x for t in priv for x in t]
        assert len(flat) == len(set(flat))                         # private pages are never shared between rows
        shared = set(rows[0][:p["n_shared"]])
        assert not (shared & set(flat)) and not (shared & used) and not (set(flat) & used)
        used |= shared | set(flat)
        assert p["prefill_pages"][u] == rows[0][:math.ceil(plen[u] / PAGE)]
    assert used == set(range(p["n_pages"]))                         # no page leaked, none double-booked
    # tail copies: exactly the non-shared prompt pages of row 0, to the same table slot of every other row of the group
    want = [(tab[u * G][j], tab[u * G + g][j]) for u in range(U) for j in range(p["n_shared"], math.ceil(plen[u] / PAGE)) for g in range(1, G)]
    assert p["tail_copies"] == want


def test_group_detection():
    ids = torch.tensor([[1, 2, 3]] * 4 + [[4, 5, 6]] * 4)
    eq = detect_group_size(ids, None, [])
    assert eq.tolist() == [False, True, True, True, False, True, True, True]
    assert group_size_from_flags(eq.tolist()) == 4
    assert group_size_from_flags([False] * 6) == 1
    assert group_size_from_flags([False, True, True, True, True, True]) == 6
    assert group_size_from_flags([False, True, False, True, False, False]) == 1      # irregular -> no grouping
    # identical text but different DNA must not be grouped
    dna = dict(input_ids=torch.tensor([[3, 5], [3, 5], [3, 6], [3, 6]]), attention_mask=torch.ones(4, 2, dtype=torch.long))
    eq = detect_group_size(torch.tensor([[1, 2]] * 4), dna, [0, 1, 2, 3])
    assert eq.tolist() == [False, True, False, True]


def test_sampling_params_from_hf_kwargs():
    from types import SimpleNamespace
    from transformers import GenerationConfig
    cfg = SimpleNamespace(eos_token_id=7, pad_token_id=None)
    p = SamplingParams.from_hf_kwargs(cfg, dict(max_new_tokens=5, do_sample=True, temperature=0.6, top_p=0.95, top_k=20))
    assert (p.max_new_tokens, p.do_sample, p.temperature, p.top_p, p.top_k, p.eos_token_id, p.pad_token_id) == (5, True, 0.6, 0.95, 20, 7, 7)
    gc = GenerationConfig(max_new_tokens=9, do_sample=True, temperature=0.6, top_p=0.95, top_k=20, pad_token_id=3)   # grpo_trainer.py:384-391
    p = SamplingParams.from_hf_kwargs(cfg, dict(generation_config=gc))
    assert (p.max_new_tokens, p.do_sample, p.top_k, p.pad_token_id, p.eos_token_id) == (9, True, 20, 3, 7)
    p = SamplingParams.from_hf_kwargs(cfg, dict(generation_config=gc, max_new_tokens=4, eos_token_id=[11, 11]))   # loose kwargs win
    assert p.max_new_tokens == 4 and p.eos_token_id == 11
    import pytest
    with pytest.raises(NotImplementedError, match="distinct eos_token_id"):                                        # never silently keep eos[0]
        SamplingParams.from_hf_kwargs(cfg, dict(eos_token_id=[11, 12]))



@pytest.mark.parametrize("R,G,Hkv,n_shared,n_sms,want", [
    (8, 8, 8, 28, 132, (14, 3)),          # config (c): one prompt x G = 8, 1852-token prompt
    (32, 8, 8, 28, 132, (3, 1)),          # four groups: the shared splits halve to 7, then 3, then the private ones to 1
    (8, 1, 8, 0, 132, (0, 4)),            # no sharing: 8 private splits would be 512 items > 396
    (1, 1, 8, 0, 132, (0, 8)),
    (16, 16, 8, 2, 132, (2, 1)),          # 16 + 384 = 400 items > 396: the private splits halve to 1
    (4, 2, 8, 1, 132, (1, 3)),
    (64, 8, 8, 28, 132, (1, 1)),          # nothing left to halve: the kernel's own argument check refuses the launch
])
def test_decode_splits(R, G, Hkv, n_shared, n_sms, want):
    from bioreason_b200.generation import DECODE_ITEMS_PER_SM, decode_splits
    ss, sp = decode_splits(R, G, Hkv, n_shared, n_sms)
    assert (ss, sp) == want
    assert ss <= n_shared and (ss == 0) == (n_shared == 0) and 1 <= sp and ss + sp <= 32
    items = (R // G) * Hkv * ss + R * Hkv * sp
    assert items <= DECODE_ITEMS_PER_SM * n_sms or (ss <= 1 and sp == 1)
