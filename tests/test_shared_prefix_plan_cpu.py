"""The shared-prefix layout plan (training.plan_shared_prefix): host-side bookkeeping checked against the dense [B, L] layout it replaces."""
import pytest
import torch

from bioreason_b200 import engine
from bioreason_b200.training import plan_shared_prefix


def _batch(U, G, P, C, pads, eos=None, seed=0):
    """Dense rows [U*G, P + C]: group u's prompt left-padded by pads[u], then per-row completions (EOS-truncated by eos[r] if given).
    Returns (values [R, L] -- a distinct value per (group, prompt position) and per (row, completion position), attention mask)."""
    g = torch.Generator().manual_seed(seed)
    R, L = U * G, P + C
    vals = torch.empty(R, L, dtype=torch.long)
    mask = torch.zeros(R, L, dtype=torch.long)
    for u in range(U):
        prompt = torch.randint(1, 1 << 30, (P,), generator=g)
        for gg in range(G):
            r = u * G + gg
            vals[r, :P] = prompt
            vals[r, P:] = torch.randint(1, 1 << 30, (C,), generator=g)
            mask[r, pads[u]:P] = 1
            n_c = C if eos is None else eos[r]
            mask[r, P:P + n_c] = 1
    return vals, mask


def _check(U, G, P, C, pads, eos=None):
    vals, mask = _batch(U, G, P, C, pads, eos)
    R, L = vals.shape
    ks, ke = engine.mask_window(mask)
    plan = plan_shared_prefix(G, P, L, ks, ke)
    Lp = 64 * ((P - 1) // 64)
    if G == 1 or Lp == 0:
        assert plan is None
        return None
    assert plan.Lp == Lp and Lp % 64 == 0 and Lp <= P - 1 and plan.Ls == L - Lp
    assert plan.N == U * Lp + R * plan.Ls
    flat = vals.reshape(-1)
    buf = flat[plan.src.long()]                                            # what the shared token buffer holds
    dense_pos = torch.arange(L).repeat(R)
    assert torch.equal(plan.positions.long(), dense_pos[plan.src.long()])   # arange over the padded row, as the dense forward
    # every row, read back through the layout (prefix rows of its group, then its own suffix), is the dense row
    for r in range(R):
        u = r // G
        pre = buf[u * Lp:(u + 1) * Lp]
        suf = buf[U * Lp + r * plan.Ls:U * Lp + (r + 1) * plan.Ls]
        assert torch.equal(torch.cat([pre, suf]), vals[r])
        pos = torch.cat([plan.positions[u * Lp:(u + 1) * Lp], plan.positions[U * Lp + r * plan.Ls:U * Lp + (r + 1) * plan.Ls]])
        assert torch.equal(pos.long(), torch.arange(L))
    # windows: per group start (shared by its rows), per row end; each dense row's visible keys are unchanged
    assert torch.equal(plan.kv_start, ks[::G]) and torch.equal(plan.kv_end, ke)
    for r in range(R):
        assert int(ks[r]) == int(plan.kv_start[r // G])
        assert int(ke[r]) >= Lp                                             # prefix queries see prefix keys only
    # scored rows: positions P-1 .. L-2 of every row, all private, in the dense [B, L-P] order
    n = L - P
    dense_rows = (torch.arange(R)[:, None] * L + torch.arange(L - 1 - n, L - 1)[None, :]).reshape(-1)
    assert torch.equal(buf[plan.scored.long()], flat[dense_rows])
    assert (plan.scored.long() >= U * Lp).all()
    assert torch.equal(plan.positions[plan.scored.long()].long(), dense_pos[dense_rows])
    return plan, vals


def _dna_pairs(plan, U, G, P, L, slots):
    """DNA features at dense positions `slots` of every row (same positions for the G rows of a group): the (feature, buffer row) pairs
    owner_of gives versus those the dense layout implies."""
    R = U * G
    row_map = torch.tensor([r * L + t for r in range(R) for t in slots] + [-1], dtype=torch.int32)     # one DNA pad row
    dest = plan.owner_of(row_map)
    assert dest[-1] == -1
    pairs = {}
    for i, (dr, ds) in enumerate(zip(row_map.tolist(), dest.tolist())):
        if dr < 0:
            continue
        r, t = divmod(dr, L)
        if t < plan.Lp:                                                     # prefix: once per group, on the group's first row
            if r % G == 0:
                assert ds == (r // G) * plan.Lp + t
            else:
                assert ds == -1
        else:                                                               # tail: every row, in its own suffix
            assert ds == U * plan.Lp + r * plan.Ls + t - plan.Lp
        if ds >= 0:
            assert int(plan.src[ds]) in {dr, (r // G) * G * L + t}
            pairs.setdefault(ds, []).append(i)
    # the dense layout has one pair per (row, slot); the shared one keeps every tail pair and one prefix pair per group
    n_pre = sum(1 for t in slots if t < plan.Lp)
    n_tail = len(slots) - n_pre
    assert len(pairs) == U * n_pre + R * n_tail
    assert all(len(v) == 1 for v in pairs.values())


def test_prompt_multiple_of_64_keeps_last_prompt_position_private():
    plan, _ = _check(U=2, G=4, P=128, C=70, pads=[0, 5])
    assert plan.Lp == 64                                                   # not 128: position P - 1 = 127 is private


def test_short_prompt_has_no_sharing():
    for P in (1, 30, 64):
        _check(U=2, G=4, P=P, C=20, pads=[0, 0])
    assert _check(U=1, G=4, P=65, C=20, pads=[0]) is not None


def test_left_padding_longer_than_the_prefix():
    plan, _ = _check(U=2, G=2, P=200, C=90, pads=[195, 3], eos=[1, 90, 40, 7])
    assert plan.Lp == 192 and int(plan.kv_start[0]) == 195 and int(plan.kv_start[1]) == 3


def test_ragged_prompts_across_groups():
    # config (e)-like: prompt groups of different real lengths, left-padded to one width, EOS-truncated completions
    plan, _ = _check(U=4, G=2, P=1852, C=130, pads=[0, 700, 1500, 1791], eos=[130, 1, 64, 65, 2, 129, 33, 100])
    assert plan.Lp == 1792
    assert plan.kv_start.tolist() == [0, 700, 1500, 1791]


@pytest.mark.parametrize("G", [1, 2, 8, 16])
def test_group_sizes(G):
    U, P, C = 2, 300, 75
    out = _check(U=U, G=G, P=P, C=C, pads=[10, 0], eos=[(r * 7) % C + 1 for r in range(U * G)])
    if G == 1:
        assert out is None
        return
    plan, _ = out
    _dna_pairs(plan, U, G, P, P + C, slots=[10, 11, 63, 64, 255, 256, 270, 298])


def test_dna_pairs_in_prefix_and_tail():
    U, G, P, C = 3, 8, 1852, 64
    plan, _ = _check(U=U, G=G, P=P, C=C, pads=[0, 0, 12])
    _dna_pairs(plan, U, G, P, P + C, slots=list(range(100, 110)) + list(range(1785, 1800)) + [1851])
