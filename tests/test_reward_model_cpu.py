"""Reward models as reward functions, host side: the float64 reference of the pooled score head against HF's pooling rule and its
one-bug variants, and the plumbing of trainer/rewards.py (paths, tokenizers, texts, names) with the device work mocked."""
import pytest
import torch

from seqcls_ref import VARIANTS, bf16r, cases, hf_pooled_index, pooled_index, seqcls_ref
from reward_fixtures import make_reward_model, make_tokenizer, save_reward_dir

from bioreason_b200 import reward_model as rmod
from bioreason_b200.trainer import rewards as rw


# ------------------------------------------------------------------------------------------------------------ reference
def test_bf16_rounding_matches_torch():
    x = torch.randn(100000, dtype=torch.float32) * torch.exp(torch.randn(100000) * 4)
    assert torch.equal(bf16r(x.double()), x.to(torch.bfloat16).double())


@pytest.mark.parametrize("pad_id", [0, 7, None])
def test_pooled_index_is_hf(pad_id):
    g = torch.Generator().manual_seed(3)
    for L in (1, 2, 7, 33):
        B = 1 if pad_id is None else 40
        ids = torch.randint(0, 10, (B, L), generator=g)             # pads anywhere: in the middle, leading, trailing
        if pad_id is not None:
            ids[0] = pad_id                                         # all pad
            ids[1, : L // 2] = pad_id                               # left padding
            ids[2, L // 2:] = pad_id                                # right padding
        assert torch.equal(pooled_index(ids, pad_id), hf_pooled_index(ids, pad_id))
    if pad_id is None:
        with pytest.raises(ValueError, match="no padding token"):
            hf_pooled_index(torch.zeros(2, 3, dtype=torch.long), None)


def test_case_families_cover_the_edges():
    h, ids, mask, nw, sw = cases(256, 3, 33, 7, pad_id=0)
    idx = pooled_index(ids, 0)
    assert (ids == 0).all(1).any()                                  # an all-pad row
    assert ((ids[:, 0] == 0) & (ids[:, -1] != 0)).any()             # left padding
    assert (torch.where(mask.bool(), ids, 1) == 0).any()            # a pad id under mask 1
    assert (idx != torch.where(mask.bool(), torch.arange(7), -1).amax(1).clamp(min=0)).any()


def _caught(variant, d, n, B, L, pad_id, seed):
    h, ids, mask, nw, sw = cases(d, n, B, L, pad_id, seed=seed)
    ref = seqcls_ref(h, ids, pad_id, nw, 1e-6, sw)
    bad = seqcls_ref(h, ids, pad_id, nw, 1e-6, sw, attention_mask=mask, variant=variant)
    return bool((bad["index"] != hf_pooled_index(ids, pad_id)).any()) or bool(((bad["out"] - ref["out"]).abs() > ref["bound"]).any())


@pytest.mark.parametrize("variant", VARIANTS)
def test_one_bug_variants_are_caught(variant):
    assert all(_caught(variant, d, n, B, L, 0, seed) for d, n, B, L, seed in ((256, 1, 33, 7, 0), (2048, 3, 8, 600, 1)))


def test_bound_is_tight():
    """Most outputs have a zero bound: the kernel must reproduce the reference's bits there."""
    h, ids, mask, nw, sw = cases(2048, 3, 33, 7, 0)
    r = seqcls_ref(h, ids, 0, nw, 1e-6, sw)
    assert (r["bound"] == 0).float().mean() > 0.5
    assert torch.equal(r["index"], hf_pooled_index(ids, 0))


# ------------------------------------------------------------------------------------------------------------ plumbing
class FakeRM:
    """Stands in for RewardModel (which packs onto the GPU): records its inputs and returns the row's token count."""
    made = []

    def __init__(self, model, device="cuda"):
        self.model, self.device, self.config = model, device, model.config
        self.num_labels = model.config.num_labels
        self.calls = []
        FakeRM.made.append(self)

    def __call__(self, input_ids, attention_mask, out=None):
        self.calls.append((input_ids, attention_mask))
        v = attention_mask.float().sum(1, keepdim=True).repeat(1, self.num_labels) + torch.arange(self.num_labels)
        if out is None:
            return v
        out.copy_(v)
        return out


@pytest.fixture
def fake_rm(monkeypatch):
    FakeRM.made = []
    monkeypatch.setattr(rw, "RewardModel", FakeRM)
    return FakeRM


def text_reward(prompts, completions, **kw):
    return [float(len(c)) for c in completions]


def test_paths_and_models_resolve(tmp_path, fake_rm):
    d = save_reward_dir(tmp_path / "org" / "my-rm")
    obj = make_reward_model(seed=1)
    obj.config._name_or_path = d                                    # its tokenizer comes from there too
    funcs, procs = rw.resolve_reward_funcs([d, obj, text_reward], None, {"dtype": torch.float32}, "cpu")
    assert isinstance(funcs[0], FakeRM) and isinstance(funcs[1], FakeRM) and funcs[2] is text_reward
    assert type(funcs[0].model).__name__ == "Qwen3ForSequenceClassification" and funcs[0].model.config.num_labels == 1
    assert funcs[1].model is obj and procs[2] is None
    assert procs[0].pad_token_id == 2 and procs[1].pad_token_id == 2
    assert [rw.reward_func_name(f, i) for i, f in enumerate(funcs)] == ["my-rm", "my-rm", "text_reward"]
    assert rw.reward_func_name(lambda **kw: 0, 3) == "<lambda>"


def test_processing_classes_defaults_and_mismatch(tmp_path, fake_rm):
    d = save_reward_dir(tmp_path / "rm")
    with pytest.raises(ValueError, match="The number of reward processing classes must match the number of reward functions."):
        rw.resolve_reward_funcs([d, text_reward], [None], None, "cpu")
    tok = make_tokenizer()
    funcs, procs = rw.resolve_reward_funcs(d, tok, None, "cpu")               # neither is a list: both are wrapped
    assert len(funcs) == 1 and procs == [tok]


def test_pad_fallback_sets_config(tmp_path, fake_rm):
    d = save_reward_dir(tmp_path / "rm", pad=False)
    funcs, procs = rw.resolve_reward_funcs([d], None, None, "cpu")
    assert procs[0].pad_token == procs[0].eos_token == "<eos>"
    assert funcs[0].config.pad_token_id == procs[0].pad_token_id == 1


def test_callables_only_is_the_parent_path(monkeypatch):
    class Boom:
        def __init__(self, *a, **k):
            raise AssertionError("no reward model for callables")
    monkeypatch.setattr(rw, "RewardModel", Boom)
    funcs, procs = rw.resolve_reward_funcs(text_reward, None, None, "cpu")
    assert funcs == [text_reward] and procs == [None]
    ids = torch.tensor([[1, 2], [3, 9]])
    kw = dict(examples=[dict(prompt="a"), dict(prompt="b")], prompts=None, completion_ids=ids, completion_mask=torch.ones(2, 2),
              prompt_ids=ids, processing_class=_Dec())
    assert torch.equal(rw.score(funcs, **kw), rw.score(funcs, reward_processing_classes=procs, **kw))


class _Dec:
    def batch_decode(self, ids, skip_special_tokens=False):
        return [" ".join(f"w{t}" for t in row) for row in ids.tolist()]


@pytest.mark.parametrize("conversational", [False, True])
def test_model_texts_and_columns(fake_rm, conversational):
    tok = make_tokenizer()
    rm = FakeRM(make_reward_model())
    ids = torch.tensor([[1, 2, 3], [4, 5, 6], [7, 8, 9]])
    if conversational:
        prompts = [[{"role": "user", "content": f"w{10 + i}"}] for i in range(3)]
    else:
        prompts = ["w10 ", "w11 w12 ", "w13 "]
    examples = [dict(prompt=p, answer=i) for i, p in enumerate(prompts)]
    out = rw.score([text_reward, rm], examples=examples, prompts=None, completion_ids=ids, completion_mask=torch.ones(3, 3),
                   prompt_ids=ids, processing_class=_Dec(), reward_processing_classes=[None, tok])
    comps = _Dec().batch_decode(ids)
    if conversational:
        texts = [tok.apply_chat_template(p + [{"role": "assistant", "content": c}], tokenize=False) for p, c in zip(prompts, comps)]
        assert texts[0] == "<user> w10\n<assistant> w1 w2 w3\n"
    else:
        texts = [p + c for p, c in zip(prompts, comps)]
    want = tok(texts, return_tensors="pt", padding=True, padding_side="right", add_special_tokens=False)
    (got_ids, got_mask), = rm.calls
    assert torch.equal(got_ids, want["input_ids"]) and torch.equal(got_mask, want["attention_mask"])
    assert (got_mask[:, 0] == 1).all()                                                    # right padded
    assert out[:, 1].tolist() == want["attention_mask"].sum(1).float().tolist()
    assert out[:, 0].tolist() == ([1.0] * 3 if conversational else [8.0] * 3)              # the text function saw the same completions


def test_multi_label_model_scores_label_0(fake_rm):
    m = make_reward_model()
    m.config.num_labels = 3
    rm = FakeRM(m)
    out = rw.score([rm], examples=[dict(prompt="w1 ")], prompts=None, completion_ids=torch.tensor([[1, 2]]),
                   completion_mask=torch.ones(1, 2), prompt_ids=torch.ones(1, 1), processing_class=_Dec(),
                   reward_processing_classes=[make_tokenizer()])
    assert out.tolist() == [[3.0]]


def test_model_without_prompts_or_tokenizer_fails_loudly(fake_rm):
    rm = FakeRM(make_reward_model())
    kw = dict(completion_ids=torch.tensor([[1, 2]]), completion_mask=torch.ones(1, 2), prompt_ids=torch.ones(1, 1), processing_class=_Dec())
    with pytest.raises(ValueError, match="prompts"):
        rw.score([rm], examples=None, prompts=None, reward_processing_classes=[make_tokenizer()], **kw)
    with pytest.raises(ValueError, match="processing class"):
        rw.score([rm], examples=[dict(prompt="w1")], prompts=None, **kw)


# ------------------------------------------------------------------------------------------------------------ refusals
def test_non_qwen3_architectures_are_refused():
    from transformers import LlamaConfig, LlamaForSequenceClassification, Qwen2Config, Qwen2ForSequenceClassification
    small = dict(hidden_size=64, intermediate_size=128, num_hidden_layers=1, num_attention_heads=2, num_key_value_heads=1, vocab_size=32)
    for cls, cfg in ((LlamaForSequenceClassification, LlamaConfig(**small)), (Qwen2ForSequenceClassification, Qwen2Config(**small))):
        with pytest.raises(NotImplementedError, match=cls.__name__):
            rmod.RewardModel(cls(cfg), "cpu")


def test_call_refusals():
    rm = object.__new__(rmod.RewardModel)
    rm.config = make_reward_model().config
    rm.config.pad_token_id = None
    with pytest.raises(ValueError, match="no padding token"):
        rm(torch.ones(2, 3, dtype=torch.long), torch.ones(2, 3))
    rmod.check_contiguous_mask(torch.tensor([[1, 1, 0], [0, 1, 1], [0, 0, 0], [0, 1, 0]]))
    with pytest.raises(ValueError, match="contiguous"):
        rmod.check_contiguous_mask(torch.tensor([[1, 0, 1]]))
    rm.config.pad_token_id = 2
    with pytest.raises(ValueError, match="contiguous"):
        rm(torch.ones(1, 4, dtype=torch.long), torch.tensor([[0, 1, 0, 1]]))
