"""Sequence-classification reward models on the GPU: br_seqcls_score against the float64 reference (tests/seqcls_ref.py), RewardModel
against HF's Qwen3ForSequenceClassification, and GRPO steps that score completions with reward models next to a text function."""
import copy

import pytest
import torch

from seqcls_ref import cases, hf_pooled_index, seqcls_ref
from reward_fixtures import make_reward_model, make_tokenizer, save_reward_dir

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------ kernel
def _check_kernel(d, n, B, L, pad_id, seed):
    from bioreason_b200 import ops
    h, ids, mask, nw, sw = cases(d, n, B, L, pad_id, seed=seed)
    ref = seqcls_ref(h, ids, pad_id, nw, 1e-6, sw)
    hc, idc, nwc, swc = h.cuda(), ids.cuda(), nw.cuda(), sw.cuda()
    out, idx = ops.seqcls_score(hc, idc, pad_id, nwc, 1e-6, swc, want_index=True)
    assert torch.equal(idx.cpu().long(), hf_pooled_index(ids, pad_id))
    err = (out.double().cpu() - ref["out"]).abs()
    assert (err <= ref["bound"]).all(), f"worst excess {(err - ref['bound']).max().item():.3e}"
    assert torch.equal(out, ops.seqcls_score(hc, idc, pad_id, nwc, 1e-6, swc))                 # same bits on every launch
    # through a strided output: columns [2, 2 + n) of a wider fp32 buffer, the rest untouched
    wide = torch.full((B, n + 4), 7.0, device="cuda")
    ops.seqcls_score(hc, idc, pad_id, nwc, 1e-6, swc, out=wide[:, 2:2 + n])
    assert torch.equal(wide[:, 2:2 + n], out) and (wide[:, :2] == 7).all() and (wide[:, 2 + n:] == 7).all()
    return (err > 0).float().mean().item()


@pytest.mark.parametrize("d", [256, 2048, 2560])
@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("B,L", [(1, 1), (1, 600), (8, 7), (8, 600), (33, 1), (33, 7), (33, 600)])
def test_kernel_against_float64(d, n, B, L):
    _check_kernel(d, n, B, L, 0, seed=d + 10 * n + B + L)


@pytest.mark.parametrize("pad_id", [None, 5])
def test_kernel_pad_edges(pad_id):
    """No pad id (B = 1: the last column), and a pad id that is a common token (pads in the middle of rows)."""
    for L in (1, 7, 600):
        _check_kernel(2048, 1, 1 if pad_id is None else 33, L, pad_id, seed=L)


# ------------------------------------------------------------------------------------------------------------ RewardModel vs HF
def _padded_batch(V, B, L, pad_id, side, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, V - 8, (B, L), generator=g)
    ids[ids == pad_id] = pad_id + 1
    mask = torch.zeros(B, L, dtype=torch.long)
    for r in range(B):
        n = L if r == 0 else int(torch.randint(1, L + 1, (1,), generator=g))
        sl = slice(0, n) if side == "right" else slice(L - n, L)
        mask[r, sl] = 1
    ids[mask == 0] = pad_id
    return ids, mask


def _hf_runs(model, ids, mask):
    """HF's fp32 forward (the oracle) and its bf16 forward of the same weights, on the GPU."""
    out = []
    for dt in (torch.float32, torch.bfloat16):
        m = copy.deepcopy(model).to(device="cuda", dtype=dt)
        with torch.no_grad():
            out.append(m(input_ids=ids.cuda(), attention_mask=mask.cuda()).logits.float())
        del m
    return out


def _assert_bar(ours, f32, b16, tag):
    e_mine, e_ref = (ours - f32).abs(), (b16 - f32).abs()
    print(f"{tag}: max|err| ours {e_mine.max():.4f} vs HF-bf16 {e_ref.max():.4f}; mean {e_mine.mean():.5f} vs {e_ref.mean():.5f}")
    assert e_mine.mean().item() <= 1.25 * e_ref.mean().item() + 1e-3
    assert e_mine.max().item() <= 1.25 * e_ref.max().item() + 2e-2


@pytest.mark.parametrize("name", ["tiny", "small"])
@pytest.mark.parametrize("side", ["right", "left"])
def test_reward_model_against_hf(name, side):
    from bioreason_b200.reward_model import RewardModel
    model = make_reward_model(name, seed=4)
    ids, mask = _padded_batch(model.config.vocab_size, 16, 45, model.config.pad_token_id, side, seed=7)
    f32, b16 = _hf_runs(model, ids, mask)
    rm = RewardModel(copy.deepcopy(model), "cuda")
    assert rm._dec.lm_head is None and rm._dec.layers[0].w_T is None
    ours = rm(ids, mask)
    assert ours.shape == (16, 1) and ours.dtype == torch.float32
    _assert_bar(ours, f32, b16, f"{name} {side}")
    assert torch.equal(ours, rm(ids.cuda(), mask.cuda()))


def test_reward_model_qwen3_1p7b_shape():
    """A Qwen3-1.7B-shaped reward model at B = 8, L = 600 (random init on the device; 28 layers)."""
    from transformers import Qwen3ForSequenceClassification
    from bioreason_b200.configs import text_config
    from bioreason_b200.reward_model import RewardModel
    cfg = text_config("qwen3-1.7b")
    cfg.num_labels = 1
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = Qwen3ForSequenceClassification(cfg).eval()
    ids, mask = _padded_batch(cfg.vocab_size, 8, 600, cfg.pad_token_id, "right", seed=3)
    f32, b16 = _hf_runs(model, ids, mask)
    before = torch.cuda.memory_allocated()
    rm = RewardModel(copy.deepcopy(model).to(torch.bfloat16), "cuda")
    resident = torch.cuda.memory_allocated() - before
    n_params = sum(p.numel() for p in model.parameters())
    del model
    _assert_bar(rm(ids, mask), f32, b16, "qwen3-1.7b B=8 L=600")
    print(f"resident {resident / 2 ** 30:.2f} GiB for {n_params / 1e9:.2f} B parameters")
    assert resident < 2.1 * n_params


# ------------------------------------------------------------------------------------------------------------ GRPO step
class WordTok:
    """The policy's processing class: token t decodes to the word w<t>; the EOS is dropped with skip_special_tokens."""

    def __init__(self, eos):
        self.eos_token_id = self.pad_token_id = eos

    def batch_decode(self, ids, skip_special_tokens=False):
        return [" ".join(f"w{t}" for t in row if not (skip_special_tokens and t == self.eos_token_id)) for row in ids.tolist()]


def text_fn(prompts, completions, **kw):
    return [0.1 * len(c.split()) for c in completions]


@pytest.mark.parametrize("extra", [{}, dict(share_prompt_prefix=True, fp8_rollout=True)], ids=["plain", "shared_fp8"])
def test_training_step_with_reward_models(tmp_path, monkeypatch, extra):
    from bioreason_b200 import dp
    from bioreason_b200.configs import dna_config, text_config
    from bioreason_b200.models import DNALLMModel
    from bioreason_b200.trainer import DNALLMGRPOConfig, DNALLMGRPOTrainer
    from bioreason_b200.trainer import rewards as rw
    from oracle import grpo as og
    from oracle.models import build_oracle, synth_batch
    tc, dc = text_config("tiny"), dna_config("tiny")
    m = DNALLMModel.from_oracle(build_oracle(tc, dc, seed=21))
    batch = synth_batch(tc, dc, batch=4, n_seq=2, dna_len=10, text_len=18, seed=14, same_prompt=True)
    batch["prompts"] = ["w3 w4 w5 "] * 4
    rm_dir = save_reward_dir(tmp_path / "org" / "rm-path", seed=1)
    rm_obj = make_reward_model(seed=2)
    rm_obj.config._name_or_path = "org/rm-object"
    hf = [copy.deepcopy(rm_obj)]
    tok = make_tokenizer()
    cfg = DNALLMGRPOConfig(num_generations=4, max_completion_length=6, per_device_train_batch_size=4, learning_rate=1e-3, lora_r=16,
                           lora_alpha=32.0, **extra)
    tr = DNALLMGRPOTrainer(m, [rm_dir, rm_obj, text_fn], cfg, processing_class=WordTok(tc.eos_token_id),
                           reward_processing_classes=[None, tok, None])
    assert [type(f).__name__ for f in tr.reward_funcs] == ["RewardModel", "RewardModel", "function"]
    seen = []
    gather = dp.gather_rewards
    monkeypatch.setattr(dp, "gather_rewards", lambda r: seen.append(r.clone()) or gather(r))
    inp = tr._generate_and_score_completions(batch, m, uniforms=torch.rand(6, 4, generator=torch.Generator().manual_seed(0)).cuda())
    rpf = seen[0]
    # the HF-scored rewards of the same texts
    comps = WordTok(tc.eos_token_id).batch_decode(inp["completion_ids"].cpu(), skip_special_tokens=True)
    texts = [p + c for p, c in zip(batch["prompts"], comps)]
    from transformers import AutoModelForSequenceClassification
    runs = []
    for model, t in ((AutoModelForSequenceClassification.from_pretrained(rm_dir, num_labels=1), tr.reward_processing_classes[0]), (hf[0], tok)):
        enc = t(texts, return_tensors="pt", padding=True, padding_side="right", add_special_tokens=False)
        runs.append(_hf_runs(model, enc["input_ids"], enc["attention_mask"]))
    f32, b16 = (torch.cat([r[k] for r in runs], 1) for k in (0, 1))
    _assert_bar(rpf[:, :2], f32, b16, "step reward-model columns")
    assert torch.allclose(rpf[:, 2].cpu(), torch.tensor(text_fn(None, comps)))
    torch.testing.assert_close(inp["advantages"].cpu(), og.group_advantages(rpf.cpu(), 4), rtol=1e-4, atol=1e-5)
    tr._step = 0
    loss = tr.training_step(inp)
    assert torch.isfinite(loss)
    met = tr.log_metrics()
    assert {"rewards/rm-path", "rewards/rm-object", "rewards/text_fn"} <= set(met)
    assert abs(met["rewards/rm-path"] - rpf[:, 0].mean().item()) < 1e-5
    assert isinstance(tr.reward_funcs[0], rw.RewardModel)
