"""The decoder's fused-linear layout on the CPU: base weights, LoRA adapters and their transposes packed as packing.LINEARS describes,
checked against a restatement of the layout written out per projection here, plus the parameter order and peft names that
gradients, checkpoints and the all-reduce rely on, and merge_and_unload_lora."""
import types

import pytest
import torch

from bioreason_b200.configs import text_config
from bioreason_b200.lora import TARGETS, LoraLinear, LoraState
from bioreason_b200.models.dna_llm import DNALLMModel
from bioreason_b200.packing import LINEARS, pack_decoder

R = 16


def _fuse(cfg, name, parts):
    """Fused [N, ...] matrix of one linear from its per-projection row blocks: q | k | v stacked, gate / up in blocks of 8 | 8 rows."""
    if name == "w_gu":
        gate, up = parts
        F = gate.shape[0]
        return torch.stack([gate.view(F // 8, 8, -1), up.view(F // 8, 8, -1)], 1).reshape(2 * F, -1)
    return torch.cat(parts, 0)


PARENT = {"q_proj": "self_attn", "k_proj": "self_attn", "v_proj": "self_attn", "o_proj": "self_attn",
          "gate_proj": "mlp", "up_proj": "mlp", "down_proj": "mlp"}
GROUPS = {"w_qkv": ("q_proj", "k_proj", "v_proj"), "w_o": ("o_proj",), "w_gu": ("gate_proj", "up_proj"), "w_down": ("down_proj",)}


def _proj(layer, t):
    return getattr(getattr(layer, PARENT[t]), t)


@pytest.fixture(scope="module")
def packed():
    from transformers import Qwen3ForCausalLM
    torch.manual_seed(0)
    cfg = text_config("tiny")
    model = Qwen3ForCausalLM(cfg).to(torch.bfloat16)
    W = pack_decoder(model, "cpu")
    st = LoraState(model, W, r=R, alpha=2.0 * R, seed=0)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for p in st.params:
            p.copy_(torch.randn(p.shape, generator=g) * 0.1)             # B != 0
    st.sync()
    W.build_transposes()
    return cfg, model, W, st


def _base(layer, t):
    w = _proj(layer, t)
    return (w.base_layer if isinstance(w, LoraLinear) else w).weight.data


def test_targets_and_description():
    assert TARGETS == ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")
    assert tuple(f.name for f in LINEARS) == tuple(GROUPS)
    for f in LINEARS:
        assert f.targets == GROUPS[f.name] and all(PARENT[t] == f.parent for t in f.targets)
        assert f.proj0 == TARGETS.index(f.targets[0])
    assert {f.name: f.norm for f in LINEARS} == {"w_qkv": "ln1", "w_o": None, "w_gu": "ln2", "w_down": None}


def test_base_weights_at_their_rows(packed):
    cfg, model, W, _ = packed
    for layer, Lw in zip(model.model.layers, W.layers):
        for name, targets in GROUPS.items():
            w = getattr(Lw, name)
            assert torch.equal(w, _fuse(cfg, name, [_base(layer, t) for t in targets])), name
            assert torch.equal(Lw.w_T[name], w.t()) and Lw.w_T[name].is_contiguous()


def test_lora_blocks(packed):
    cfg, model, W, st = packed
    for li, mods in enumerate(st.modules):
        for name, targets in GROUPS.items():
            ad = st.w.layers[li][name]
            n = len(targets)
            A = [mods[t].lora_A["default"].weight.to(torch.bfloat16) for t in targets]
            B = [mods[t].lora_B["default"].weight.to(torch.bfloat16) for t in targets]
            assert torch.equal(ad.a, torch.cat(A, 0))
            # B block-diagonal: target i's rows, columns i r .. (i+1) r, zeros elsewhere
            Bcols = [torch.nn.functional.pad(b, (i * R, (n - 1 - i) * R)) for i, b in enumerate(B)]
            assert torch.equal(ad.b, _fuse(cfg, name, Bcols)), name
            ba = _fuse(cfg, name, [b.double() @ a.double() for a, b in zip(A, B)])
            torch.testing.assert_close(ad.b.double() @ ad.a.double(), ba, rtol=0, atol=1e-12)
            assert torch.equal(ad.a_T, ad.a.t()) and torch.equal(ad.b_T, ad.b.t())
            assert ad.a_T.is_contiguous() and ad.b_T.is_contiguous()


def test_param_order_and_names(packed):
    cfg, model, W, st = packed
    names = {id(p): n for n, p in model.named_parameters()}
    want = [f"model.layers.{li}.{PARENT[t]}.{t}.lora_{ab}.default.weight"
            for li in range(cfg.num_hidden_layers) for t in TARGETS for ab in "AB"]
    assert [names[id(p)] for p in st.params] == want
    assert all(p.shape[1] == R for p in st.params[1::2])
    assert [n for n, p in model.named_parameters() if p.requires_grad] == want
    all_names = set(names.values())
    assert all(f"model.layers.{li}.{PARENT[t]}.{t}.base_layer.weight" in all_names for li in range(cfg.num_hidden_layers) for t in TARGETS)


def test_merge_and_unload_covers_every_target_once():
    from transformers import Qwen3ForCausalLM
    torch.manual_seed(2)
    cfg = text_config("tiny")
    model = Qwen3ForCausalLM(cfg).to(torch.bfloat16)
    W = pack_decoder(model, "cpu")
    st = LoraState(model, W, r=R, alpha=2.0 * R, seed=0)
    with torch.no_grad():
        for p in st.params:
            p.normal_(0, 0.1)
    with torch.no_grad():                                                  # W + bf16(s B A), added in bf16
        want = {(li, t): st.modules[li][t].base_layer.weight + (st.scale * st.modules[li][t].lora_B["default"].weight
                                                                @ st.modules[li][t].lora_A["default"].weight).to(torch.bfloat16)
                for li in range(cfg.num_hidden_layers) for t in TARGETS}
    host = types.SimpleNamespace(_lora=st, text_model=model, _dec=W)
    DNALLMModel.merge_and_unload_lora(host)
    assert host._lora is None
    for li, layer in enumerate(model.model.layers):
        for t in TARGETS:
            lin = _proj(layer, t)
            assert type(lin) is torch.nn.Linear, t
            assert torch.equal(lin.weight.data, want[(li, t)]), t                # merged exactly once
        for name, targets in GROUPS.items():
            assert torch.equal(getattr(W.layers[li], name), _fuse(cfg, name, [want[(li, t)] for t in targets])), name
        assert W.layers[li].w_T is None
