"""Weight layout in HBM for the hot path.

The parameter *containers* stay HF-shaped (`Qwen3ForCausalLM`, `EsmForMaskedLM`: same module tree and
state_dict keys the reference's callers walk, SURVEY.md §8b) but their storage is re-pointed into fused
buffers laid out for the kernels:

  decoder layer : w_qkv [(Hq+2Hkv)*D, d]   rows = q heads | k heads | v heads       (one QKV GEMM)
                  w_gu  [2F, d]            blocks of 16 rows = 8 gate rows | 8 up rows (SwiGLU fused in the GEMM epilogue,
                                           16-byte-aligned gate/up column groups for the backward kernels)
                  w_o   [d, Hq*D], w_down [d, F]
  encoder layer : w_qkv [3*d, d] (+ b_qkv), w_o, w_gu [2F, d] interleaved (x1_j, x2_j), w_down
Frozen weights additionally get a transposed copy (`w_T`, [in, out]) so that the backward dX GEMMs are also
K-major x K-major (no MN-major descriptors); 180 GB of HBM makes the second copy (≈8 GB for Qwen3-4B) free.

`LINEARS` is the one description of the decoder's fused linears: which peft projections each stacks and where their rows sit.
Packing, the LoRA adapters' kernel layout, the forward and backward passes and the rollout merge all read it.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch


def proj_shape(cfg, target: str) -> Tuple[int, int]:
    """(out_features, in_features) of one Qwen3 decoder projection."""
    d, F, D = cfg.hidden_size, cfg.intermediate_size, cfg.head_dim
    q, kv = cfg.num_attention_heads * D, cfg.num_key_value_heads * D
    return {"q_proj": (q, d), "k_proj": (kv, d), "v_proj": (kv, d), "o_proj": (d, q),
            "gate_proj": (F, d), "up_proj": (F, d), "down_proj": (d, F)}[target]


@dataclass(frozen=True)
class FusedLinear:
    """One fused linear of a decoder layer.  Its LoRA adapters are packed the same way: A stacked by rows in target order
    ([n r, in]), B block-diagonal ([out, n r]: target i's rows, columns i r .. (i+1) r)."""
    name: str                    # the DecoderLayerW matrix
    parent: str                  # HF module holding the projections
    targets: Tuple[str, ...]     # peft targets, in packed order
    blocked: bool = False        # rows in blocks of 8 | 8 (gate | up, gu_views) instead of one consecutive range per target
    norm: Optional[str] = None   # DecoderLayerW norm gain folded into the columns of the decode copy (the input is RMS-normed)

    @property
    def proj0(self) -> int:
        """LoRA dropout projection id of the first target (its TARGETS index); target i is proj0 + i."""
        return TARGETS.index(self.targets[0])

    def rows(self, cfg) -> List[slice]:
        """Output rows of each target; a blocked linear interleaves its targets over all of its rows."""
        outs = [proj_shape(cfg, t)[0] for t in self.targets]
        if self.blocked:
            return [slice(0, sum(outs))] * len(outs)
        ends = [sum(outs[:i + 1]) for i in range(len(outs))]
        return [slice(e - n, e) for e, n in zip(ends, outs)]

    def shape(self, cfg) -> Tuple[int, int]:
        """(out, in) of the fused matrix."""
        return sum(proj_shape(cfg, t)[0] for t in self.targets), proj_shape(cfg, self.targets[0])[1]

    def block(self, w: torch.Tensor, i: int, cfg) -> torch.Tensor:
        """Target i's rows of a buffer laid out like this linear's output: [out_i, ...], or [out_i / 8, 8, ...] when blocked."""
        return gu_views(w)[i] if self.blocked else w[self.rows(cfg)[i]]


LINEARS = (
    FusedLinear("w_qkv", "self_attn", ("q_proj", "k_proj", "v_proj"), norm="ln1"),
    FusedLinear("w_o", "self_attn", ("o_proj",)),
    FusedLinear("w_gu", "mlp", ("gate_proj", "up_proj"), blocked=True, norm="ln2"),
    FusedLinear("w_down", "mlp", ("down_proj",)),
)
TARGETS = tuple(t for f in LINEARS for t in f.targets)     # LoRA dropout projection id = index; LoraState.params order


def gu_views(w_gu: torch.Tensor):
    """(gate, up) views [F/8, 8, ...] of a gate/up-blocked buffer whose leading dim is 2F (blocks of 8 gate | 8 up)."""
    F2 = w_gu.shape[0]
    v = w_gu.view(F2 // 16, 2, 8, *w_gu.shape[1:])
    return v[:, 0], v[:, 1]


def _repoint(param: torch.nn.Parameter, view: torch.Tensor):
    with torch.no_grad():
        view.copy_(param.data.to(view.dtype))
    param.data = view


@dataclass
class DecoderLayerW:
    ln1: torch.Tensor
    ln2: torch.Tensor
    q_norm: torch.Tensor
    k_norm: torch.Tensor
    w_qkv: torch.Tensor
    w_o: torch.Tensor
    w_gu: torch.Tensor
    w_down: torch.Tensor
    w_T: Optional[Dict[str, torch.Tensor]] = None     # transpose of each fused matrix, keyed by FusedLinear.name


@dataclass
class DecoderW:
    cfg: object
    embed: torch.Tensor            # [V, d] (tied lm_head)
    lm_head: Optional[torch.Tensor]   # [V, d]; None for a sequence classifier (RewardModel), which has a score head instead
    final_norm: torch.Tensor
    layers: List[DecoderLayerW] = field(default_factory=list)
    lm_head_T: Optional[torch.Tensor] = None   # [d, V] for dH = dlogits @ W

    def build_transposes(self):
        for L in self.layers:
            if L.w_T is None:
                L.w_T = {f.name: getattr(L, f.name).t().contiguous() for f in LINEARS}
        if self.lm_head_T is None:
            self.lm_head_T = self.lm_head.t().contiguous()


def pack_decoder(model, device="cuda", lm_head: bool = True) -> DecoderW:
    """Fuse a HF Qwen3ForCausalLM's weights into kernel layout (bf16, on `device`) and re-point its parameters.

    lm_head=False packs the trunk of a frozen forward-only model without an lm_head (Qwen3ForSequenceClassification): W.lm_head is
    None, and the container's gate / up parameters move to the host, so the kernel copy is the only device copy of them (about
    2 bytes per parameter resident)."""
    cfg = model.config
    d = cfg.hidden_size
    bf = torch.bfloat16
    emb_p = model.model.embed_tokens.weight
    embed = torch.empty(emb_p.shape, device=device, dtype=bf)
    _repoint(emb_p, embed)
    if not lm_head:
        lm_head = None
    elif cfg.tie_word_embeddings:
        model.lm_head.weight = model.model.embed_tokens.weight
        lm_head = embed
    else:
        lm_head = torch.empty(model.lm_head.weight.shape, device=device, dtype=bf)
        _repoint(model.lm_head.weight, lm_head)
    fn = torch.empty(d, device=device, dtype=bf)
    _repoint(model.model.norm.weight, fn)
    W = DecoderW(cfg=cfg, embed=embed, lm_head=lm_head, final_norm=fn)
    for layer in model.model.layers:
        mats = {}
        for f in LINEARS:
            w = mats[f.name] = torch.empty(f.shape(cfg), device=device, dtype=bf)
            for t, rows in zip(f.targets, f.rows(cfg)):
                p = getattr(getattr(layer, f.parent), t).weight
                if f.blocked:
                    # own storage: _copy_blocked fills the kernel copy.  Nothing re-derives a forward-only trunk's copy (lm_head=False), so
                    # its container keeps that storage on the host
                    p.data = p.data.to(device=device, dtype=bf) if lm_head is not None else p.data.to("cpu")
                else:
                    _repoint(p, w[rows])
        small = {}
        for name, p in (("ln1", layer.input_layernorm.weight), ("ln2", layer.post_attention_layernorm.weight),
                        ("q_norm", layer.self_attn.q_norm.weight), ("k_norm", layer.self_attn.k_norm.weight)):
            t = torch.empty(p.shape, device=device, dtype=bf)
            _repoint(p, t)
            small[name] = t
        W.layers.append(DecoderLayerW(**mats, **small))
        _copy_blocked(layer, W.layers[-1], cfg)
    # buffers (rotary inv_freq) are not used by the kernels; leave them where they are
    return W


def _copy_blocked(layer, Lw: DecoderLayerW, cfg):
    """Blocked kernel copies (gate/up) from the container's parameters.  A [F, d] parameter cannot alias the blocked layout as one
    strided view, so the container keeps its own (frozen) storage and refresh_decoder_gu re-derives the copy after a load."""
    with torch.no_grad():
        for f in LINEARS:
            if f.blocked:
                for i, t in enumerate(f.targets):
                    dst = f.block(getattr(Lw, f.name), i, cfg)
                    dst.copy_(getattr(getattr(layer, f.parent), t).weight.data.view(dst.shape))


def refresh_decoder_gu(model, W: DecoderW):
    """Re-derive the blocked gate/up kernel copies from the container's gate_proj / up_proj (after loading weights)."""
    for layer, Lw in zip(model.model.layers, W.layers):
        _copy_blocked(layer, Lw, W.cfg)
        Lw.w_T = None
    W.lm_head_T = None


@dataclass
class EncoderLayerW:
    ln1_w: torch.Tensor
    ln1_b: torch.Tensor
    ln2_w: torch.Tensor
    ln2_b: torch.Tensor
    w_qkv: torch.Tensor
    b_qkv: torch.Tensor
    w_o: torch.Tensor
    b_o: torch.Tensor
    w_gu: torch.Tensor           # gated: [2F, d] interleaved; plain GELU FFN is not on the NT-v2 path
    b_gu: Optional[torch.Tensor]
    w_down: torch.Tensor
    b_down: Optional[torch.Tensor]


@dataclass
class EncoderW:
    cfg: object
    embed: torch.Tensor
    final_ln_w: torch.Tensor
    final_ln_b: torch.Tensor
    layers: List[EncoderLayerW] = field(default_factory=list)


def pack_encoder(model, device="cuda") -> EncoderW:
    """Fuse a (NT-v2 patched) HF EsmForMaskedLM encoder into kernel layout; the MLM head is never packed (unused,
    SURVEY.md §8a A2: the reference computes it for nothing)."""
    cfg = model.config
    d, F = cfg.hidden_size, cfg.intermediate_size
    bf = torch.bfloat16
    if not getattr(cfg, "gated_mlp", False):
        raise NotImplementedError("only the NT-v2 gated-SiLU FFN encoder is on the hot path")
    if getattr(cfg, "position_embedding_type", "absolute") != "rotary" or cfg.emb_layer_norm_before or cfg.token_dropout:
        raise NotImplementedError("encoder kernels implement the NT-v2 configuration (rotary, no emb-LN-before, no token dropout)")

    def mv(p):
        t = torch.empty(p.shape, device=device, dtype=bf)
        _repoint(p, t)
        return t

    esm = model.esm
    W = EncoderW(cfg=cfg, embed=mv(esm.embeddings.word_embeddings.weight),
                 final_ln_w=mv(esm.encoder.emb_layer_norm_after.weight), final_ln_b=mv(esm.encoder.emb_layer_norm_after.bias))
    for layer in esm.encoder.layer:
        sa = layer.attention.self
        w_qkv = torch.empty(3 * d, d, device=device, dtype=bf)
        b_qkv = torch.empty(3 * d, device=device, dtype=bf)
        for i, lin in enumerate((sa.query, sa.key, sa.value)):
            _repoint(lin.weight, w_qkv[i * d:(i + 1) * d])
            _repoint(lin.bias, b_qkv[i * d:(i + 1) * d])
        w_gu = torch.empty(2 * F, d, device=device, dtype=bf)
        inter = layer.intermediate.dense                      # [2F, d]: rows [0,F) = x1 (gate), [F,2F) = x2
        gv, uv = gu_views(w_gu)
        with torch.no_grad():
            gv.copy_(inter.weight.data[:F].to(bf).view(F // 8, 8, d))
            uv.copy_(inter.weight.data[F:].to(bf).view(F // 8, 8, d))
        # the container keeps a [2F, d] parameter; give it its own bf16 storage (frozen, forward-only)
        inter.weight.data = inter.weight.data.to(device=device, dtype=bf)
        b_gu = None
        if inter.bias is not None:
            b_gu = torch.empty(2 * F, device=device, dtype=bf)
            with torch.no_grad():
                bg, bu = gu_views(b_gu)
                bg.copy_(inter.bias.data[:F].to(bf).view(F // 8, 8)); bu.copy_(inter.bias.data[F:].to(bf).view(F // 8, 8))
            inter.bias.data = inter.bias.data.to(device=device, dtype=bf)
        out = layer.output.dense
        W.layers.append(EncoderLayerW(
            ln1_w=mv(layer.attention.LayerNorm.weight), ln1_b=mv(layer.attention.LayerNorm.bias),
            ln2_w=mv(layer.LayerNorm.weight), ln2_b=mv(layer.LayerNorm.bias),
            w_qkv=w_qkv, b_qkv=b_qkv, w_o=mv(layer.attention.output.dense.weight), b_o=mv(layer.attention.output.dense.bias),
            w_gu=w_gu, b_gu=b_gu, w_down=mv(out.weight), b_down=mv(out.bias) if out.bias is not None else None))
    return W
