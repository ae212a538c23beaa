"""LoRA adapters for the Qwen3 decoder in kernel layout (peft is not installed in this image; SURVEY.md §8b).

`inject_lora` mirrors what the reference's callers do with peft (`reason.py:362-394`, `train_dna_qwen.py:136-177`):
every nn.Linear leaf of the text model except `lm_head` gets rank-r adapters (r=32, alpha=64, gaussian init:
A ~ N(0, 1/r), B = 0), base weights frozen.  Module / parameter names follow peft (`base_layer`,
`lora_A.default.weight`, `lora_B.default.weight`) so checkpoints keep their keys.  The fp32 master parameters are
what the optimizer sees; `LoraState.sync()` re-packs them (bf16, fused/blocked like the base weights, plus the
transposes the backward GEMMs read) after every optimizer step.

LoRA dropout is opt-in (`DNALLMModel.set_lora_dropout(p, seed)`; default p = 0, the undropped path).  When on, the training passes
compute peft's y = base(x) + s * B(A(dropout(x))) with one counter-based mask per projection, regenerated in the backward instead
of stored (rule next to br_lora_dropout in include/bioreason_b200.h).  It applies to the passes that train: the loss pass, the
old-log-prob pass when num_iterations > 1, the SFT step with backward and the autograd bridge.  It never applies to the
reference policy, to forward / per_token_logps, or to the rollout: the rollout samples from the merged, dropout-free policy
(W + s B A), whereas the reference trainer stays in train mode through generate and samples through the dropped adapters.
Dropout in decode would need unmerged adapters in the weight-streaming loop.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List

import torch
import torch.nn as nn

from . import ops
from .engine import LoraDropout, LoraLinearW, LoraW
from .packing import LINEARS, TARGETS, DecoderLayerW, DecoderW


class LoraLinear(nn.Module):
    """Container only (its forward is never on the product path): peft-shaped names around a frozen base Linear."""

    def __init__(self, base: nn.Linear, r: int, alpha: float, generator=None):
        super().__init__()
        self.base_layer = base
        base.weight.requires_grad_(False)
        dev = base.weight.device
        a = nn.Linear(base.in_features, r, bias=False, device=dev, dtype=torch.float32)
        b = nn.Linear(r, base.out_features, bias=False, device=dev, dtype=torch.float32)
        with torch.no_grad():
            a.weight.copy_(torch.randn(a.weight.shape, generator=generator, device="cpu").to(dev) / r)   # peft 'gaussian': std 1/r
            b.weight.zero_()
        self.lora_A = nn.ModuleDict({"default": a})
        self.lora_B = nn.ModuleDict({"default": b})
        self.r, self.lora_alpha, self.scaling = r, alpha, alpha / r

    @property
    def weight(self):
        return self.base_layer.weight

    def forward(self, x):                                                  # pragma: no cover - reference semantics only
        return self.base_layer(x) + self.lora_B["default"](self.lora_A["default"](x.float())).to(x.dtype) * self.scaling


@dataclass
class LoraFlat:
    params: List[nn.Parameter]
    flat_grad: torch.Tensor


class LoraState:
    def __init__(self, text_model, dec_w, r: int, alpha: float, seed: int = 0):
        self.r, self.scale = r, alpha / r
        cfg = text_model.config
        self.cfg = cfg
        g = torch.Generator().manual_seed(seed)
        self.modules: List[Dict[str, LoraLinear]] = []
        for layer in text_model.model.layers:
            mods = {}
            for f in LINEARS:
                parent = getattr(layer, f.parent)
                for n in f.targets:
                    lin = getattr(parent, n)
                    if not isinstance(lin, LoraLinear):
                        lin = LoraLinear(lin, r, alpha, g)
                        setattr(parent, n, lin)
                    mods[n] = lin
            self.modules.append(mods)
        for p in text_model.parameters():
            p.requires_grad_(False)
        self.params: List[nn.Parameter] = []
        for mods in self.modules:
            for n in TARGETS:
                for p in (mods[n].lora_A["default"].weight, mods[n].lora_B["default"].weight):
                    p.requires_grad_(True)
                    self.params.append(p)
        dev = dec_w.embed.device
        # one flat fp32 gradient buffer; every .grad is a contiguous view into it (single all-reduce bucket, C2)
        n = sum(p.numel() for p in self.params)
        self.flat_grad = torch.zeros(n, device=dev, dtype=torch.float32)
        off = 0
        self.grad_views: List[torch.Tensor] = []
        for p in self.params:
            self.grad_views.append(self.flat_grad[off:off + p.numel()].view_as(p))
            off += p.numel()
        self._alloc_packed(dev)
        self.sync()
        self.dropout = None                # (p, threshold T, seed) while LoRA dropout is on
        self.dropout_pass = 0              # pass counter c of the masks: advanced once per dropout-applying pass

    # ------------------------------------------------------------------
    def set_dropout(self, p: float, seed: int = 0):
        """p = 0 turns dropout off; 0 < p < 1 turns it on with T = round(p * 65536) (p_eff = T / 65536)."""
        p = float(p)
        if not 0.0 <= p < 1.0:
            raise ValueError(f"LoRA dropout must lie in [0, 1), got {p}")
        T = int(round(p * 65536))
        if T >= 65536:
            raise ValueError(f"LoRA dropout {p} rounds to p_eff = 1 at 16-bit resolution")
        if T > 0 and self.r not in (16, 32, 64):
            raise NotImplementedError(f"the LoRA dropout kernels are built for ranks 16, 32 and 64 (r = {self.r})")
        self.dropout = (p, T, int(seed)) if T > 0 else None

    def new_dropout_pass(self) -> int:
        pid = self.dropout_pass
        self.dropout_pass = (self.dropout_pass + 1) & 0xFFFFFFFF
        return pid

    def dropout_for(self, pass_id: int, row_offset: int) -> LoraDropout:
        _, T, seed = self.dropout
        return LoraDropout(seed=seed, pass_id=pass_id, threshold=T, row_offset=row_offset)

    # ------------------------------------------------------------------
    def _alloc_packed(self, dev):
        r = self.r
        z = lambda *s: torch.zeros(*s, device=dev, dtype=torch.bfloat16)
        self.w = LoraW(r=r, scale=self.scale, layers=[])
        for _ in self.modules:
            layer = {}
            for f in LINEARS:
                (N, K), n = f.shape(self.cfg), len(f.targets) * r
                layer[f.name] = LoraLinearW(a=z(n, K), b=z(N, n), a_T=z(K, n), b_T=z(n, N))
            self.w.layers.append(layer)

    @torch.no_grad()
    def sync(self):
        """fp32 masters -> bf16 kernel layout (+ transposes).  Off-block entries of the block-diagonal B stay zero."""
        r = self.r
        for mods, layer in zip(self.modules, self.w.layers):
            for f in LINEARS:
                ad = layer[f.name]
                for i, n in enumerate(f.targets):
                    ad.a[i * r:(i + 1) * r].copy_(mods[n].lora_A["default"].weight)
                    dst = f.block(ad.b, i, self.cfg)[..., i * r:(i + 1) * r]
                    dst.copy_(mods[n].lora_B["default"].weight.view(dst.shape))
                ad.a_T.copy_(ad.a.t())
                ad.b_T.copy_(ad.b.t())

    def zero_grad(self):
        self.flat_grad.zero_()

    def attach_grads(self):
        """Expose the flat buffer as the parameters' .grad (what a torch optimizer / DDP-style all-reduce consumes)."""
        for p, g in zip(self.params, self.grad_views):
            p.grad = g

    def layer_slice(self, layer: int):
        """[lo, hi) of the flat gradient buffer holding every adapter gradient of one decoder layer (parameters are laid out layer by layer)."""
        per = len(TARGETS) * 2
        lo = sum(g.numel() for g in self.grad_views[:layer * per])
        return lo, lo + sum(g.numel() for g in self.grad_views[layer * per:(layer + 1) * per])

    def grad_view(self, layer: int, name: str, which: str) -> torch.Tensor:
        idx = (layer * len(TARGETS) + TARGETS.index(name)) * 2 + (0 if which == "A" else 1)
        return self.grad_views[idx]


def _merge_into(dst, f, Lw, lora, i):
    """dst <- W + scale * B A of fused linear f of layer i (W alone without adapters), then the norm gain folded in where the input
    is normed."""
    base = getattr(Lw, f.name)
    if lora is not None:
        ad = lora.w.layers[i][f.name]
        # [N, K] = B[N, r'] @ (A^T)[K, r']^T ; K-major operands: A_op = B (K = r'), B_op = A^T ([K, r'])
        ops.gemm(ad.b, ad.a_T, alpha=lora.scale, residual=base, out=dst)
    else:
        dst.copy_(base)
    if f.norm is not None:
        ops.scale_columns_(dst, getattr(Lw, f.norm))


def _rollout_shell(dec_w, make):
    """DecoderW sharing the embedding, with its own final-norm-folded lm_head and per layer the matrices make(Lw, f) returns."""
    out = DecoderW(cfg=dec_w.cfg, embed=dec_w.embed, lm_head=torch.empty_like(dec_w.lm_head), final_norm=dec_w.final_norm)
    out.folded = True
    for Lw in dec_w.layers:
        out.layers.append(DecoderLayerW(ln1=Lw.ln1, ln2=Lw.ln2, q_norm=Lw.q_norm, k_norm=Lw.k_norm,
                                        **{f.name: make(Lw, f) for f in LINEARS}))
    out.lm_head.copy_(dec_w.lm_head)
    ops.scale_columns_(out.lm_head, dec_w.final_norm)                      # frozen: folded once
    return out


@torch.no_grad()
def build_rollout_weights(dec_w, lora: "LoraState | None", out=None):
    """Decode-time weights: W_eff = W + scale * B A per fused weight (the policy that rolls out is base + LoRA; merged with the
    wgmma GEMM, base weight as the epilogue residual), with the RMSNorm gains folded into the columns of the matrices that
    consume a normed input (w_qkv <- ln1, w_gu <- ln2, lm_head <- final norm) so the decode step needs no norm launches."""
    if out is None:
        # without adapters w_o / w_down need neither a merge nor a fold: the frozen base matrices are used as they are
        out = _rollout_shell(dec_w, lambda Lw, f: torch.empty_like(getattr(Lw, f.name)) if lora is not None or f.norm is not None
                             else getattr(Lw, f.name))
    for i, (Lw, Lo) in enumerate(zip(dec_w.layers, out.layers)):
        if lora is not None and any(getattr(Lo, f.name).data_ptr() == getattr(Lw, f.name).data_ptr() for f in LINEARS):
            raise RuntimeError("rollout weights alias the frozen base weights (built before enable_lora); rebuild them with out=None")
        for f in LINEARS:
            if lora is not None or f.norm is not None:
                _merge_into(getattr(Lo, f.name), f, Lw, lora, i)
    return out


@torch.no_grad()
def build_rollout_weights_fp8(dec_w, lora: "LoraState | None", out=None):
    """The decode weights of build_rollout_weights with the four layer matrices in weight-only FP8 (ops.Fp8Weight: e4m3 codes, one
    fp32 scale per output row); the embedding and the folded lm_head stay bf16.  Each matrix is merged and folded into one reusable
    bf16 scratch buffer (the largest matrix) and quantized from there, so no bf16 merged copy of the layers is kept."""
    if out is None:
        dev = dec_w.embed.device
        out = _rollout_shell(dec_w, lambda Lw, f: ops.fp8_weight_empty(*getattr(Lw, f.name).shape, dev))
        n_max = max(getattr(Lw, f.name).numel() for Lw in dec_w.layers for f in LINEARS)
        out.fp8_scratch = torch.empty(n_max, device=dev, dtype=torch.bfloat16)
    for i, (Lw, Lo) in enumerate(zip(dec_w.layers, out.layers)):
        for f in LINEARS:
            if lora is None and f.norm is None:
                ops.quantize_rows_e4m3(getattr(Lw, f.name), out=getattr(Lo, f.name))
            else:
                N, K = getattr(Lw, f.name).shape
                tmp = out.fp8_scratch[:N * K].view(N, K)
                _merge_into(tmp, f, Lw, lora, i)
                ops.quantize_rows_e4m3(tmp, out=getattr(Lo, f.name))
    return out
