"""Sequence-classification reward models on the CUDA decoder (the `PreTrainedModel` kind of the reference's reward functions,
bioreason/trainer/grpo_trainer.py:343-368, :655-666).

A Qwen3ForSequenceClassification is the policy's decoder trunk plus a [num_labels, d] score head read at one token per row, so its
forward is embed_gather -> engine.decoder_forward (without the final norm) -> br_seqcls_score, which norms and scores only the pooled
row.  The weights are packed once, bf16 on the device, with no transposed copies: the reward model is frozen and forward-only.
"""
from __future__ import annotations

import torch

from . import engine, ops
from .packing import _repoint, pack_decoder

SUPPORTED = ("Qwen3ForSequenceClassification",)


def check_contiguous_mask(attention_mask: torch.Tensor):
    """Raise ValueError unless every row of the 0/1 mask is one contiguous run of ones (the attention windows are [start, end))."""
    m = attention_mask != 0
    n = m.sum(1, keepdim=True)
    start = torch.where(m.any(1, keepdim=True), m.int().argmax(1, keepdim=True), torch.zeros_like(n))
    col = torch.arange(m.shape[1], device=m.device)[None, :]
    if not torch.equal(m, (col >= start) & (col < start + n)):
        raise ValueError("reward model: every attention-mask row must be one contiguous run of ones (left or right padding)")


class RewardModel:
    """One HF sequence classifier packed onto `device`.  `rm(input_ids, attention_mask)` returns the pooled logits, fp32
    [B, num_labels], as HF's forward(...).logits does, computed in bf16 like the policy.  The wrapped model's parameters are re-pointed
    to the packed bf16 storage (as DNALLMModel does for the policy); its config stays shared, so config.pad_token_id set later applies."""

    def __init__(self, model, device="cuda"):
        name = type(model).__name__
        if name not in SUPPORTED:
            raise NotImplementedError(f"reward model {name}: only {', '.join(SUPPORTED)} runs on the CUDA decoder "
                                      "(Qwen2 has a qkv bias and Llama no qk-norm; neither is implemented)")
        self.config = model.config
        self.num_labels = model.score.weight.shape[0]
        with torch.no_grad():
            self._dec = pack_decoder(model, device, lm_head=False)
            self.score_w = torch.empty(model.score.weight.shape, device=device, dtype=torch.bfloat16)
            _repoint(model.score.weight, self.score_w)
        self.device = self.score_w.device

    @torch.no_grad()
    def __call__(self, input_ids: torch.Tensor, attention_mask: torch.Tensor, out: torch.Tensor = None) -> torch.Tensor:
        """input_ids / attention_mask [B, L] (any device); out: optional fp32 [B, num_labels] device destination with contiguous rows."""
        B, L = input_ids.shape
        pad = self.config.pad_token_id
        if pad is None and B != 1:
            raise ValueError("Cannot handle batch sizes > 1 if no padding token is defined.")
        check_contiguous_mask(attention_mask)
        dev = self.device
        ids = input_ids.to(dev, torch.int64)
        mask = attention_mask.to(dev)
        h = ops.embed_gather(ids, self._dec.embed)
        # HF passes no position_ids: arange over the padded row
        h = engine.decoder_forward(self._dec, h, B, L, engine.forward_positions(B, L, dev), *engine.mask_window(mask), final_norm=False)
        return ops.seqcls_score(h, ids, pad, self._dec.final_norm, self.config.rms_norm_eps, self.score_w, out=out)
