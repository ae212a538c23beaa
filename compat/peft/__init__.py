"""Stand-in for the `peft` entry points the reference's scripts call (reason.py:24,362-394,428-446; train_dna_qwen.py:136-177) when the
text model is a `bioreason_b200.DNALLMModel.text_model`.  peft itself is not needed (and not installed in this image): the adapters live
in the kernel layout of libbioreason_b200 (bioreason_b200/lora.py) under peft's own module / parameter names
(`<linear>.base_layer`, `<linear>.lora_A.default.weight`, `<linear>.lora_B.default.weight`), so state dicts keep their keys.

Put `compat/` on PYTHONPATH *instead of* peft only when training through bioreason_b200; it refuses any other model loudly."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Union

__all__ = ["LoraConfig", "get_peft_model", "prepare_model_for_kbit_training", "PeftModel", "TaskType"]


class TaskType:
    CAUSAL_LM = "CAUSAL_LM"


@dataclass
class LoraConfig:
    """Field names and defaults of peft.LoraConfig that the reference sets (reason.py:376-384)."""
    r: int = 8
    lora_alpha: int = 8
    lora_dropout: float = 0.0
    target_modules: Optional[Union[List[str], str]] = None
    init_lora_weights: Union[bool, str] = True
    bias: str = "none"
    task_type: Optional[str] = None
    modules_to_save: Optional[List[str]] = None
    inference_mode: bool = False
    extra: dict = field(default_factory=dict)


_KERNEL_TARGETS = {"q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj"}


def _owner(text_model):
    ref = getattr(text_model, "_b200_owner", None)
    owner = ref() if ref is not None else None
    if owner is None:
        raise TypeError("compat.peft only adapts the text_model of a bioreason_b200.DNALLMModel (use the real peft package for anything else)")
    return owner


def prepare_model_for_kbit_training(model, use_gradient_checkpointing: bool = True, gradient_checkpointing_kwargs=None):
    """reason.py:385: freezes the base weights (that is all it does for a bf16, non-quantised model)."""
    for p in model.parameters():
        p.requires_grad_(False)
    return model


def get_peft_model(model, peft_config: LoraConfig, adapter_name: str = "default", **kwargs):
    """reason.py:386 `model.text_model = get_peft_model(model.text_model, lora_config)`: every nn.Linear of the decoder named in
    `target_modules` gets rank-r adapters.  The kernels fuse q|k|v and gate|up, so the seven decoder projections are adapted together;
    a target list that leaves one of them out is refused rather than silently widened."""
    owner = _owner(model)
    targets = peft_config.target_modules
    if isinstance(targets, str):
        targets = [targets]
    if targets is not None:
        missing = _KERNEL_TARGETS - set(targets)
        if missing:
            raise NotImplementedError(f"LoRA on a subset of the decoder projections is not built (missing {sorted(missing)}); "
                                      "the reference adapts all of them (reason.py:83-113)")
    if peft_config.bias != "none":
        raise NotImplementedError("LoRA bias training is not on this path (the reference uses bias='none', reason.py:382)")
    if adapter_name != "default":
        raise NotImplementedError("one adapter named 'default'")
    owner.lora_dropout = float(peft_config.lora_dropout)       # recorded; the trainer applies it with DNALLMGRPOConfig.apply_lora_dropout
    owner.enable_lora(r=int(peft_config.r), alpha=float(peft_config.lora_alpha))
    return model


class PeftModel:
    """`PeftModel.from_pretrained(model.text_model, adapter_dir, is_trainable=True)` + `.merge_and_unload()` (reason.py:428-446)."""

    @staticmethod
    def from_pretrained(model, model_id, is_trainable: bool = False, **kwargs):
        owner = _owner(model)
        owner.load_checkpoint(model_id)                           # enables the adapters with the directory's rank / alpha
        model.active_adapter = "default"
        model.merge_and_unload = lambda: owner.merge_and_unload_lora() or model
        return model
