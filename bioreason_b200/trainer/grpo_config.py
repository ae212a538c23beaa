"""`DNALLMGRPOConfig` -- field names and defaults of bioreason/trainer/grpo_config.py:22-364 that the hot path reads.

The reference subclasses HF `TrainingArguments` (which needs `accelerate`, absent here); this is a plain dataclass with
the same names so scripts that build the config by keyword keep working.  vLLM fields (`grpo_config.py:231-281`) are
accepted and ignored exactly as the reference trainer ignores them.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Optional, Union


@dataclass
class DNALLMGRPOConfig:
    output_dir: str = "grpo_out"
    # data / generation (grpo_config.py:146-228)
    model_init_kwargs: Optional[dict] = None
    remove_unused_columns: Optional[bool] = False
    max_prompt_length: Optional[int] = 512
    num_generations: Optional[int] = 8
    max_completion_length: Optional[int] = 800
    ds3_gather_for_generation: bool = True
    temperature: float = 0.6      # NOTE: the reference trainer hard-codes T=0.6 / top_p=0.95 / top_k=20 (grpo_trainer.py:384-391)
    top_p: float = 0.95
    top_k: Optional[int] = 20
    min_p: Optional[float] = None
    repetition_penalty: float = 1.0
    cache_implementation: Optional[str] = None
    # vLLM (never read by the reference trainer)
    use_vllm: Optional[bool] = False
    vllm_device: Optional[str] = "auto"
    vllm_gpu_memory_utilization: float = 0.9
    vllm_dtype: Optional[str] = "auto"
    vllm_max_model_len: Optional[int] = None
    vllm_enable_prefix_caching: Optional[bool] = True
    vllm_guided_decoding_regex: Optional[str] = None
    # optimisation (grpo_config.py:284-340)
    learning_rate: float = 1e-6
    beta: float = 0.04
    num_iterations: int = 1
    epsilon: float = 0.2
    epsilon_high: Optional[float] = None
    reward_weights: Optional[list] = None
    sync_ref_model: bool = False
    ref_model_mixup_alpha: float = 0.6
    ref_model_sync_steps: int = 512
    log_completions: bool = True
    report_to: Union[None, str, list] = "none"
    logging_first_step: bool = False
    logging_steps: float = 2
    # the TrainingArguments fields the trainer touches
    per_device_train_batch_size: int = 8
    per_device_eval_batch_size: int = 8
    gradient_accumulation_steps: int = 1
    max_steps: int = -1
    num_train_epochs: float = 1.0
    weight_decay: float = 0.0
    adam_beta1: float = 0.9
    adam_beta2: float = 0.999
    adam_epsilon: float = 1e-8
    max_grad_norm: float = 1.0
    seed: int = 42
    bf16: bool = True
    gradient_checkpointing: bool = False
    eval_strategy: str = "no"
    save_steps: int = 0                   # > 0: fire the callbacks' on_save every save_steps optimizer steps (HF save_strategy="steps")
    save_safetensors: bool = False        # reason.py:597 sets it; saving itself is the callbacks' job (reason.py:46-81)
    lora_dropout: float = 0.05            # the rate apply_lora_dropout uses when compat.peft recorded none
    apply_lora_dropout: bool = False      # train through LoRA dropout (off: the undropped path, bit-identical to before)
    # additions of this implementation
    lora_r: int = 32
    lora_alpha: float = 64.0
    micro_rows: Optional[int] = None      # rows per forward/backward chunk (None = as many as the device memory holds)
    suppress_eos: bool = False            # fixed-length rollouts (bench config c)
    share_prompt_prefix: bool = False     # ref / old / policy passes compute each prompt group's full prompt tiles once (same log-probs)
    fp8_rollout: bool = False             # rollout decode streams e4m3 layer weights (per-row scales); samples from the quantized policy
    rollout_is_correction: bool = False   # weight each token's policy-gradient term by min(exp(old - rollout logp), rollout_is_cap)
    rollout_is_cap: float = 2.0           # truncation of that importance weight (> 0; inf: untruncated)
    sampling_from_config: bool = False    # rollout takes temperature / top_p / top_k / min_p / repetition_penalty from this config (later
                                          # TRL releases); off: the reference's hard-coded T = 0.6, top_p = 0.95, top_k = 20
    top_entropy_quantile: float = 1.0     # keep the policy-gradient term on the top rho fraction of completion tokens by entropy, over
                                          # all ranks per loss call (TRL; "Beyond the 80/20 Rule"); 1.0: off
    log_entropy: bool = False             # log the policy's mean token entropy (`entropy`) without masking
    # the objectives of later TRL releases (DESIGN.md §3); the defaults are the reference's objective
    loss_type: str = "grpo"               # "grpo": per-row token means, then the mean over rows; "bnpo": token mean over the local batch;
                                          # "dr_grpo": token sum / (rows * max_completion_length); "dapo": token sum / (N / world), N the
                                          # completion tokens of the micro-step over all ranks (TRL's num_items_in_batch)
    importance_sampling_level: str = "token"   # "token"; "sequence": one ratio per row, exp(masked mean of lp - old) (GSPO)
    delta: Optional[float] = None         # > 0: coef_1 <- min(coef_1, delta), two-sided clipping (INTELLECT-2); None: off
    scale_rewards: str = "group"          # advantage divisor: "group" std, "batch" std, or "none"; True / False mean "group" / "none"
    mask_truncated_completions: bool = False   # completions without EOS carry no loss (DAPO); not with suppress_eos

    def __post_init__(self):
        if isinstance(self.scale_rewards, bool) or str(self.scale_rewards).lower() in ("true", "false"):
            self.scale_rewards = "group" if str(self.scale_rewards).lower() == "true" else "none"
        if self.scale_rewards not in ("group", "batch", "none"):
            raise ValueError(f"scale_rewards must be 'group', 'batch' or 'none' (or a bool), got {self.scale_rewards!r}")
        if self.loss_type not in ("grpo", "bnpo", "dr_grpo", "dapo"):
            raise ValueError(f"loss_type must be 'grpo', 'bnpo', 'dr_grpo' or 'dapo', got {self.loss_type!r}")
        if self.importance_sampling_level not in ("token", "sequence"):
            raise ValueError(f"importance_sampling_level must be 'token' or 'sequence', got {self.importance_sampling_level!r}")
        if self.delta is not None and not (isinstance(self.delta, (int, float)) and not isinstance(self.delta, bool)
                                           and math.isfinite(self.delta) and self.delta > 0):
            raise ValueError(f"delta must be None or a finite value > 0, got {self.delta!r}")
        if self.mask_truncated_completions and self.suppress_eos:
            raise ValueError("mask_truncated_completions with suppress_eos masks every completion: there would be nothing to train on")
        if not (0.0 <= self.top_entropy_quantile <= 1.0):
            raise ValueError(f"top_entropy_quantile must lie in [0, 1] (1.0: off), got {self.top_entropy_quantile}")
        if not (self.rollout_is_cap > 0):
            raise ValueError(f"rollout_is_cap must be > 0 (inf for untruncated importance sampling), got {self.rollout_is_cap}")
