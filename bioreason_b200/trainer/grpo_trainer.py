"""CUDA-native `DNALLMGRPOTrainer`: the tensor math of bioreason/trainer/grpo_trainer.py on libbioreason_b200.

Kept from the reference: `RepeatRandomSampler` semantics (:72-119), the rollout with the hard-coded sampling config
(:384-391), EOS-inclusive completion mask (:605-609), ref log-probs with the frozen reference policy, old log-probs only
when num_iterations > 1 (:617-640), all-gather of rewards then group-normalised advantages with unbiased std and +1e-4
(:679-699), the clipped-ratio + beta*k3-KL loss with per-row masked mean (:786-812), the metric names (:703-716, :803, :812).
Re-designed: one fused lm_head+log-softmax+gather kernel instead of [B, L, V] logits; rollout on the paged-KV decode
engine with the G samples sharing one prefill; hand-written backward; one flat NCCL all-reduce of the LoRA+projector
gradients (SURVEY.md §8e C1/C2).  Not HF-Trainer based (accelerate/trl/peft are not installed in this image).
"""
from __future__ import annotations

import time
from collections import defaultdict
from typing import Any, Callable, Dict, List, Optional, Sized, Union

import torch
import torch.distributed as dist
from torch.utils.data import Sampler

from .. import dp, generation, ops, training
from . import rewards as rw
from .grpo_config import DNALLMGRPOConfig


class RepeatRandomSampler(Sampler):
    """grpo_trainer.py:72-119 -- each index repeated `mini_repeat_count` times, chunks of `batch_size` unique indices,
    the whole chunk repeated `repeat_count` times; same seed on every rank."""

    def __init__(self, data_source: Sized, mini_repeat_count: int, batch_size: int = 1, repeat_count: int = 1, seed: Optional[int] = None):
        self.data_source, self.mini_repeat_count, self.batch_size, self.repeat_count = data_source, mini_repeat_count, batch_size, repeat_count
        self.num_samples = len(data_source)
        self.seed = seed
        self.generator = torch.Generator()
        if seed is not None:
            self.generator.manual_seed(seed)

    def __iter__(self):
        indexes = torch.randperm(self.num_samples, generator=self.generator).tolist()
        indexes = [indexes[i:i + self.batch_size] for i in range(0, len(indexes), self.batch_size)]
        indexes = [chunk for chunk in indexes if len(chunk) == self.batch_size]
        for chunk in indexes:
            for _ in range(self.repeat_count):
                for index in chunk:
                    for _ in range(self.mini_repeat_count):
                        yield index

    def __len__(self) -> int:
        return self.num_samples * self.mini_repeat_count * self.repeat_count


def _world():
    return (dist.get_rank(), dist.get_world_size()) if dist.is_available() and dist.is_initialized() else (0, 1)


class TrainerState:
    """The fields of transformers.TrainerState that callbacks on this path read (reason.py:46-81 uses global_step)."""

    def __init__(self):
        self.global_step, self.epoch, self.max_steps = 0, 0.0, 0
        self.log_history: List[Dict[str, float]] = []
        self.is_world_process_zero = _world()[0] == 0
        self.is_local_process_zero = self.is_world_process_zero


class TrainerControl:
    def __init__(self):
        self.should_save = self.should_log = self.should_training_stop = self.should_evaluate = self.should_epoch_stop = False


class CallbackHandler:
    """Duck-typed transformers.TrainerCallback dispatch: event(args, state, control, model=, processing_class=, optimizer=, ...);
    a callback may return a (modified) control object."""

    def __init__(self, callbacks, trainer):
        self.callbacks, self.trainer = list(callbacks or []), trainer

    def fire(self, event: str, **extra):
        tr = self.trainer
        for cb in self.callbacks:
            fn = getattr(cb, event, None)
            if fn is None:
                continue
            out = fn(tr.args, tr.state, tr.control, model=tr.model, processing_class=tr.processing_class, tokenizer=tr.processing_class,
                     optimizer=tr.optimizer, train_dataloader=None, eval_dataloader=None, **extra)
            if out is not None:
                tr.control = out
        return tr.control


class DNALLMGRPOTrainer:
    def __init__(self, model, reward_funcs: Union[Callable, List[Callable]], args: Optional[DNALLMGRPOConfig] = None, dna_module=None,
                 train_dataset=None, eval_dataset=None, processing_class=None, reward_processing_classes=None, callbacks=None,
                 optimizers=(None, None), peft_config=None, freeze_dna_modules: bool = False, attn_implementation: str = "flash_attention_2",
                 torch_dtype: str = "bfloat16", **kwargs):
        assert not isinstance(model, str), "model must be a DNALLMModel instance"             # grpo_trainer.py:241
        self.model, self.args = model, args or DNALLMGRPOConfig()
        a = self.args
        self.dna_module, self.processing_class = dna_module, processing_class
        self.train_dataset, self.eval_dataset = train_dataset, eval_dataset
        self.num_generations, self.max_completion_length = a.num_generations, a.max_completion_length
        self.beta, self.num_iterations = a.beta, a.num_iterations
        self.epsilon_low = a.epsilon
        self.epsilon_high = a.epsilon_high if a.epsilon_high is not None else a.epsilon
        rank, world = _world()
        global_bs = a.per_device_train_batch_size * world
        possible = [n for n in range(2, global_bs + 1) if global_bs % n == 0]
        if self.num_generations not in possible:                                            # grpo_trainer.py:428-436
            raise ValueError(f"The global train batch size ({world} x {a.per_device_train_batch_size}) must be evenly divisible by the "
                             f"number of generations per prompt ({self.num_generations}). Given the current train batch size, the valid "
                             f"values for the number of generations are: {possible}.")
        if getattr(a, "share_prompt_prefix", False) and a.apply_lora_dropout:
            raise ValueError("share_prompt_prefix cannot be combined with apply_lora_dropout: the dropout masks differ between the G copies "
                             "of a prompt, so the prompt cannot be computed once")
        # reward models (paths or sequence classifiers) are packed next to the policy now, so an unsupported one fails before any step
        self.reward_funcs, self.reward_processing_classes = rw.resolve_reward_funcs(reward_funcs, reward_processing_classes,
                                                                                    a.model_init_kwargs, model._dec.embed.device)
        if model._lora is None:
            model.enable_lora(r=a.lora_r, alpha=a.lora_alpha, seed=a.seed)
        # each rank quantizes its own (identical) merged weights; the quantizer is deterministic, so the ranks agree
        model.set_fp8_rollout(getattr(a, "fp8_rollout", False))
        model.sync_adapters(rollout=True)
        if a.apply_lora_dropout:                                            # peft's rate; per-rank masks (set_seed(device_specific=True))
            p = getattr(model, "lora_dropout", None)
            model.set_lora_dropout(a.lora_dropout if p is None else p, seed=a.seed + rank)
        self.eos_token_id = getattr(processing_class, "eos_token_id", None) if processing_class is not None else None
        if self.eos_token_id is None:
            self.eos_token_id = model.text_config.eos_token_id
        self.pad_token_id = getattr(processing_class, "pad_token_id", None) if processing_class is not None else None
        if self.pad_token_id is None:
            self.pad_token_id = model.text_config.pad_token_id
        # hard-coded exactly like grpo_trainer.py:384-391 (args.temperature/top_p/top_k are NOT consulted there either)
        self.generation_kwargs = dict(max_new_tokens=self.max_completion_length, do_sample=True, temperature=0.6, top_p=0.95, top_k=20,
                                      pad_token_id=self.pad_token_id, eos_token_id=None if a.suppress_eos else self.eos_token_id)
        if getattr(a, "sampling_from_config", False):
            # later TRL releases read the sampling fields of the config (min_p None: off, as in HF)
            self.generation_kwargs.update(temperature=a.temperature, top_p=a.top_p, top_k=a.top_k, min_p=a.min_p,
                                          repetition_penalty=a.repetition_penalty)
        if getattr(a, "rollout_is_correction", False):
            # the sampler's own log-probs of the tokens it drew (behaviour policy: merged / FP8 decode weights) for the IS weights
            self.generation_kwargs["return_logprobs"] = True
        opt = optimizers[0]
        if opt is None:
            opt = torch.optim.AdamW(model.trainable_parameters(), lr=a.learning_rate, betas=(a.adam_beta1, a.adam_beta2), eps=a.adam_epsilon,
                                    weight_decay=a.weight_decay, fused=True)
        self.optimizer = opt
        self._metrics = defaultdict(list)
        self._buffered_inputs = [None] * a.gradient_accumulation_steps
        self._step = 0
        self.state, self.control = TrainerState(), TrainerControl()
        self.state.max_steps = a.max_steps
        self.callback_handler = CallbackHandler(callbacks, self)
        self.reward_d2h_bytes = 0          # bytes of completion ids copied to the host for text reward functions (last step)
        # per-rank distinct sampling stream (set_seed(seed, device_specific=True), grpo_trainer.py:451)
        self._gen = torch.Generator(device="cuda")
        self._gen.manual_seed(a.seed + rank)
        self.timings = defaultdict(float)
        self._ev = []                      # (phase, start_event, end_event): GPU-side phase times, read by gpu_phase_ms()

    @property
    def global_step(self):
        return self.state.global_step

    @global_step.setter
    def global_step(self, v):
        self.state.global_step = v

    def add_callback(self, cb):
        self.callback_handler.callbacks.append(cb)

    def _mark(self, phase):
        """Context manager: CUDA-event bracket of a phase on the current stream (no host sync)."""
        tr = self

        class _M:
            def __enter__(self_m):
                self_m.e0 = torch.cuda.Event(enable_timing=True); self_m.e1 = torch.cuda.Event(enable_timing=True)
                self_m.e0.record()

            def __exit__(self_m, *a):
                self_m.e1.record()
                tr._ev.append((phase, self_m.e0, self_m.e1))
        return _M()

    def gpu_phase_ms(self, reset=True):
        torch.cuda.synchronize()
        out = defaultdict(float)
        for ph, e0, e1 in self._ev:
            out[ph] += e0.elapsed_time(e1)
        if reset:
            self._ev = []
        return dict(out)

    # ------------------------------------------------------------------ data
    def _get_train_sampler(self):                                                          # grpo_trainer.py:883-897
        _, world = _world()
        a = self.args
        eff = a.per_device_train_batch_size * world * a.gradient_accumulation_steps
        return RepeatRandomSampler(self.train_dataset, self.num_generations, eff // self.num_generations, self.num_iterations, a.seed)

    def _prepare_prompt_inputs(self, inputs) -> Dict[str, Any]:
        """Pre-tokenised batches pass through; raw examples go through dna_module + processor like :538-567.  Returns the model
        inputs plus `_examples` (the raw example dicts, for the reward columns) and `_prompts`."""
        if isinstance(inputs, dict) and "input_ids" in inputs:
            out = dict(inputs)
            out.setdefault("_examples", inputs.get("examples"))
            out.setdefault("_prompts", inputs.get("prompts"))
            return out
        if self.dna_module is None or self.processing_class is None:
            raise ValueError("raw examples need dna_module and processing_class (no tokenizer files exist offline); pass a tokenised batch")
        prompts_text = self.dna_module.prepare_prompt(self.processing_class, inputs)
        dnas = [x["dna_sequences"] for x in inputs]
        out = dict(self.dna_module.prepare_model_inputs(self.processing_class, self.model, prompts_text, dnas, return_tensors="pt", padding=True,
                                                        padding_side="left", add_special_tokens=False))
        out["_examples"] = list(inputs)
        out["_prompts"] = [x["prompt"] for x in inputs]                                     # grpo_trainer.py:537
        return out

    # ------------------------------------------------------------------ log-probs
    def _get_per_token_logps(self, model, input_ids, attention_mask, keep_last=None, lora="policy", dropout=False, group_size=None, **mm):
        """grpo_trainer.py:510-520 (+ the [:, P-1:] slice of :779 when keep_last is given), no-grad version."""
        n = input_ids.shape[1] - 1 if keep_last is None else keep_last
        with torch.no_grad():
            lp, _ = training.policy_forward(model, input_ids, attention_mask, mm.get("dna_tokenized"), mm.get("batch_idx_map"), n,
                                            save=False, lora=lora, dropout=dropout, **({"group_size": group_size} if group_size else {}))
        return lp

    def _get_per_token_logps_and_entropies(self, model, input_ids, attention_mask, keep_last, lora="policy", dropout=False, group_size=None,
                                           dropout_pass=None, row_offset=0, **mm):
        """No-grad (log-probs, entropies) [B, keep_last] of the fused lm-head pass (TRL's method of this name; T = 1).  dropout_pass /
        row_offset as training.policy_forward takes them, so a row chunk reproduces the LoRA dropout masks of a whole pass."""
        kw = dict(group_size=group_size) if group_size else {}
        if dropout_pass is not None:
            kw.update(dropout_pass=dropout_pass, row_offset=row_offset)
        with torch.no_grad():
            lp, _, ent = training.policy_forward(model, input_ids, attention_mask, mm.get("dna_tokenized"), mm.get("batch_idx_map"), keep_last,
                                                 save=False, lora=lora, dropout=dropout, want_entropy=True, **kw)
        return lp, ent

    def _entropy_threshold(self, entropies, completion_mask, rho):
        """Device fp32 [1]: TRL's threshold torch.quantile(valid entropies of all ranks, 1 - rho); +inf when no token is valid."""
        vals, valid = dp.gather_masked(entropies, completion_mask)
        return ops.entropy_threshold(vals, valid, 1.0 - rho)

    def _local_group_size(self, prompt_ids, mm) -> Optional[int]:
        """Rows per prompt group in this rank's rows when share_prompt_prefix is on (None when off): consecutive identical prompts
        (text and DNA), so a rank holding part of a group still shares it.  One host sync."""
        if not getattr(self.args, "share_prompt_prefix", False):
            return None
        eq = generation.detect_group_size(prompt_ids, mm.get("dna_tokenized"), mm.get("batch_idx_map"))
        return generation.group_size_from_flags([bool(x) for x in eq.tolist()])

    # ------------------------------------------------------------------ rollout + scoring
    @torch.no_grad()
    def _generate_and_score_completions(self, inputs, model, uniforms=None, rewards_per_func=None) -> Dict[str, Any]:
        t0 = time.perf_counter()
        pi = self._prepare_prompt_inputs(inputs)
        dev = model._dec.embed.device
        prompt_ids, prompt_mask = pi["input_ids"].to(dev), pi["attention_mask"].to(dev)
        dna = pi.get("dna_tokenized")
        if dna is not None:                                                # device-resident once: the three passes of the step reuse the tensors
            dna = {k: dna[k].to(dev) for k in ("input_ids", "attention_mask")}
        mm = dict(dna_tokenized=dna, batch_idx_map=pi.get("batch_idx_map"))
        B, P = prompt_ids.shape
        C = self.max_completion_length
        if uniforms is None:
            uniforms = torch.rand(C, B, device=dev, generator=self._gen)
        with self._mark("rollout"):
            completion_ids = model.generate(prompt_ids, prompt_mask, mm["dna_tokenized"], mm["batch_idx_map"], uniforms=uniforms, **self.generation_kwargs)
        sampling_lp = None
        if self.generation_kwargs.get("return_logprobs"):
            completion_ids, sampling_lp = completion_ids
        self.timings["rollout"] += time.perf_counter() - t0
        eos = self.eos_token_id if not self.args.suppress_eos else -1
        lengths = None
        if getattr(self.args, "mask_truncated_completions", False):
            # TRL: rows without EOS carry no loss and are masked out of the scoring passes too; rewards and completion_length see the
            # completions as they were generated
            completion_mask, lengths = ops.eos_mask_truncated(completion_ids, eos)
            reward_mask = (torch.arange(completion_ids.shape[1], device=dev)[None, :] < lengths[:, None]).to(torch.int32)
        else:
            completion_mask = ops.eos_mask(completion_ids, eos)                                                       # :605-609
            reward_mask = completion_mask
        # text reward functions need the ids on the host: start the copy now (side stream, pinned), wait for it only after the
        # reference-policy forward has been queued -> decode + CPU rewards overlap that forward
        need_text = rewards_per_func is None and any(not rw.wants_token_protocol(f) for f in self.reward_funcs)
        host_copy = rw.AsyncHostCopy(completion_ids) if need_text else None
        self.reward_d2h_bytes = host_copy.nbytes if host_copy is not None else 0
        ids = torch.cat([prompt_ids, completion_ids], dim=1)
        attention_mask = torch.cat([prompt_mask, completion_mask.to(prompt_mask.dtype)], dim=1)                       # :612
        Cc = completion_ids.shape[1]
        gs = self._local_group_size(prompt_ids, mm)
        with self._mark("ref_logps"):
            # the reference computes old log-probs in train mode: through the LoRA dropout when it is on
            old_lp = (self._get_per_token_logps(model, ids, attention_mask, keep_last=Cc, dropout=True, group_size=gs, **mm)
                      if self.num_iterations > 1 else None)
            ref_lp = self._get_per_token_logps(model, ids, attention_mask, keep_last=Cc, lora=None, group_size=gs, **mm) if self.beta != 0.0 else None
        # rewards: the reference protocol f(prompts=, completions=, **columns) on decoded text (:640-676); functions that name a
        # `completion_ids` parameter get device tensors instead (trainer/rewards.py)
        if rewards_per_func is None:
            t_r = time.perf_counter()
            rewards_per_func = rw.score(self.reward_funcs, examples=pi.get("_examples"), prompts=pi.get("_prompts"), completion_ids=completion_ids,
                                        completion_mask=reward_mask, prompt_ids=prompt_ids, processing_class=self.processing_class,
                                        host_copy=host_copy, extra_columns=pi.get("reward_kwargs"),
                                        reward_processing_classes=self.reward_processing_classes)
            self.timings["reward_host"] += time.perf_counter() - t_r
        rewards_all = dp.gather_rewards(rewards_per_func)                                                              # C1, :679
        scale = getattr(self.args, "scale_rewards", "group")
        if scale != "group":
            adv_all, std_used, zero_std = ops.grpo_advantages_scaled(rewards_all, self.num_generations, scale)
            reward_std = std_used.mean()
            self._metrics["frac_reward_zero_std"].append(zero_std.float().mean())
        else:
            adv_all, gmean, gstd = ops.grpo_advantages(rewards_all, self.num_generations, return_stats=True)           # :682-692
            reward_std = gstd.mean()
        advantages = dp.local_slice(adv_all, B)                                                                        # :695-699
        self._metrics["completion_length"].append((lengths if lengths is not None else completion_mask.sum(1)).float().mean())
        self._metrics["reward"].append(rewards_all.sum(1).mean())
        self._metrics["reward_std"].append(reward_std)
        for i, f in enumerate(self.reward_funcs):
            self._metrics[f"rewards/{rw.reward_func_name(f, i)}"].append(rewards_all[:, i].mean())
        self.timings["score"] += time.perf_counter() - t0
        out = dict(prompt_ids=prompt_ids, prompt_mask=prompt_mask, completion_ids=completion_ids, completion_mask=completion_mask,
                   old_per_token_logps=old_lp, ref_per_token_logps=ref_lp, advantages=advantages, multimodal_inputs=mm,
                   local_group_size=gs)
        if sampling_lp is not None:
            out["sampling_per_token_logps"] = sampling_lp
        if getattr(self.args, "loss_type", "grpo") == "dapo":
            # buffered with the inputs, so the num_iterations > 1 passes over this batch reuse it
            out["num_items_in_batch"] = self._num_items_in_batch(lengths if lengths is not None else completion_mask)
        return out

    @staticmethod
    def _num_items_in_batch(counts):
        """TRL's num_items_in_batch: the completion tokens (EOS-masked, counted before mask_truncated_completions) of all ranks, a
        device fp32 [1]; one scalar all-reduce, no host sync."""
        n = counts.sum().float().reshape(1)
        if _world()[1] > 1:
            dist.all_reduce(n)
        return n

    @staticmethod
    def _auto_micro_rows(model, B, L):
        """Rows per forward/backward chunk when the config leaves `micro_rows` open: the most rows whose saved activations fit in
        three quarters of the memory this process can still get -- free device memory (other processes' allocations excluded) plus
        what the caching allocator holds but has not handed out; the rest is headroom for the backward's transients.  The loss is
        row-separable, so the chunking changes only the fp32 order of the gradient sums."""
        dev = model._dec.embed.device
        free = torch.cuda.mem_get_info(dev)[0] + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
        per_row = L * training.activation_bytes_per_token(model)
        return max(1, min(B, int(0.75 * free) // per_row))

    @staticmethod
    def _auto_micro_groups(model, U, G, P, L):
        """Rows per chunk of the shared-prefix passes when `micro_rows` is open: whole groups, as many as fit like _auto_micro_rows,
        a group costing Lp + G * Ls tokens of saved activations (one group per chunk when even one exceeds the estimate)."""
        dev = model._dec.embed.device
        free = torch.cuda.mem_get_info(dev)[0] + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
        Lp = training.SHARED_TILE * ((P - 1) // training.SHARED_TILE)
        per_group = (Lp + G * (L - Lp)) * training.activation_bytes_per_token(model)
        return G * max(1, min(U, int(0.75 * free) // per_group))

    # ------------------------------------------------------------------ loss (+ backward through the kernels)
    def compute_loss(self, model, inputs, return_outputs=False, num_items_in_batch=None, backward: bool = True):
        if return_outputs:
            raise ValueError("The GRPOTrainer does not support returning outputs")          # grpo_trainer.py:752-753
        if self.global_step % self.num_iterations == 0 or self._buffered_inputs[self._step % self.args.gradient_accumulation_steps] is None:
            if "completion_ids" not in inputs:
                inputs = self._generate_and_score_completions(inputs, model)
            self._buffered_inputs[self._step % self.args.gradient_accumulation_steps] = inputs
        else:
            inputs = self._buffered_inputs[self._step % self.args.gradient_accumulation_steps]
        self._step += 1
        prompt_ids, prompt_mask = inputs["prompt_ids"], inputs["prompt_mask"]
        completion_ids, completion_mask = inputs["completion_ids"], inputs["completion_mask"]
        mm = inputs["multimodal_inputs"]
        ids = torch.cat([prompt_ids, completion_ids], dim=1)
        mask = torch.cat([prompt_mask, completion_mask.to(prompt_mask.dtype)], dim=1)
        B, C = completion_ids.shape
        adv, old, ref = inputs["advantages"], inputs["old_per_token_logps"], inputs["ref_per_token_logps"]
        gs = inputs["local_group_size"] if "local_group_size" in inputs else self._local_group_size(prompt_ids, mm)
        if gs is not None and gs > 1:
            # shared prompt prefix: chunks hold whole groups
            if self.args.micro_rows and self.args.micro_rows % gs != 0:
                raise ValueError(f"micro_rows ({self.args.micro_rows}) must be a multiple of the local group size ({gs}) with share_prompt_prefix")
            mr = self.args.micro_rows or (self._auto_micro_groups(model, B // gs, gs, prompt_ids.shape[1], ids.shape[1]) if ids.is_cuda else B)
        else:
            mr = self.args.micro_rows or (self._auto_micro_rows(model, B, ids.shape[1]) if ids.is_cuda else B)
        ga = self.args.gradient_accumulation_steps
        loss_acc = torch.zeros(3, device=ids.device)
        tis = getattr(self.args, "rollout_is_correction", False)
        if tis:
            samp = inputs.get("sampling_per_token_logps")
            if samp is None:
                raise ValueError("rollout_is_correction needs the rollout's log-probs: inputs lack 'sampling_per_token_logps' "
                                 "(model.generate(..., return_logprobs=True))")
            is_cap = getattr(self.args, "rollout_is_cap", 2.0)
            is_acc = torch.zeros(4, device=ids.device)
        # one LoRA-dropout pass for all row chunks; each chunk passes its first row so the masks ignore the chunking
        pid = model.new_lora_dropout_pass() if getattr(model, "_lora", None) is not None else None
        # high-entropy token selection (TRL's top_entropy_quantile): one threshold per call over the valid completion tokens of all
        # ranks.  It must not depend on the row chunking, so with several chunks a no-grad pre-pass (same dropout pass, same row
        # offsets: the same entropies, checked below) scores every row first; with one chunk the loss pass's own entropies are used.
        rho = float(getattr(self.args, "top_entropy_quantile", 1.0))
        masking = rho < 1.0
        want_ent = masking or bool(getattr(self.args, "log_entropy", False))
        tau = pre_ent = ent_diff = None
        if want_ent:
            ent_acc = torch.zeros(1, device=ids.device)
            if not masking:
                tau = torch.full((1,), -float("inf"), device=ids.device)    # keeps every token: the loss of grpo_loss_raw, bit for bit
            elif mr < B:
                t0 = time.perf_counter()
                with self._mark("entropy_prepass"):
                    parts = []
                    for lo in range(0, B, mr):
                        hi = min(B, lo + mr)
                        mm_c = _slice_mm(mm, lo, hi)
                        parts.append(self._get_per_token_logps_and_entropies(
                            model, ids[lo:hi], mask[lo:hi], C, dropout=pid is not None, group_size=gs, dropout_pass=pid, row_offset=lo,
                            **mm_c)[1])
                    pre_ent = torch.cat(parts)
                    tau = self._entropy_threshold(pre_ent, completion_mask, rho)
                    ent_diff = torch.zeros((), dtype=torch.bool, device=ids.device)
                self.timings["entropy_prepass"] += time.perf_counter() - t0
        # the objectives of later TRL releases (loss_type, sequence-level ratios, delta) run on br_grpo_objective_fwd_bwd, whose outputs
        # are sums over a chunk's rows; the defaults keep the calls above
        loss_type = getattr(self.args, "loss_type", "grpo")
        seq_level = getattr(self.args, "importance_sampling_level", "token") == "sequence"
        delta = getattr(self.args, "delta", None)
        objective = loss_type != "grpo" or seq_level or delta is not None
        if objective:
            obj_acc = torch.zeros(7, device=ids.device)
            if loss_type == "grpo":
                norm_kw = dict(norm_rows=B)
            elif loss_type == "bnpo":
                norm_kw = dict(norm=completion_mask.sum().float().clamp(min=1).reshape(1))
            elif loss_type == "dr_grpo":
                norm_kw = dict(norm=torch.full((1,), float(B * self.max_completion_length), device=ids.device))
            else:                                                           # dapo: the gradient average over ranks makes it the global mean
                n = inputs.get("num_items_in_batch")
                if n is None:
                    n = self._num_items_in_batch(completion_mask)
                norm_kw = dict(norm=n.clamp(min=1) / _world()[1])
        for lo in range(0, B, mr):
            hi = min(B, lo + mr)
            sl = slice(lo, hi)
            mm_c = _slice_mm(mm, lo, hi)
            t0 = time.perf_counter()
            with self._mark("policy_fwd"):
                drop_kw = dict(dropout=True, dropout_pass=pid, row_offset=lo) if pid is not None else {}
                ent_kw = dict(want_entropy=True) if want_ent else {}
                out = training.policy_forward(model, ids[sl], mask[sl], mm_c["dna_tokenized"], mm_c["batch_idx_map"], C, save=backward,
                                              **({"group_size": gs} if gs else {}), **drop_kw, **ent_kw)
                lp, ctx = out[0], out[1]
            if want_ent:
                ent = out[2]
                if pre_ent is not None:
                    ent_diff |= (ent != pre_ent[sl]).any()
                if tau is None:                                             # masking with one chunk: the threshold of this pass
                    tau = self._entropy_threshold(ent, completion_mask, rho)
            if objective:
                out7, is_stats, ent_sum, dlp = ops.grpo_objective_raw(
                    lp, old[sl] if old is not None else None, ref[sl] if ref is not None else None, adv[sl], completion_mask[sl], self.beta,
                    self.epsilon_low, self.epsilon_high, sequence_level=seq_level, delta=delta, rollout_lp=samp[sl] if tis else None,
                    is_cap=is_cap if tis else 2.0, entropy=ent if want_ent else None, tau=tau if want_ent else None, want_grad=backward,
                    **norm_kw)
                obj_acc += out7
                if tis:
                    is_acc += is_stats
                if want_ent:
                    ent_acc += ent_sum
            elif want_ent:
                out3, is_stats, ent_sum, dlp = ops.grpo_loss_ent_raw(
                    lp, old[sl] if old is not None else None, ref[sl] if ref is not None else None, samp[sl] if tis else None, adv[sl],
                    completion_mask[sl], ent, tau, self.beta, self.epsilon_low, self.epsilon_high, is_cap if tis else 2.0,
                    want_grad=backward)
                ent_acc += ent_sum
            elif tis:
                out3, is_stats, dlp = ops.grpo_loss_is_raw(lp, old[sl] if old is not None else None, ref[sl] if ref is not None else None,
                                                           samp[sl], adv[sl], completion_mask[sl], self.beta, self.epsilon_low,
                                                           self.epsilon_high, is_cap, want_grad=backward)
            else:
                out3, dlp = ops.grpo_loss_raw(lp, old[sl] if old is not None else None, ref[sl] if ref is not None else None, adv[sl],
                                              completion_mask[sl], self.beta, self.epsilon_low, self.epsilon_high, want_grad=backward)
            if objective:
                w = 1.0                                                     # sums: the chunks add up
            else:
                w = (hi - lo) / B
                loss_acc += out3 * w                                        # row-mean of row-means is separable over row chunks
                if tis:
                    is_acc += is_stats * w                                  # token means, row-weighted across chunks like clip_ratio
            self.timings["policy_fwd"] += time.perf_counter() - t0
            if backward:
                t0 = time.perf_counter()
                # the last chunk of the last accumulation micro-step completes the gradients: all-reduce each layer's slice as the
                # backward leaves it (C2 overlapped with the remaining backward)
                hook = None
                if hi == B and self._step % ga == 0 and _world()[1] > 1 and getattr(model, "_lora", None) is not None:
                    self._reducer = dp.OverlappedGradReduce(model._lora.flat_grad)
                    hook = lambda li, _m=model: self._reducer.reduce_slice(*_m._lora.layer_slice(li))
                with self._mark("policy_bwd"):
                    training.policy_backward(model, ctx, dlp * (w / ga), on_layer_done=hook)
                self.timings["policy_bwd"] += time.perf_counter() - t0
        if objective:
            # token means exact across row chunks; kl keeps its row-mean definition
            n_tok = obj_acc[6].clamp(min=1)
            loss_acc = torch.stack([obj_acc[0], obj_acc[1] / B, obj_acc[2] / n_tok])
            for name, v in zip(("low_mean", "high_mean", "region_mean"), obj_acc[3:6] / n_tok):
                self._metrics[f"clip_ratio/{name}"].append(v)
            if tis:
                is_acc = is_acc / n_tok
        # clip_ratio is a ratio of sums; with row chunks it is weighted by rows (exact when chunks have equal mask counts)
        if self.beta > 0:
            self._metrics["kl"].append(loss_acc[1])
        self._metrics["clip_ratio"].append(loss_acc[2])
        if tis:
            for name, v in zip(("ratio_mean", "capped_frac", "logp_diff", "kl"), is_acc):
                self._metrics[f"rollout_is/{name}"].append(v)
        if want_ent:
            if ent_diff is not None and bool(ent_diff):
                raise RuntimeError("the entropy pre-pass and the loss pass disagree: the token mask would depend on the row chunking")
            self._metrics["entropy"].append(ent_acc[0] / completion_mask.sum().clamp(min=1))
            if masking:
                self._metrics["entropy/threshold"].append(tau[0])
        return loss_acc[0]

    # ------------------------------------------------------------------ one optimizer step
    def training_step(self, inputs) -> torch.Tensor:
        model = self.model
        if self._step % self.args.gradient_accumulation_steps == 0:
            model.zero_grad_buffers()
        loss = self.compute_loss(model, inputs)
        if self._step % self.args.gradient_accumulation_steps == 0:
            self._optimizer_step()
        return loss

    def _optimizer_step(self):
        model = self.model
        t0 = time.perf_counter()
        with self._mark("grad_allreduce"):
            red = getattr(self, "_reducer", None)
            if red is not None:                                            # slices already in flight under the backward; wait + the rest
                red.finish([model._proj_grad_w, model._proj_grad_b])
                self._reducer = None
            else:
                dp.allreduce_mean_([model._lora.flat_grad, model._proj_grad_w, model._proj_grad_b])     # C2: sum then / world (DDP average)
        with self._mark("optimizer"):
            model.attach_grads()
            if self.args.max_grad_norm and self.args.max_grad_norm > 0:
                torch.nn.utils.clip_grad_norm_(model.trainable_parameters(), self.args.max_grad_norm, foreach=True)
            self.optimizer.step()
        with self._mark("adapter_sync"):
            model.sync_adapters(rollout=True)
        self.global_step += 1
        self.timings["optimizer"] += time.perf_counter() - t0
        a = self.args
        self.control = self.callback_handler.fire("on_step_end")
        if getattr(a, "logging_steps", 0) and self.callback_handler.callbacks and self.global_step % max(1, int(a.logging_steps)) == 0:
            logs = self.log_metrics()
            self.state.log_history.append(dict(logs, step=self.global_step))
            self.control = self.callback_handler.fire("on_log", logs=logs)
        if getattr(a, "save_steps", 0) and self.global_step % int(a.save_steps) == 0:
            self.control.should_save = True
        if self.control.should_save:
            self.control = self.callback_handler.fire("on_save")               # reason.py:46-81 SaveWithPyTorchCallback hooks here
            self.control.should_save = False

    def train(self, batches=None, max_steps: Optional[int] = None):
        """Iterate tokenised batches (or the dataset through RepeatRandomSampler) for max_steps optimizer steps."""
        a = self.args
        steps = max_steps if max_steps is not None else (a.max_steps if a.max_steps > 0 else None)
        if batches is None:
            sampler = list(iter(self._get_train_sampler()))
            batches = ([self.train_dataset[i] for i in idx] for idx in dp.rank_batches(sampler, a.per_device_train_batch_size))
        out = []
        self.control = self.callback_handler.fire("on_train_begin")
        for b in batches:
            self.control = self.callback_handler.fire("on_step_begin")
            out.append(self.training_step(b))
            if (steps is not None and self.global_step >= steps) or self.control.should_training_stop:
                break
        self.control = self.callback_handler.fire("on_train_end")
        return out

    def log_metrics(self) -> Dict[str, float]:
        m = {k: float(torch.stack([torch.as_tensor(x, dtype=torch.float32, device="cuda") for x in v]).mean()) for k, v in self._metrics.items()}
        self._metrics.clear()
        return m


def _slice_mm(mm, lo, hi):
    """Row-chunk the multimodal inputs (dna rows follow batch_idx_map)."""
    if mm.get("dna_tokenized") is None or not mm.get("batch_idx_map"):
        return dict(dna_tokenized=None, batch_idx_map=[])
    idx = [i for i, b in enumerate(mm["batch_idx_map"]) if lo <= b < hi]
    it = torch.tensor(idx, device=mm["dna_tokenized"]["input_ids"].device)
    return dict(dna_tokenized={k: v[it] for k, v in mm["dna_tokenized"].items() if k in ("input_ids", "attention_mask")},
                batch_idx_map=[mm["batch_idx_map"][i] - lo for i in idx])
