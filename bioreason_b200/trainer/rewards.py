"""Reward-function plumbing of the GRPO step (bioreason/trainer/grpo_trainer.py:640-676).

The reference decodes the completions with `processing_class.batch_decode(..., skip_special_tokens=True)`, wraps them as
`[{"role": "assistant", "content": text}]` when the examples are conversational, and calls every reward function as
`reward_func(prompts=prompts, completions=completions, **columns)` where `columns` are the remaining keys of the examples
(one list entry per row).  That protocol is the default here.  Two additions for the CUDA path:

* a reward function may opt into the token-level fast path by NAMING a `completion_ids` parameter
  (`def f(completion_ids, completion_mask=None, prompt_ids=None, **kw)`): it then receives device tensors and nothing is
  decoded for it;
* the device->host copy of the completion ids is asynchronous (pinned buffer, side stream, CUDA event): the host waits
  for that event only, so decoding + the CPU reward functions overlap the reference-policy forward that is already
  queued on the compute stream (SURVEY.md §8f-2).

A reward function may also be a sequence-classification model (a path or a `PreTrainedModel`, grpo_trainer.py:343-368), run as a
`RewardModel` on the CUDA decoder: the texts are built and tokenized on the host as the reference does (:656-663) and the model writes
its column of rewards_per_func on the device.

Everything in this file is host logic (the reward model's device work is in reward_model.py): it is covered by
tests/test_rewards_cpu.py and tests/test_reward_model_cpu.py.
"""
from __future__ import annotations

import inspect
from typing import Any, Callable, Dict, List, Optional, Sequence

import torch

from ..reward_model import RewardModel


def is_conversational(example: Dict[str, Any]) -> bool:
    """trl.data_utils.is_conversational restated: a prompt/completion/messages value that is a list of {role, content} dicts."""
    for key in ("prompt", "chosen", "rejected", "completion", "messages"):
        v = example.get(key) if isinstance(example, dict) else None
        if isinstance(v, list) and v and isinstance(v[0], dict) and "role" in v[0] and "content" in v[0]:
            return True
    return False


def wants_token_protocol(f: Callable) -> bool:
    """True when the callable names a `completion_ids` parameter and no `completions` parameter (the opt-in fast path)."""
    try:
        params = inspect.signature(f).parameters
    except (TypeError, ValueError):
        return False
    return "completion_ids" in params and "completions" not in params


def reward_columns(examples: Optional[Sequence[Dict[str, Any]]]) -> Dict[str, List[Any]]:
    """grpo_trainer.py:664-670: every example key except prompt / completion becomes a per-row list."""
    if not examples:
        return {}
    keys = [k for k in examples[0].keys() if k not in ("prompt", "completion")]
    return {k: [ex[k] for ex in examples] for k in keys}


class AsyncHostCopy:
    """completion ids -> pinned host memory on a side stream; `.wait()` blocks on the copy's event only."""

    def __init__(self, t: torch.Tensor):
        self.host = torch.empty(t.shape, dtype=t.dtype, pin_memory=True) if t.is_cuda else t
        self.event = None
        if t.is_cuda:
            side = _side_stream(t.device)
            side.wait_stream(torch.cuda.current_stream(t.device))           # the rollout that produced `t`
            with torch.cuda.stream(side):
                self.host.copy_(t, non_blocking=True)
                self.event = torch.cuda.Event()
                self.event.record(side)
            t.record_stream(side)
        self.nbytes = t.numel() * t.element_size()

    def wait(self) -> torch.Tensor:
        if self.event is not None:
            self.event.synchronize()
        return self.host


_SIDE = {}


def _side_stream(device):
    key = (device.type, device.index)
    if key not in _SIDE:
        _SIDE[key] = torch.cuda.Stream(device=device)
    return _SIDE[key]


def apply_chat_template(example: Dict[str, Any], tokenizer) -> Dict[str, str]:
    """trl.data_utils.apply_chat_template restated for the "messages" key, the only one the reward-model texts use."""
    return {"text": tokenizer.apply_chat_template(example["messages"], tokenize=False)}


def reward_func_name(f, i: int) -> str:
    """The metric suffix of reward function i (grpo_trainer.py:707-711): a model's last path component, else the function name."""
    if isinstance(f, RewardModel):
        return f.config._name_or_path.split("/")[-1]
    return getattr(f, "__name__", f"reward_{i}")


def resolve_reward_funcs(reward_funcs, reward_processing_classes, model_init_kwargs, device):
    """grpo_trainer.py:341-370: paths load as AutoModelForSequenceClassification(num_labels=1), every model gets a tokenizer (its own
    directory's by default, pad = eos when it has none, config.pad_token_id set to it) and is packed as a RewardModel on `device`.
    Returns (reward_funcs, reward_processing_classes), one entry per function (None for callables)."""
    funcs = list(reward_funcs) if isinstance(reward_funcs, (list, tuple)) else [reward_funcs]
    if reward_processing_classes is None:
        procs = [None] * len(funcs)
    elif not isinstance(reward_processing_classes, list):
        procs = [reward_processing_classes]
    else:
        if len(reward_processing_classes) != len(funcs):
            raise ValueError("The number of reward processing classes must match the number of reward functions.")
        procs = list(reward_processing_classes)
    procs += [None] * (len(funcs) - len(procs))
    from transformers import AutoModelForSequenceClassification, AutoTokenizer, PreTrainedModel
    for i, f in enumerate(funcs):
        if isinstance(f, str):
            f = AutoModelForSequenceClassification.from_pretrained(f, num_labels=1, **(model_init_kwargs or {}))
        if not isinstance(f, PreTrainedModel):
            continue
        proc = procs[i]
        if proc is None:
            proc = AutoTokenizer.from_pretrained(f.config._name_or_path)
        if proc.pad_token_id is None:
            proc.pad_token = proc.eos_token
        # the pooled token is the rightmost one that is not the tokenizer's pad
        f.config.pad_token_id = proc.pad_token_id
        funcs[i], procs[i] = RewardModel(f, device), proc
    return funcs, procs


def model_reward_texts(tokenizer, prompts, completions, conversational: bool) -> List[str]:
    """grpo_trainer.py:656-660: the prompt + completion text each row is scored on."""
    if conversational:
        return [apply_chat_template({"messages": p + c}, tokenizer)["text"] for p, c in zip(prompts, completions)]
    return [p + c for p, c in zip(prompts, completions)]


def decode_completions(processing_class, completion_ids_host: torch.Tensor, conversational: bool):
    """grpo_trainer.py:640-645."""
    if processing_class is None or not hasattr(processing_class, "batch_decode"):
        raise ValueError("text reward functions (f(prompts=, completions=, **columns), grpo_trainer.py:664-676) need a "
                         "processing_class with batch_decode(); pass one, or name a `completion_ids` parameter in the reward "
                         "function to receive token tensors instead")
    texts = processing_class.batch_decode(completion_ids_host, skip_special_tokens=True)
    if conversational:
        return texts, [[{"role": "assistant", "content": t}] for t in texts]
    return texts, texts


def score(reward_funcs: Sequence[Callable], *, examples: Optional[Sequence[Dict[str, Any]]], prompts: Optional[List[Any]],
          completion_ids: torch.Tensor, completion_mask: torch.Tensor, prompt_ids: torch.Tensor, processing_class,
          host_copy: Optional[AsyncHostCopy] = None, extra_columns: Optional[Dict[str, List[Any]]] = None,
          reward_processing_classes: Optional[Sequence[Any]] = None) -> torch.Tensor:
    """rewards_per_func [B, n_funcs] fp32 on completion_ids.device, reference protocol by default (see module docstring).
    reward_processing_classes: the tokenizer of each RewardModel function (resolve_reward_funcs), None elsewhere."""
    B = completion_ids.shape[0]
    dev = completion_ids.device
    out = torch.zeros(B, len(reward_funcs), device=dev, dtype=torch.float32)
    text_funcs = [i for i, f in enumerate(reward_funcs) if not wants_token_protocol(f)]
    completions = None
    if text_funcs:
        conv = bool(examples) and is_conversational(examples[0])
        ids_host = (host_copy or AsyncHostCopy(completion_ids)).wait()
        _, completions = decode_completions(processing_class, ids_host, conv)
        if prompts is None:
            prompts = [ex["prompt"] for ex in examples] if examples and "prompt" in examples[0] else [None] * B
        columns = reward_columns(examples)
        if extra_columns:
            columns.update(extra_columns)
    for i, f in enumerate(reward_funcs):
        if isinstance(f, RewardModel):
            if any(not isinstance(p, (str, list)) for p in prompts):
                raise ValueError("a reward model scores prompt + completion text: the batch needs its prompts (examples with a "
                                 "'prompt' key, or a 'prompts' list next to a tokenised batch)")
            tok = reward_processing_classes[i] if reward_processing_classes is not None else None
            if tok is None:
                raise ValueError(f"reward function {i} is a reward model and needs its reward processing class (tokenizer)")
            texts = model_reward_texts(tok, prompts, completions, conv)
            enc = tok(texts, return_tensors="pt", padding=True, padding_side="right", add_special_tokens=False)
            if f.num_labels == 1:
                f(enc["input_ids"], enc["attention_mask"], out=out[:, i:i + 1])
            else:                                                   # the reference takes logits[:, 0]
                out[:, i] = f(enc["input_ids"], enc["attention_mask"])[:, 0]
            continue
        if i in text_funcs:
            vals = f(prompts=prompts, completions=completions, **columns)
        else:
            vals = f(completion_ids=completion_ids, prompt_ids=prompt_ids, completion_mask=completion_mask)
        out[:, i] = torch.as_tensor(vals, dtype=torch.float32).to(dev)
    return out
