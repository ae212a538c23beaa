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

Everything in this file is host logic (no kernels): it is covered by tests/test_rewards_cpu.py.
"""
from __future__ import annotations

import inspect
from typing import Any, Callable, Dict, List, Optional, Sequence

import torch


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
          host_copy: Optional[AsyncHostCopy] = None, extra_columns: Optional[Dict[str, List[Any]]] = None) -> torch.Tensor:
    """rewards_per_func [B, n_funcs] fp32 on completion_ids.device, reference protocol by default (see module docstring)."""
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
        if i in text_funcs:
            vals = f(prompts=prompts, completions=completions, **columns)
        else:
            vals = f(completion_ids=completion_ids, prompt_ids=prompt_ids, completion_mask=completion_mask)
        out[:, i] = torch.as_tensor(vals, dtype=torch.float32).to(dev)
    return out
