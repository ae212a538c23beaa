"""Data-parallel plumbing of the GRPO step (SURVEY.md §8e): one process per GPU, two collectives per step.

C1  all-gather of `rewards_per_func [B_local, n_funcs]` before the group statistics (grpo_trainer.py:679) -- groups are
    G consecutive rows of the GLOBAL batch, so they may straddle ranks when per_device_batch % G != 0;
C2  one all-reduce (sum, then / world: DDP averaging) of the flat LoRA + projector gradient buffers.
Rollouts, ref log-probs and policy forward/backward are rank-local.  Works on any torch.distributed backend
(NCCL over NVLink on the GPU box, gloo in the CPU tests).
"""
from __future__ import annotations

from typing import Iterable, List

import torch
import torch.distributed as dist


def world():
    return (dist.get_rank(), dist.get_world_size()) if dist.is_available() and dist.is_initialized() else (0, 1)


def gather_rewards(rewards_per_func: torch.Tensor) -> torch.Tensor:
    rank, ws = world()
    if ws == 1:
        return rewards_per_func
    parts = [torch.empty_like(rewards_per_func) for _ in range(ws)]
    dist.all_gather(parts, rewards_per_func.contiguous())
    return torch.cat(parts, 0)


def gather_masked(values: torch.Tensor, mask: torch.Tensor):
    """All ranks' values and int32 masks, flattened and concatenated in rank order (for a statistic over the valid entries of the
    whole batch, such as the entropy threshold).  Ranks may hold different numbers of entries (completion widths differ): each pads
    to the largest with mask 0, so the padding is never valid.  One host sync for the sizes when world > 1."""
    v = values.reshape(-1)
    m = mask.reshape(-1).to(torch.int32)
    rank, ws = world()
    if ws == 1:
        return v, m
    n = torch.tensor([v.numel()], device=v.device, dtype=torch.int64)
    sizes = [torch.empty_like(n) for _ in range(ws)]
    dist.all_gather(sizes, n)
    n_max = max(int(x.item()) for x in sizes)
    vp = torch.zeros(n_max, device=v.device, dtype=v.dtype)
    mp = torch.zeros(n_max, device=v.device, dtype=torch.int32)
    vp[:v.numel()] = v
    mp[:m.numel()] = m
    parts_v = [torch.empty_like(vp) for _ in range(ws)]
    parts_m = [torch.empty_like(mp) for _ in range(ws)]
    dist.all_gather(parts_v, vp)
    dist.all_gather(parts_m, mp)
    return torch.cat(parts_v), torch.cat(parts_m)


def local_slice(x: torch.Tensor, rows_local: int) -> torch.Tensor:
    """grpo_trainer.py:695-699."""
    rank, _ = world()
    return x[rank * rows_local:(rank + 1) * rows_local]


def allreduce_mean_(buffers: Iterable[torch.Tensor]) -> None:
    rank, ws = world()
    if ws == 1:
        return
    for b in buffers:
        dist.all_reduce(b)
        b.div_(ws)


class OverlappedGradReduce:
    """C2 overlapped with the backward (the reference's DeepSpeed config sets overlap_comm, ds_config_stage2.json:28-33): the flat LoRA
    gradient buffer is laid out layer by layer, and the backward finishes layers from the last to the first, so each layer's slice is
    all-reduced (async, on NCCL's stream) as soon as its kernels are enqueued -- it runs under the remaining backward.  `finish()`
    waits for the outstanding slices, reduces whatever was not covered (the projector buffers) and divides by the world size.
    Averaging order: every element is summed over ranks exactly once, then divided -- same result as one all-reduce of the buffer."""

    def __init__(self, flat: torch.Tensor):
        self.flat, self.works, self.covered = flat, [], []
        self.rank, self.ws = world()

    def reduce_slice(self, lo: int, hi: int):
        if self.ws == 1 or hi <= lo:
            return
        self.works.append(dist.all_reduce(self.flat[lo:hi], async_op=True))
        self.covered.append((lo, hi))

    def finish(self, extra: Iterable[torch.Tensor] = ()):
        if self.ws == 1:
            return
        # slices of the flat buffer nobody reduced yet (e.g. overlap disabled for this step)
        pos = 0
        for lo, hi in sorted(self.covered):
            if lo > pos:
                self.works.append(dist.all_reduce(self.flat[pos:lo], async_op=True))
            pos = max(pos, hi)
        if pos < self.flat.numel():
            self.works.append(dist.all_reduce(self.flat[pos:], async_op=True))
        extra = list(extra)
        for b in extra:
            self.works.append(dist.all_reduce(b, async_op=True))
        for w in self.works:
            w.wait()
        self.flat.div_(self.ws)
        for b in extra:
            b.div_(self.ws)
        self.works, self.covered = [], []


def rank_batches(sampler_indices: List[int], per_device: int):
    """Contiguous per-rank slices of the globally repeated index stream (what accelerate's batch sharding yields for
    the reference's RepeatRandomSampler, grpo_trainer.py:883-897): yields this rank's index list per global batch."""
    rank, ws = world()
    step = per_device * ws
    for s in range(0, len(sampler_indices) - step + 1, step):
        yield sampler_indices[s + rank * per_device: s + (rank + 1) * per_device]
