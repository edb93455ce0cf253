"""Multi-GPU: shard the MODEL axis of a sweep across ranks — one process per GPU, no data-path collective.

The reference already parallelises this way (cluster_runs.py:110-130: one OS process per ensemble/GPU, zero
communication; big_sweep_experiments.py:265-291 builds 8 GPUs x 16 L1 values): models of an ensemble never
exchange anything, so there is no gradient traffic at all. What this module adds is the launch model a multi-GPU box
uses (torchrun / torch.distributed, rank = GPU) and the only exchange the path has:

  * ``shard_slices`` / ``shard_models``: contiguous, balanced split of M_total models over the ranks;
  * ``gather_metrics``: END-OF-CHUNK all_gather of the per-model scalars ([M_local, K] -> [M_total, K]; a few KB) —
    NCCL over NVLink/NVSwitch on GPUs, gloo in the CPU tests;
  * ``gather_learned_dicts``: exported dictionaries to rank 0 for the single-file ``learned_dicts.pt``.
Every rank consumes the same activation stream (its own H2D copy of the chunk); nothing is communicated per step.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import torch
import torch.distributed as dist


def shard_slices(n_items: int, world: int) -> List[Tuple[int, int]]:
    """[start, stop) of every rank; the first ``n_items % world`` ranks get one extra item."""
    base, extra = divmod(n_items, world)
    out, start = [], 0
    for r in range(world):
        size = base + (1 if r < extra else 0)
        out.append((start, start + size))
        start += size
    return out


def shard_models(models: Sequence, rank: int, world: int) -> list:
    lo, hi = shard_slices(len(models), world)[rank]
    return list(models[lo:hi])


def gather_metrics(local: torch.Tensor, sizes: Sequence[int] = None) -> torch.Tensor:
    """all_gather of a [M_local, K] tensor along dim 0 (ragged shards allowed via ``sizes`` = M_local of each
    rank). Returns [M_total, K] on every rank. No-op when torch.distributed is not initialised."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return local
    world = dist.get_world_size()
    if sizes is None:
        sizes = [local.shape[0]] * world
    pad = max(sizes)
    buf = local
    if local.shape[0] < pad:
        buf = torch.cat([local, local.new_zeros((pad - local.shape[0],) + tuple(local.shape[1:]))])
    outs = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(outs, buf.contiguous())
    return torch.cat([o[:s] for o, s in zip(outs, sizes)])


def gather_learned_dicts(local_dicts: list, dst: int = 0):
    """Collect every rank's [(LearnedDict, hyperparams)] on ``dst`` in rank order (CPU tensors; pickled)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return local_dicts
    world = dist.get_world_size()
    gathered = [None] * world if dist.get_rank() == dst else None
    dist.gather_object(local_dicts, gathered, dst=dst)
    if dist.get_rank() != dst:
        return None
    return [item for part in gathered for item in part]
