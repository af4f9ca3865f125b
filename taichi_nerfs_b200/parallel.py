"""Ray-sharded data parallelism: the only multi-GPU structure the hot path needs (SURVEY.md §8e).

Rays are independent units, so a global batch of ``world * n`` rays is split into contiguous shards,
every rank renders its shard with replicated parameters, and ONE all-reduce (sum) of the flat gradient
buffer ``[hash grad | MLP grads]`` per step makes the replicas agree.  Each rank's loss is a mean over
its own shard, so the all-reduced sum is divided by ``world`` (folded into the fused Adam's
``inv_scale``): the update equals the single-process update on the concatenated batch.
Backend: NCCL over NVLink/NVSwitch on GPUs; gloo in the CPU tests (tests/test_dist.py).
"""
from __future__ import annotations

import torch
import torch.distributed as dist


def world_info(group=None):
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(group), dist.get_world_size(group)
    return 0, 1


def shard_bounds(n_global: int, rank: int, world: int):
    """Contiguous [begin, end) slice of the global ray batch owned by ``rank`` (remainder to low ranks)."""
    base, rem = divmod(n_global, world)
    begin = rank * base + min(rank, rem)
    return begin, begin + base + (1 if rank < rem else 0)


def allreduce_gradients(flat_grad: torch.Tensor, group=None) -> torch.Tensor:
    """In-place sum of the flat gradient buffer over all ranks (a single collective per step)."""
    rank, world = world_info(group)
    if world > 1:
        dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM, group=group)
    return flat_grad


def allreduce_found_inf(found_inf: torch.Tensor, group=None) -> torch.Tensor:
    """If any rank saw a non-finite gradient every rank must skip the step (GradScaler semantics)."""
    rank, world = world_info(group)
    if world > 1:
        dist.all_reduce(found_inf, op=dist.ReduceOp.MAX, group=group)
    return found_inf


def inv_grad_scale(loss_scale: float, world: int) -> float:
    """Factor that turns the all-reduced, loss-scaled gradient sum into the global-batch mean gradient."""
    return 1.0 / (float(loss_scale) * world)


def optimizer_shard(n_table: int, rank: int, world: int):
    """[begin, end) of the flat table parameter owned by ``rank`` in the peer-memory optimizer step (NGPTrainer): equal
    shards, each a multiple of 4 floats so that every shard stays 16-byte aligned for the float4 Adam sweep."""
    if n_table % (4 * world) != 0:
        raise ValueError(f"table size {n_table} is not a multiple of 4 * world ({world})")
    shard = n_table // world
    return rank * shard, (rank + 1) * shard

