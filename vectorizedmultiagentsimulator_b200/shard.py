"""NCCL-free sharding of ``batch_dim`` across GPUs (one process per GPU).

Envs are independent, so a job of ``total_envs`` is split into contiguous shards, each stepped by
its own process on its own device with no data-path collective.  ``torch.distributed`` is used
only for control-plane reductions (timings, counters).  The one batch-coupled piece of the
reference — the batch-wide broad-phase activation of line/box pairs (ref core.py:2797-2801) — is
evaluated per shard; ``exact_global_broad_phase`` is the hook where an OR-all-reduce of the pair
mask would go if bit-equality with an unsharded run were required (off: envs stay independent).
"""
from __future__ import annotations

import os
from typing import Tuple

import torch
import torch.distributed as dist


def dist_env() -> Tuple[int, int, int]:
    """(rank, world_size, local_rank) from the torchrun environment (defaults: single process)."""
    return (
        int(os.environ.get("RANK", "0")),
        int(os.environ.get("WORLD_SIZE", "1")),
        int(os.environ.get("LOCAL_RANK", "0")),
    )


def shard_bounds(total_envs: int, rank: int, world_size: int) -> Tuple[int, int]:
    """[lo, hi) of the contiguous env range owned by ``rank`` (sizes differ by at most one)."""
    assert 0 <= rank < world_size
    base, extra = divmod(total_envs, world_size)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def max_over_ranks(value: float, device=None) -> float:
    """MAX-all-reduce of a scalar (the slowest rank defines a multi-GPU time)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return float(value)
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def sum_over_ranks(value: float, device=None) -> float:
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return float(value)
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return float(t.item())


def aggregate_throughput(local_units: float, local_seconds: float, device=None) -> float:
    """Whole-job units/s = sum of the units every rank processed / the slowest rank's time."""
    return sum_over_ranks(local_units, device) / max_over_ranks(local_seconds, device)


def make_shard_env(scenario, total_envs: int, rank: int, world_size: int, device, seed: int = 0,
                   obs_dtype: torch.dtype = torch.float32, **kwargs):
    """This rank's shard of a job of ``total_envs`` envs: ``make_env`` with the shard's size, plus
    the shard's position in the job (``world.env_offset``) so that every reset — including the one
    that builds the initial state — places entities exactly where the unsharded job would place
    them for the same envs (the respawn kernel numbers its random streams by global env index).
    That holds for scenarios whose reset draws all come from ``ScenarioUtils`` / ``World.spawn_positions``
    (the four shipped ones); draws taken from torch's generator are reproducible per shard but differ
    from the unsharded job's.  ``obs_dtype``: as ``make_env`` takes it.
    """
    from .make_env import make_env

    lo, hi = shard_bounds(total_envs, rank, world_size)
    env = make_env(scenario, num_envs=hi - lo, device=device, seed=seed, obs_dtype=obs_dtype, **kwargs)
    env.world.env_offset = lo
    env.world.reset_count.zero_()  # the construction-time reset above does not count as an episode
    env.reset(seed=seed)
    return env
