"""Multi-GPU: the path shards by layout (every layout's T-step trajectory is independent; SURVEY.md 8e).
One process per GPU (torch.distributed); the model handle is replicated, the batch is split into contiguous shards,
noise is keyed by the GLOBAL layout index so the result does not depend on the number of GPUs, and the only
collective is one all-gather of the final ids (NCCL over NVLink on GPUs, gloo in the CPU tests)."""
from __future__ import annotations

import inspect
from typing import Callable, Dict, Optional, Tuple

import torch
import torch.distributed as dist


def shard_bounds(total: int, world: int, rank: int) -> Tuple[int, int]:
    """contiguous shard [lo, hi) of `total` layouts for `rank`; sizes differ by at most one"""
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_cond(cond: Optional[Dict], lo: int, hi: int) -> Optional[Dict]:
    if not cond:
        return None
    out = {}
    for k, v in cond.items():
        if isinstance(v, torch.Tensor) and v.dim() >= 1 and k not in ("refine_table", "rel_centers"):
            out[k] = v[lo:hi] if v.shape[0] > 1 else v          # a single condition broadcasts (task.py:235-248)
        else:
            out[k] = v
    return out


def all_gather_ids(local: torch.Tensor, total: int, group=None) -> torch.Tensor:
    """local (b_r, S) int64 on this rank's device -> (total, S) on every rank (ragged shards are padded to the max)"""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    sizes = [shard_bounds(total, world, r)[1] - shard_bounds(total, world, r)[0] for r in range(world)]
    mx = max(sizes)
    buf = local
    if local.shape[0] < mx:
        buf = torch.cat([local, local.new_zeros(mx - local.shape[0], local.shape[1])])
    out = torch.empty(world * mx, local.shape[1], dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, buf.contiguous(), group=group)
    if all(s == mx for s in sizes):
        return out
    return torch.cat([out[r * mx: r * mx + sizes[r]] for r in range(world)])


def sample_sharded(sample_fn: Callable[..., torch.Tensor], total: int, cond: Optional[Dict] = None, group=None, **kw) -> torch.Tensor:
    """sample_fn(batch_size=, cond=, b_global0=, **kw) -> (b, S) ids on this rank's device; returns all `total` layouts.
    A sample_fn with a `total_layouts` parameter gets the global batch size: torch-generator noise draws each shard's slice of
    the whole batch's draw."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    lo, hi = shard_bounds(total, world, rank)
    if "total_layouts" in inspect.signature(sample_fn).parameters:
        kw["total_layouts"] = total
    local = sample_fn(batch_size=hi - lo, cond=shard_cond(cond, lo, hi), b_global0=lo, **kw)
    return all_gather_ids(local, total, group)
