"""Batch-parallel (one process per GPU) helpers.

Every mixture is independent end to end (all reductions of the forward are
within a sample), so the path shards by splitting the batch; there is NO
collective inside the step.  The only communication is ONE broadcast of the
weights at load time -- the H100-native replacement for ``nn.DataParallel``'s
per-forward module replication (run_improved_sudormrf.py:118 of the reference).
"""
from __future__ import annotations

from typing import Tuple

import torch
import torch.distributed as dist


def shard_bounds(total: int, world_size: int, rank: int) -> Tuple[int, int]:
    """Contiguous split of ``total`` mixtures over ``world_size`` ranks (the first
    ``total % world_size`` ranks take one extra), like DataParallel's scatter on dim 0."""
    if not (0 <= rank < world_size) or total < 0:
        raise ValueError("bad shard request")
    base, rem = divmod(total, world_size)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def broadcast_parameters(model: torch.nn.Module, src: int = 0, group=None) -> int:
    """One flat broadcast of every parameter from ``src`` (NCCL over NVLink on the
    GPU box, gloo in the CPU tests).  Returns the number of bytes broadcast."""
    params = [p for p in model.parameters()]
    if not params:
        return 0
    flat = torch.cat([p.detach().reshape(-1).to(torch.float32) for p in params])
    dist.broadcast(flat, src=src, group=group)
    off = 0
    with torch.no_grad():
        for p in params:
            n = p.numel()
            p.copy_(flat[off:off + n].view_as(p))
            off += n
    return flat.numel() * 4


def gather_estimates(local: torch.Tensor, total: int, group=None) -> torch.Tensor:
    """Optional, outside the timed step: collect per-rank estimates [b_r, S, T] on every
    rank in batch order (ranks may hold different b_r)."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    sizes = [shard_bounds(total, world, r) for r in range(world)]
    pad = max(hi - lo for lo, hi in sizes)
    buf = local.new_zeros((pad,) + tuple(local.shape[1:]))
    buf[: local.shape[0]] = local
    parts = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(parts, buf, group=group)
    assert sizes[rank][1] - sizes[rank][0] == local.shape[0]
    return torch.cat([parts[r][: hi - lo] for r, (lo, hi) in enumerate(sizes)], dim=0)
