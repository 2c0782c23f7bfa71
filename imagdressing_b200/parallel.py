"""Multi-GPU leg of the path (SURVEY.md §8e): samples are independent, so the global batch is split contiguously
over ranks (one process per GPU), each rank runs garment pass + 50 steps with zero communication, and the output
latents meet in ONE all-gather (NCCL over NVLink between the GPUs; gloo in the CPU tests)."""
from __future__ import annotations

from typing import List, Tuple

import torch
import torch.distributed as dist


def shard_range(global_batch: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous [lo, hi) of the global batch owned by `rank` (first ranks take the remainder)."""
    base, rem = divmod(global_batch, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def sample_seeds(seed: int, lo: int, hi: int) -> List[int]:
    """Per-sample seeds derived from the GLOBAL sample index, so results do not depend on the rank count."""
    return [(seed * 1000003 + i) % (2 ** 63 - 1) for i in range(lo, hi)]


def gather_latents(local: torch.Tensor, global_batch: int) -> torch.Tensor:
    """All-gather of per-rank output latents [b_r, 4, h, w] -> [global_batch, 4, h, w] on every rank."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return local
    world = dist.get_world_size()
    sizes = [shard_range(global_batch, r, world) for r in range(world)]
    bmax = max(hi - lo for lo, hi in sizes)
    pad = torch.zeros(bmax, *local.shape[1:], device=local.device, dtype=local.dtype)
    pad[: local.shape[0]] = local
    out = torch.empty(world * bmax, *local.shape[1:], device=local.device, dtype=local.dtype)
    dist.all_gather_into_tensor(out, pad)
    if all(hi - lo == bmax for lo, hi in sizes):
        return out
    return torch.cat([out[r * bmax: r * bmax + (hi - lo)] for r, (lo, hi) in enumerate(sizes)], 0)
