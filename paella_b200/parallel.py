"""Multi-GPU plumbing for the sampling path: one process per GPU, batch sharding, one weight broadcast.

The path shards by sample — every latent grid in the batch is independent (GRN, LayerNorm and attention are
per sample; BatchNorm is eval-mode affine), so there is NO collective inside the step loop.  The only
communication is (1) one broadcast of the packed weight blob at start-up (NCCL over NVLink on the GPU box;
gloo in the CPU tests) and (2) an optional final all-gather of the sampled token grids (B*H*W*8 bytes).
"""
from __future__ import annotations

from typing import List, Tuple

import torch
import torch.distributed as dist


def shard_range(n: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous [lo, hi) slice of ``n`` samples owned by ``rank``; sizes differ by at most one."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def rank_seed(base_seed: int, rank: int) -> int:
    """Per-shard generator seed.  Multi-GPU parity is defined per shard against a single-GPU run of that
    shard with this seed (SURVEY.md §8e).  With per-sample generators instead (``sample(..., generator=generators)``), a
    shard given ``generators[lo:hi]`` draws exactly what rows [lo, hi) of the single-GPU run draw, whatever the shard
    layout, and reproduces their tokens exactly where the forward is batch-invariant (DESIGN.md §3: on the default model with
    ``model.batch_invariant = True`` on every rank)."""
    return base_seed + rank


def blob_checksum(blob: torch.Tensor) -> torch.Tensor:
    """64-bit wrap-around sum of the whole blob viewed as int64 words (+ the tail bytes): one pass over HBM."""
    flat = blob.reshape(-1).view(torch.uint8)
    n8 = flat.numel() // 8 * 8
    s = flat[:n8].view(torch.int64).sum()
    if n8 < flat.numel():
        s = s + flat[n8:].to(torch.int64).sum()
    return s.reshape(1)


def assert_same_across_ranks(value: torch.Tensor, what: str = "value") -> None:
    """Every rank holds the same int64 ``value`` (one tiny all-reduce: max(v) == -max(-v)), else raise on every rank."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return
    v = value.reshape(-1).to(torch.int64)
    both = torch.cat([v, -v])
    dist.all_reduce(both, op=dist.ReduceOp.MAX)
    n = v.numel()
    if not torch.equal(both[:n], -both[n:]):
        raise RuntimeError(f"rank {dist.get_rank()}: {what} differs between ranks (max {both[:n].tolist()}, min {(-both[n:]).tolist()}, "
                           f"mine {v.tolist()})")


def broadcast_blob(blob: torch.Tensor, src: int = 0, verify: bool = True) -> torch.Tensor:
    """The one collective of a multi-GPU run: the packed (fp16/fp32) weight blob, rank ``src`` -> all, followed by a
    checksum agreement check (non-source ranks start from zeros: a short or skipped broadcast must not go unnoticed)."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.broadcast(blob, src=src)
        if verify:
            assert_same_across_ranks(blob_checksum(blob), "packed weight blob checksum after broadcast")
    return blob


def gather_tokens(local_tokens: torch.Tensor, sizes: List[int]) -> torch.Tensor:
    """All-gather the per-rank token grids [b_r, H, W] into [sum b_r, H, W] in rank order (ragged shards padded)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return local_tokens
    world = dist.get_world_size()
    mx = max(sizes)
    pad = torch.zeros((mx,) + tuple(local_tokens.shape[1:]), dtype=local_tokens.dtype, device=local_tokens.device)
    pad[: local_tokens.shape[0]] = local_tokens
    out = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(out, pad)
    return torch.cat([o[:s] for o, s in zip(out, sizes)], dim=0)
