"""Data-parallel execution over the GPUs of one box: one process per GPU, weights replicated, the batch sharded
contiguously, and exactly one collective -- an all-gather of the [B_local, num_classes] logits.

The encoder has no cross-sample operation (no BatchNorm; reference vit.py / simple_vit.py), so nothing else is
exchanged.  Backend: NCCL over NVLink/NVSwitch on GPUs, gloo in the CPU tests.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist


def shard_bounds(total: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous [lo, hi) slice of `total` items owned by `rank`; the first (total % world) ranks get one extra."""
    if not (0 <= rank < world):
        raise ValueError(f"rank {rank} outside world {world}")
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_sizes(total: int, world: int) -> List[int]:
    return [shard_bounds(total, r, world)[1] - shard_bounds(total, r, world)[0] for r in range(world)]


def balanced_bounds(costs: Sequence[float], world: int) -> List[Tuple[int, int]]:
    """Contiguous [lo, hi) slices of a list of items with per-item `costs`, one per rank, minimising the largest
    slice cost (binary search on the bottleneck + greedy fill).  For NaViT the
    items are images and the cost of an image with n tokens is `navit_image_cost(n, ...)`: an even split by image
    COUNT can leave one rank with several times the tokens of another.  Every rank computes the same bounds."""
    n = len(costs)
    if world <= 0:
        raise ValueError("world must be positive")
    if n == 0:
        return [(0, 0)] * world

    def parts_needed(cap: float) -> int:
        parts, acc = 1, 0.0
        for c in costs:
            if acc + c > cap and acc > 0.0:
                parts, acc = parts + 1, 0.0
            acc += c
        return parts

    lo, hi = float(max(costs)), float(sum(costs))
    for _ in range(60):                              # smallest cap for which `world` slices suffice
        mid = 0.5 * (lo + hi)
        if parts_needed(mid) <= world:
            hi = mid
        else:
            lo = mid
    cap = hi * (1 + 1e-9)
    bounds, start, acc = [], 0, 0.0
    for i, c in enumerate(costs):
        if acc + c > cap and acc > 0.0:
            bounds.append((start, i))
            start, acc = i, 0.0
        acc += c
    bounds.append((start, n))
    assert len(bounds) <= world
    bounds += [(n, n)] * (world - len(bounds))      # fewer non-empty slices than ranks: the rest get nothing
    return bounds


def navit_image_cost(tokens: int, dim: int, mlp_dim: int, inner_dim: int) -> float:
    """Multiply-accumulates of one image per encoder layer: the GEMMs are linear in its token count, its attention
    quadratic (block-diagonal: tokens only attend inside their image, reference na_vit.py:335-337)."""
    return float(tokens) * (3 * dim * inner_dim + inner_dim * dim + 2 * dim * mlp_dim) + 2.0 * tokens * tokens * inner_dim


def all_gather_logits(local: torch.Tensor, total: Optional[int] = None,
                      group: Optional[dist.ProcessGroup] = None,
                      sizes: Optional[Sequence[int]] = None) -> torch.Tensor:
    """Gather per-rank logits [B_r, C] into [sum_r B_r, C] on every rank, rank order = batch order.

    Equal shards (the benchmark case) use a single all_gather_into_tensor on the current stream; ragged shards
    (total % world != 0 with sizes from shard_sizes, or explicit per-rank `sizes` -- the balanced NaViT split) pad to
    the largest shard and trim after the one collective."""
    if not (dist.is_available() and dist.is_initialized()):
        return local
    world = dist.get_world_size(group)
    if world == 1:
        return local
    local = local.contiguous()
    if sizes is not None:
        sizes = [int(v) for v in sizes]
        if len(sizes) != world or sizes[dist.get_rank(group)] != local.shape[0]:
            raise ValueError(f"sizes {sizes} do not describe this world / this rank's {local.shape[0]} rows")
    elif total is None or total % world == 0:
        out = torch.empty((local.shape[0] * world,) + tuple(local.shape[1:]), device=local.device, dtype=local.dtype)
        dist.all_gather_into_tensor(out, local, group=group)
        return out
    else:
        sizes = shard_sizes(total, world)
    mx = max(max(sizes), 1)
    pad = torch.zeros((mx,) + tuple(local.shape[1:]), device=local.device, dtype=local.dtype)
    pad[: local.shape[0]] = local
    out = torch.empty((mx * world,) + tuple(local.shape[1:]), device=local.device, dtype=local.dtype)
    dist.all_gather_into_tensor(out, pad, group=group)
    return torch.cat([out[r * mx: r * mx + sizes[r]] for r in range(world)], dim=0)


@torch.no_grad()
def data_parallel_forward(model: torch.nn.Module, local_images: torch.Tensor, total: Optional[int] = None,
                          group: Optional[dist.ProcessGroup] = None) -> torch.Tensor:
    """Forward this rank's shard and return the logits of the WHOLE batch on every rank."""
    return all_gather_logits(model(local_images), total=total, group=group)


@torch.no_grad()
def navit_data_parallel_forward(model: torch.nn.Module, images: Sequence[torch.Tensor],
                                group: Optional[dist.ProcessGroup] = None) -> torch.Tensor:
    """NaViT over the GPUs of one box: every rank holds the same LIST of variable-resolution images (or at least their
    shapes and its own slice's pixels), takes the contiguous slice that balances the per-layer work
    (`balanced_bounds` over `navit_image_cost`), runs it through the padding-free path and all-gathers the logits --
    one collective, output in the input order on every rank."""
    world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
    rank = dist.get_rank(group) if world > 1 else 0
    p = model.patch_size
    attn, ff = model.transformer.layers[0][0], model.transformer.layers[0][1]
    dim = model.pos_embed_height.shape[1]
    inner = attn.to_q.weight.shape[0]
    mlp = next(m for m in ff.modules() if isinstance(m, torch.nn.Linear)).weight.shape[0]
    costs = [navit_image_cost((im.shape[-2] // p) * (im.shape[-1] // p), dim, mlp, inner) for im in images]
    bounds = balanced_bounds(costs, world)
    lo, hi = bounds[rank]
    classes = model.mlp_head[-1].weight.shape[0]
    ref = images[0]
    if hi > lo:
        local = model(list(images[lo:hi]))
    else:
        local = torch.empty(0, classes, device=ref.device, dtype=ref.dtype)
    return all_gather_logits(local, group=group, sizes=[b - a for a, b in bounds])
