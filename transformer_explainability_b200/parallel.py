"""Multi-GPU plumbing: one process per GPU, the batch sharded embarrassingly, ONE collective.

Every explanation is independent (and must be computed independently, SURVEY.md §0-6), so the only
exchange on the path is the start-up broadcast of the flat frozen-weight buffer from rank 0 (NCCL over
NVLink / NVSwitch on a multi-GPU H100 node; gloo in the CPU tests).  No collective runs on the per-sample path;
results are gathered with one small all_gather of [B/G, N] maps when the caller asks for it.
"""
import os

import torch
import torch.distributed as dist


def shard_range(total, rank, world):
    """Contiguous slice [lo, hi) of ``total`` items owned by ``rank``; sizes differ by at most one."""
    if world <= 0 or not (0 <= rank < world):
        raise ValueError("bad rank/world")
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def init_from_env(backend=None):
    """Initialise torch.distributed from torchrun's env (RANK / WORLD_SIZE / MASTER_*); no-op if single process."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world <= 1:
        return 0, 1, 0
    rank = int(os.environ["RANK"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    if not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
        dist.init_process_group(backend=backend)
    return rank, world, local


def broadcast_flat_weights(weights, src=0, group=None):
    """The single collective of the path: broadcast the flat fp32 weight buffer (346 MB ViT-B, 1.2 GB ViT-L)."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.broadcast(weights, src=src, group=group)
    return weights


def gather_maps(local_maps, total, group=None):
    """all_gather of per-rank [b_r, N] results into [total, N] (ragged shards padded to the largest)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return local_maps
    world = dist.get_world_size(group)
    biggest = (total + world - 1) // world
    pad = torch.zeros(biggest, local_maps.shape[1], dtype=local_maps.dtype, device=local_maps.device)
    pad[:local_maps.shape[0]] = local_maps
    out = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(out, pad, group=group)
    parts = []
    for r in range(world):
        lo, hi = shard_range(total, r, world)
        parts.append(out[r][:hi - lo])
    return torch.cat(parts, dim=0)


def explain_sharded(engine, images, index=None, start_layer=0, gather=False, chunk=None, graph=False):
    """Run this rank's contiguous shard of ``images`` through ``engine.explain``.
    ``images`` may be the full batch (sliced here) — per-rank result, or the gathered [B,N] if ``gather``.
    graph: replay the shard's step from a CUDA graph (``ViTEngine.explain_graphed``) — small shards of a fixed global
    batch are otherwise bound by launch gaps."""
    rank = dist.get_rank() if dist.is_initialized() else 0
    world = dist.get_world_size() if dist.is_initialized() else 1
    total = images.shape[0]
    lo, hi = shard_range(total, rank, world)
    idx = None if index is None else torch.as_tensor(index)[lo:hi]
    if graph and hasattr(engine, "explain_graphed"):
        maps, cls = engine.explain_graphed(images[lo:hi], index=idx, start_layer=start_layer)
    else:
        maps, cls = engine.explain(images[lo:hi], index=idx, start_layer=start_layer, chunk=chunk)
    if gather:
        return gather_maps(maps, total), cls
    return maps, cls
