"""Data-parallel plumbing for independent images (SURVEY section 8e): every image (seed) is an independent two-stage
trajectory, so images are sharded round-robin over ranks with NO collective inside the denoising loop.  The only
collectives are one broadcast of the weights from rank 0 at start-up and one all-gather of the final latents
(128 KiB per image).  torch.distributed (NCCL over NVLink between GPUs, gloo in the CPU tests) is the transport."""
from typing import Dict, List

import torch
import torch.distributed as dist


def shard_indices(n_items: int, rank: int, world: int) -> List[int]:
    """image j -> rank j mod world."""
    return list(range(rank, n_items, world))


def flat_layout(shapes: Dict[str, tuple], align: int = 128):
    """name -> (offset, numel) of a state dict packed into ONE flat buffer (deterministic key order, every tensor
    starts on an `align`-element boundary so that the views stay 256 B aligned for TMA), and the total length."""
    layout, off = {}, 0
    for k in sorted(shapes):
        n = 1
        for d in shapes[k]:
            n *= d
        layout[k] = (off, n)
        off += (n + align - 1) // align * align
    return layout, off


def flatten_state_dict(sd: Dict[str, torch.Tensor], dtype=torch.float16):
    """Pack a state dict into one contiguous buffer; returns (flat, views) where views alias the buffer."""
    shapes = {k: tuple(v.shape) for k, v in sd.items()}
    layout, total = flat_layout(shapes)
    dev = next(iter(sd.values())).device
    flat = torch.empty(total, dtype=dtype, device=dev)
    views = {}
    for k, (off, n) in layout.items():
        views[k] = flat[off:off + n].view(shapes[k])
        views[k].copy_(sd[k])
    return flat, views


def empty_flat_state_dict(shapes: Dict[str, tuple], device, dtype=torch.float16):
    """The receiving side of broadcast_flat: an uninitialised flat buffer with the same layout, and its views."""
    layout, total = flat_layout(shapes)
    flat = torch.empty(total, dtype=dtype, device=device)
    return flat, {k: flat[off:off + n].view(tuple(shapes[k])) for k, (off, n) in layout.items()}


def broadcast_flat(flat: torch.Tensor, src: int = 0) -> torch.Tensor:
    """ONE ncclBroadcast of the whole weight set (5.1 GB for the SDXL UNet: a few ms over NVLink; the per-tensor form
    issued ~1700 collectives and was launch-bound)."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.broadcast(flat, src=src)
    return flat


def broadcast_state_dict(sd: Dict[str, torch.Tensor], src: int = 0) -> Dict[str, torch.Tensor]:
    """Broadcast every tensor of `sd` (same keys/shapes on every rank) through one flat buffer per dtype group; the
    tensors are updated in place."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return sd
    flat, views = flatten_state_dict(sd, dtype=next(iter(sd.values())).dtype)
    broadcast_flat(flat, src)
    for k in sd:
        sd[k].copy_(views[k])
    return sd


def gather_latents(local: torch.Tensor, n_items: int) -> torch.Tensor:
    """local: (n_local, ...) latents of this rank's images in shard order -> (n_items, ...) in image order on every
    rank.  Ranks may hold different counts (n_items not divisible by world): shards are padded to the maximum."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return local
    world, rank = dist.get_world_size(), dist.get_rank()
    per = (n_items + world - 1) // world
    pad = torch.zeros((per, *local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    bufs = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(bufs, pad)
    out = torch.empty((n_items, *local.shape[1:]), dtype=local.dtype, device=local.device)
    for r in range(world):
        idx = shard_indices(n_items, r, world)
        out[idx] = bufs[r][: len(idx)]
    return out
