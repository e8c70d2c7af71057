"""Multi-GPU plumbing for the batch-sharded path.

The path shards by image: every rank holds a full replica of the packed weights and
processes its own slice of the batch; there is exactly ONE collective, at load time
(rank 0 broadcasts one contiguous blob of packed filters + epilogue vectors), and
none on the step path. ``torch.distributed`` is the plumbing: NCCL over NVLink on
the GPU box, gloo in the CPU tests (``tests/test_parallel_gloo.py``).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist


def shard_range(rank: int, world: int, batch: int):
    """Images [lo, hi) of a global batch owned by `rank`: contiguous, sizes differ by
    at most one (config 3: 1024 / 8 = 128 per GPU)."""
    base, rem = divmod(batch, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def pack_weight_blob(layers):
    """Flatten [{filter:int32[...], mul:f32[C], bias:f32[C]} | {filter, thresholds}] into one
    int32 vector + a manifest of (shape, kind) so a single broadcast moves the model."""
    parts, manifest = [], []
    for lay in layers:
        entry = {}
        for key in ("filter", "mul", "bias", "thresholds"):
            if lay.get(key) is None:
                continue
            a = np.ascontiguousarray(lay[key])
            entry[key] = (a.shape, a.dtype.str)
            parts.append(a.reshape(-1).view(np.int32))
        manifest.append(entry)
    blob = np.concatenate(parts) if parts else np.zeros(0, np.int32)
    return blob, manifest


def unpack_weight_blob(blob: torch.Tensor, manifest):
    """Views into the (device or host) blob; no copies."""
    out, off = [], 0
    for entry in manifest:
        lay = {}
        for key, (shape, dtype) in entry.items():
            n = int(np.prod(shape)) if len(shape) else 1
            piece = blob[off:off + n]
            off += n
            if np.dtype(dtype) == np.float32:
                piece = piece.view(torch.float32)
            lay[key] = piece.view(*shape)
        out.append(lay)
    return out


def broadcast_model(layers, device, src=0):
    """Rank `src` passes its layers; every rank gets tensors on `device`. One
    broadcast of the manifest (host object) + ONE tensor broadcast of the weights."""
    world = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    if rank == src:
        blob_np, manifest = pack_weight_blob(layers)
        meta = [manifest, int(blob_np.size)]
    else:
        blob_np, meta = None, [None, 0]
    if world > 1:
        dist.broadcast_object_list(meta, src=src)
    manifest, n = meta
    blob = torch.empty(n, dtype=torch.int32, device=device)
    if rank == src:
        blob.copy_(torch.from_numpy(blob_np))
    if world > 1:
        dist.broadcast(blob, src=src)
    return unpack_weight_blob(blob, manifest), blob


def gather_outputs(local: torch.Tensor, batch: int):
    """Host-side concat of per-rank results in batch order ('outputs are
    copied D2H per rank and concatenated on the host' -- not a step collective)."""
    world = dist.get_world_size() if dist.is_initialized() else 1
    if world == 1:
        return local.cpu()
    pieces = [None] * world
    dist.all_gather_object(pieces, local.cpu())
    return torch.cat(pieces, dim=0)
