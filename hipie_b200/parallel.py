"""Data-parallel plumbing of the hot path: image sharding + the single all-gather of fixed-shape outputs.

The reference's inference is pure data parallel: each rank owns a contiguous shard of the dataset
(/root/reference/detectron2/data/samplers/distributed_sampler.py:245-278 `InferenceSampler._get_local_indices`) and
no collective is issued during the forward pass.  Here the global image batch is split the same way and the
fixed-shape per-image outputs (class logits, boxes, MaskDINO logits, optionally bit-packed masks) are all-gathered
once after the last kernel (NCCL over NVLink between GPUs; gloo in the CPU tests).
"""
from typing import Dict, List

import torch
import torch.distributed as dist


def shard_indices(total_size: int, world_size: int, rank: int) -> range:
    """Contiguous shards, the first `total_size % world_size` ranks get one extra item (InferenceSampler convention)."""
    shard_size = total_size // world_size
    left = total_size % world_size
    shard_sizes = [shard_size + int(r < left) for r in range(world_size)]
    begin = sum(shard_sizes[:rank])
    end = min(sum(shard_sizes[:rank + 1]), total_size)
    return range(begin, end)


def all_gather_outputs(out: Dict[str, torch.Tensor], keys: List[str], group=None) -> Dict[str, torch.Tensor]:
    """All-gather `out[k]` (leading dim = local images) into the global batch order.  Equal shard sizes use one
    `all_gather_into_tensor` per key; ragged shards are padded to the largest shard and trimmed."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return {k: out[k] for k in keys}
    world = dist.get_world_size(group)
    n_local = torch.tensor([out[keys[0]].shape[0]], device=out[keys[0]].device)
    counts = [torch.zeros_like(n_local) for _ in range(world)]
    dist.all_gather(counts, n_local, group=group)
    counts = [int(c) for c in counts]
    mx = max(counts)
    res = {}
    for k in keys:
        t = out[k].contiguous()
        if t.shape[0] < mx:
            pad = torch.zeros((mx - t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
            t = torch.cat([t, pad], 0)
        buf = torch.empty((world * mx,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        if dist.get_backend(group) == "nccl":
            dist.all_gather_into_tensor(buf, t, group=group)
        else:
            parts = list(buf.chunk(world, 0))
            dist.all_gather(parts, t, group=group)
        res[k] = torch.cat([buf[r * mx:r * mx + counts[r]] for r in range(world)], 0)
    return res


class PackedAllGather:
    """The data-parallel path's single collective: the fixed-shape per-image outputs of one step (class logits, boxes, IoU
    logits, MaskDINO logits / boxes) are packed into ONE preallocated buffer and exchanged with ONE all-gather per step
    (NCCL over NVLink / NVSwitch; gloo in the CPU tests) -- no count exchange, no host sync, no per-key launches.  Shards must be
    equal (the bench / serving case: every rank holds the same number of images); ragged shards go through all_gather_outputs."""

    def __init__(self, group=None):
        self.group = group
        self._layout = None
        self._send = None
        self._recv = None

    def __call__(self, out: Dict[str, torch.Tensor], keys: List[str]) -> Dict[str, torch.Tensor]:
        if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(self.group) == 1:
            return {k: out[k] for k in keys}
        world = dist.get_world_size(self.group)
        layout = tuple((k, tuple(out[k].shape)) for k in keys)
        dev = out[keys[0]].device
        if layout != self._layout:
            total = sum(out[k].numel() for k in keys)
            self._send = torch.empty(total, dtype=torch.float32, device=dev)
            self._recv = torch.empty(world * total, dtype=torch.float32, device=dev)
            self._layout = layout
        off = 0
        for k in keys:                       # pack (device-side copies into the static buffer)
            n = out[k].numel()
            self._send[off:off + n].copy_(out[k].reshape(-1))
            off += n
        if dist.get_backend(self.group) == "nccl":
            dist.all_gather_into_tensor(self._recv, self._send, group=self.group)
        else:
            parts = list(self._recv.chunk(world, 0))
            dist.all_gather(parts, self._send, group=self.group)
        total = self._send.numel()
        rv = self._recv.view(world, total)
        res, off = {}, 0
        for k in keys:                       # views into the receive buffer, global batch order = rank-major
            shp = tuple(out[k].shape)
            n = out[k].numel()
            res[k] = rv[:, off:off + n].reshape((world * shp[0],) + shp[1:])
            off += n
        return res
