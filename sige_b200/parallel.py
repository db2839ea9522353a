"""Multi-GPU plumbing: edits are independent, so the only exchange is ONE broadcast of the cached
original-image state before the step loop (SURVEY.md §8e).  No collective on the per-step path.

The reference has no distributed code at all (SURVEY.md §2.3); this is the green-field multi-GPU part:
one process per GPU, NCCL over NVLink / NVSwitch through torch.distributed (gloo in CPU tests).
"""
from __future__ import annotations

from typing import List, Tuple

import torch
import torch.distributed as dist

from .nn import Scatter, ScatterGather, ScatterWithBlockResidual


def cache_tensors(model) -> List[Tuple[str, torch.Tensor]]:
    """Every tensor that the dense pass on the ORIGINAL image leaves behind and the sparse pass reads:
    Scatter*/ScatterGather caches and the folded GroupNorm (scale, shift) vectors — in a
    deterministic (module, key) order that is identical on all ranks."""
    found: List[Tuple[str, torch.Tensor]] = []
    for name, m in model.named_modules():
        if isinstance(m, (Scatter, ScatterGather)):
            for cid in sorted(m.original_outputs):
                found.append(("%s.out.%s" % (name, cid), m.original_outputs[cid]))
        elif isinstance(m, ScatterWithBlockResidual):
            for cid in sorted(m.original_outputs):
                found.append(("%s.out.%s" % (name, cid), m.original_outputs[cid]))
                found.append(("%s.res.%s" % (name, cid), m.original_residuals[cid]))
        for attr in ("scale1s", "shift1s", "scale2s", "shift2s", "scales", "shifts"):
            v = getattr(m, attr, None)
            if isinstance(v, dict):
                for cid in sorted(v):
                    found.append(("%s.%s.%s" % (name, attr, cid), v[cid]))
            elif isinstance(v, torch.Tensor):
                found.append(("%s.%s" % (name, attr), v))
    return found


def broadcast_caches(model, src: int = 0, group=None) -> int:
    """Overwrite every rank's caches with rank `src`'s, using a single flat broadcast.  Returns the
    number of bytes sent per receiving rank."""
    items = cache_tensors(model)
    if not items:
        return 0
    by_dtype = {}
    for _, t in items:
        by_dtype.setdefault(t.dtype, []).append(t)
    total = 0
    for dtype, tensors in by_dtype.items():
        flat = torch.cat([t.reshape(-1) if t.is_contiguous() else t.contiguous(memory_format=torch.channels_last).permute(0, 2, 3, 1).reshape(-1)
                          for t in tensors])
        dist.broadcast(flat, src=src, group=group)
        total += flat.numel() * flat.element_size()
        off = 0
        for t in tensors:
            n = t.numel()
            chunk = flat[off:off + n]
            if t.is_contiguous():
                t.copy_(chunk.view_as(t))
            else:  # channels-last cache: the flat order is its physical (N, H, W, C) order
                b, c, h, w = t.shape
                t.copy_(chunk.view(b, h, w, c).permute(0, 3, 1, 2))
            off += n
    return total


def shard_edits(num_edits: int, rank: int, world: int) -> List[int]:
    """Edit e runs on GPU e mod world (SURVEY.md §8e)."""
    return [e for e in range(num_edits) if e % world == rank]
