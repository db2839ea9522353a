"""sige_b200 — H100-native (sm_90a) implementation of SIGE's tile-sparse
gather -> conv -> scatter hot path behind the reference's operator surface.

    sige_b200.nn       SIGEModel / SIGEModule / SIGEConv2d / Gather / Scatter /
                       ScatterWithBlockResidual / ScatterGather   (reference sige/nn)
    sige_b200.masks    reduce_mask / dilate_mask / compute_difference_mask / downsample_mask
                       (reference sige/utils.py)
    sige_b200.ops      torch-facing wrappers of the C-ABI (include/sige_b200.h)
    sige_b200.lazy     deferred execution: one forward recorded on lazy tensor handles
    sige_b200.fused    that tape lowered to one fused launch per layer + CUDA graph (what SIGEModel runs in sparse mode)

``import sige`` (the thin alias package at the repo root) exposes the same objects under the
reference's module paths, so unmodified model files keep working.
"""
__version__ = "0.3.0+b200.1"

from . import masks, nn  # noqa: E402,F401
