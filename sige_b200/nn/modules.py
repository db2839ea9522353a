"""The SIGE operator modules: SIGEConv2d, Gather, Scatter, ScatterWithBlockResidual, ScatterGather.

Constructor and forward signatures, the attributes model code reads (``block_size``,
``active_indices``, ``offset``, ``model_stride``, ``kernel_size``, ``mask``, ``input_res``,
``mode``, ``cache_id``, ``sparse_update``) and the per-mode behaviour follow the reference
(sige/nn/base.py:80-92, gather.py:12-108, scatter.py:9-136, scatter_gather.py:10-117) so the
reference's DDPM / Stable-Diffusion / GauGAN model files import and run unmodified.  The sparse
branches call the sm_90a library through ``sige_b200.ops`` instead of ``sige.cuda``/cuDNN:

    Gather            -> sige_gather             (NCHW or channels-last, fp32/fp16/bf16)
    SIGEConv2d        -> sige_tile_conv          (tensor cores; channels % 64 == 0, fp16/bf16)
                         sige_tile_conv_generic  (CUDA cores; everything else, exact fp32)
    Scatter*          -> sige_scatter / sige_scatter_with_block_residual
    ScatterGather     -> sige_scatter_gather (+ sige_get_scatter_map at set_masks time)

Tile stacks follow the memory layout of the tensor they were gathered from, so a model kept in
the default NCHW layout sees exactly the reference's contiguous ``[B*N, C, R, S]`` stacks, and a
channels-last model gets the coalesced NHWC kernels.
"""
from __future__ import annotations

import warnings
from typing import Dict, Optional, Tuple, Union

import torch
from torch import nn
from torch.nn import functional as F

from .. import lazy, ops
from ..masks import reduce_mask, reduce_mask_batched
from .state import SIGEModule, SIGEModuleWrapper, bump_cache_generation


def activation(x: torch.Tensor, activation_name: str) -> torch.Tensor:
    """Pointwise activation by name (reference sige/nn/utils.py:4-16) — used by profile mode."""
    table = {
        "relu": torch.relu,
        "sigmoid": torch.sigmoid,
        "tanh": torch.tanh,
        "swish": lambda t: t * torch.sigmoid(t),
        "identity": lambda t: t,
    }
    if activation_name not in table:
        raise ValueError("Unknown activation: [%s]!!!" % activation_name)
    return table[activation_name](x)


def _dummy_like(probe: torch.Tensor, shape) -> torch.Tensor:
    """A tensor of `shape` whose value depends on `probe` (profile mode only: lets a tracing MAC
    counter follow the graph without running any tile kernel; reference gather.py:59-70)."""
    return probe.reshape(-1)[0] + torch.zeros(shape, dtype=probe.dtype, device=probe.device)


def _on(t: Optional[torch.Tensor], ref: torch.Tensor) -> Optional[torch.Tensor]:
    return t if (t is None or t.device == ref.device) else t.to(ref.device)


class SIGEConv2d(nn.Conv2d, SIGEModule):
    """nn.Conv2d that, in sparse/profile mode, convolves already-padded tile stacks with
    padding 0 (reference sige/nn/base.py:80-92)."""

    def __init__(self, *args, **kwargs):
        nn.Conv2d.__init__(self, *args, **kwargs)
        SIGEModule.__init__(self, call_super=False)
        self._packed = None  # (key, packed weight [taps, Cout, Cin], fp32 bias)

    def _packed_weight(self, dtype: torch.dtype, pad_cin: int = 0):
        """Packed weights for the tensor-core kernels; ``pad_cin`` > Cin appends zero input channels (exact)."""
        key = (self.weight.data_ptr(), self.weight._version, dtype, self.weight.device, pad_cin,
               None if self.bias is None else (self.bias.data_ptr(), self.bias._version))
        if self._packed is None or self._packed[0] != key:
            w = self.weight
            if pad_cin > w.shape[1]:
                w = F.pad(w.detach(), (0, 0, 0, 0, 0, pad_cin - w.shape[1]))
            wp = ops.pack_conv_weight(w, dtype)
            b32 = None if self.bias is None else self.bias.detach().float().contiguous()
            self._packed = (key, wp, b32)
        return self._packed[1], self._packed[2]

    def _sparse_forward(self, x: torch.Tensor) -> torch.Tensor:
        if lazy.is_lazy(x):      # deferred execution (sige_b200.fused): recorded, fused with its gather / scatter later
            ro = (x.shape[2] - self.dilation[0] * (self.kernel_size[0] - 1) - 1) // self.stride[0] + 1
            so = (x.shape[3] - self.dilation[1] * (self.kernel_size[1] - 1) - 1) // self.stride[1] + 1
            return lazy.record_module_call("sige.conv", self, (x,), (x.shape[0], self.out_channels, ro, so), x)
        if not x.is_cuda:
            raise RuntimeError("SIGEConv2d sparse mode needs a CUDA tensor (no CPU backend); got %s" % x.device)
        if isinstance(self.padding, str) or self.padding_mode != "zeros":
            raise NotImplementedError("SIGEConv2d: unsupported padding configuration")
        if x.shape[0] == 0:
            ro = (x.shape[2] - self.dilation[0] * (self.kernel_size[0] - 1) - 1) // self.stride[0] + 1
            so = (x.shape[3] - self.dilation[1] * (self.kernel_size[1] - 1) - 1) // self.stride[1] + 1
            return x.new_empty((0, self.out_channels, ro, so))
        if ops.tile_conv_tc_supported(x, self.weight, self.stride, self.dilation, self.groups):
            wp, b32 = self._packed_weight(x.dtype)
            was_nchw = ops.layout_of(x) != ops.NHWC
            out = ops.tile_conv_stack(x, wp, b32, self.kernel_size, self.stride[0])
            return out.contiguous() if was_nchw else out
        cin = self.weight.shape[1]
        if (x.dtype in (torch.float16, torch.bfloat16) and self.groups == 1 and cin % 64 != 0 and cin >= 8
                and ops.tile_conv_tc_supported(x, self.weight, self.stride, self.dilation, self.groups, ignore_cin=True)):
            # few-channel inputs on the tensor cores (GauGAN's 36-channel label maps, gaugan/models/sige_normalization.py): zero
            # channels are appended to the stack and to the weights — exact, and ~15x faster than the CUDA-core kernel
            cpad = (cin + 63) // 64 * 64
            wp, b32 = self._packed_weight(x.dtype, pad_cin=cpad)
            was_nchw = ops.layout_of(x) != ops.NHWC
            xp = torch.empty((x.shape[0], cpad, x.shape[2], x.shape[3]), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
            xp[:, :cin].copy_(x)
            xp[:, cin:].zero_()
            out = ops.tile_conv_stack(xp, wp, b32, self.kernel_size, self.stride[0])
            return out.contiguous() if was_nchw else out
        return ops.tile_conv_generic(x, self.weight, self.bias, self.stride, self.dilation, self.groups)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.mode == "full":
            return nn.Conv2d.forward(self, x)
        if self.mode == "sparse":
            return self._sparse_forward(x)
        if self.mode == "profile":
            return F.conv2d(x, self.weight, self.bias, self.stride, (0, 0), self.dilation, self.groups)
        raise self._unknown_mode()


class Gather(SIGEModule):
    """Cuts the halo-padded active tiles out of the full activation.

    Geometry (reference gather.py:26-43): for the paired conv (kernel k, stride s, padding p) and a
    requested block b, n = max(b - k, 0) // s; the effective block is n*s + k (warns if it had to be
    adjusted), consecutive tiles are (n+1)*s apart, and the tile frame is shifted by `offset`
    (defaults to p) so that the conv's own zero padding is reproduced by the zero halo."""

    def __init__(
        self,
        conv: nn.Conv2d,
        block_size: Union[int, Tuple[int, int]],
        offset: Optional[Union[int, Tuple[int, int]]] = None,
        activation_name: str = "identity",
        activation_first: bool = False,
        verbose: bool = False,
    ):
        super().__init__()
        want = (block_size, block_size) if isinstance(block_size, int) else tuple(block_size)
        k, s = conv.kernel_size, conv.stride
        per_tile = tuple(max(want[d] - k[d], 0) // s[d] for d in (0, 1))  # conv outputs per tile - 1
        block = tuple(per_tile[d] * s[d] + k[d] for d in (0, 1))
        if block != want:
            warnings.warn("Change the block size from (%d, %d) to (%d, %d)" % (*want, *block))
        self.model_stride = s
        self.kernel_size = k
        self.block_size = block
        self.block_stride = tuple((per_tile[d] + 1) * s[d] for d in (0, 1))
        if offset is None:
            self.offset = conv.padding
        else:
            self.offset = (offset, offset) if isinstance(offset, int) else offset
        self.activation_name = activation_name
        self.activation_first = activation_first
        self.verbose = verbose
        self.load_runtime("gather")
        self.input_res: Optional[Tuple[int, int]] = None
        self.active_indices: Optional[torch.Tensor] = None
        # a batch of INDEPENDENT EDITS (3-D masks [E, H, W] given to set_masks): active_indices is the concatenation of the
        # per-edit tile lists and tile_images[i] names the edit of tile i; None = the reference's shared tile list
        self.tile_images: Optional[torch.Tensor] = None

    def forward(self, x: torch.Tensor, scale: Optional[torch.Tensor] = None, shift: Optional[torch.Tensor] = None) -> torch.Tensor:
        self.check_dtype(x, scale, shift)
        self.check_dim(x, scale, shift)
        if self.mode == "full":
            # dense pass: nothing to cut, only remember which mask resolution this layer needs
            assert scale is None and shift is None
            self.input_res = x.shape[2:]
            return x
        if self.mode == "sparse":
            if lazy.is_lazy(x, scale, shift):
                n = self.active_indices.size(0)
                rows = n if self.tile_images is not None else x.shape[0] * n
                return lazy.record_module_call("sige.gather", self, (x, scale, shift), (rows, x.shape[1], *self.block_size), x)
            self._no_batched_edits()
            idx = self.active_indices = _on(self.active_indices, x)
            return ops.gather(x, self.block_size[0], self.block_size[1], idx, scale, shift, self.activation_name,
                              self.activation_first)
        if self.mode == "profile":
            b, c = x.shape[:2]
            out = _dummy_like(x, (b * self.active_indices.size(0), c, *self.block_size))
            if scale is not None:
                out = out * scale.reshape(-1)[0]
            if shift is not None:
                out = out + shift.reshape(-1)[0]
            return activation(out, self.activation_name)
        raise self._unknown_mode()

    def set_mask(self, masks: Dict, cache: Dict, timestamp: int):
        if self.timestamp == timestamp:
            return  # already visited in this set_masks call (a ScatterGather may get here first)
        super().set_mask(masks, cache, timestamp)
        assert self.input_res is not None, "run one `full` forward before set_masks"
        res = tuple(self.input_res)
        self.mask = masks[res]
        key = ("active_indices", *res, *self.block_size, *self.block_stride, *self.offset)
        if key not in cache:
            if self.mask.dim() == 3:      # [E, H, W]: one mask per edit
                cache[key] = reduce_mask_batched(self.mask, self.block_size, self.block_stride, self.offset)
            else:
                cache[key] = (reduce_mask(self.mask, self.block_size, self.block_stride, self.offset, verbose=self.verbose), None)
        self.active_indices, self.tile_images = cache[key]

    @property
    def num_edits(self) -> Optional[int]:
        return None if self.tile_images is None else int(self.mask.shape[0])

    def _no_batched_edits(self):
        if self.tile_images is not None:
            raise NotImplementedError("a batch of independent edits (3-D masks) runs as a fused step only: CUDA fp16/bf16 "
                                      "(or set_fused(True, dtype=...)); the eager operator modules share one tile list across the batch")


def prefill_active_indices(modules, masks: Dict, cache: Dict) -> int:
    """All mask reductions of one ``set_masks`` call with ONE host synchronisation: every distinct (resolution, tile
    geometry) of the model's Gathers is launched first, then the counts come back in a single device->host copy (the
    reference pays one ``torch.nonzero`` sync per geometry, sige/utils.py:30).  Fills `cache` with the entries
    ``Gather.set_mask`` looks up.  Returns the number of launches."""
    pending = []
    for g in modules:
        if not isinstance(g, Gather) or g.input_res is None:
            continue
        res = tuple(g.input_res)
        mask = masks.get(res)
        if mask is None or not mask.is_cuda or mask.dim() != 2:
            continue
        key = ("active_indices", *res, *g.block_size, *g.block_stride, *g.offset)
        if key in cache or any(k == key for k, _, _ in pending):
            continue
        m = (mask > 0.5) if mask.is_floating_point() else (mask != 0)      # same binarisation as masks.reduce_mask
        out, count = ops.reduce_mask_cuda_launch(m, g.block_size, g.block_stride, g.offset)
        pending.append((key, out, count))
    if pending:
        counts = torch.cat([c for _, _, c in pending]).cpu().tolist()      # the one sync
        for (key, out, _), n in zip(pending, counts):
            cache[key] = (out[:n].contiguous(), None)
    return len(pending)


class Scatter(SIGEModule):
    """Pastes the conv's output tiles into (a copy of) the cached original output
    (reference scatter.py:9-63)."""

    def __init__(self, gather: Gather):
        super().__init__()
        self.gather = SIGEModuleWrapper(gather)
        self.load_runtime("scatter")
        self.output_res = None
        self.original_outputs: Dict[int, torch.Tensor] = {}

    def clear_cache(self):
        self.original_outputs = {}

    def forward(self, x: torch.Tensor, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
        self.check_dtype(x, residual)
        self.check_dim(x, residual)
        if self.mode == "full":
            out = x if residual is None else x + residual
            self.output_res = out.shape[2:]
            self.original_outputs[self.cache_id] = out if ops.layout_of(out) >= 0 else out.contiguous()
            bump_cache_generation()
            return out
        if self.mode == "sparse":
            g = self.gather.module
            cached = self.original_outputs[self.cache_id]
            if lazy.is_lazy(x, residual):
                shape = tuple(cached.shape) if g.num_edits is None else (g.num_edits, *cached.shape[1:])
                return lazy.record_module_call("sige.scatter", self, (x, residual), shape, x if lazy.is_lazy(x) else residual)
            g._no_batched_edits()
            out = ops.scatter(x, cached, g.offset[0], g.offset[1], g.model_stride[0], g.model_stride[1],
                              _on(g.active_indices, x), residual)
            if self.sparse_update:
                cached.copy_(out)
            return out
        if self.mode == "profile":
            cached = self.original_outputs[self.cache_id]
            out = _dummy_like(x, (cached.size(0), x.shape[1], *self.output_res))
            return out if residual is None else out + residual
        raise self._unknown_mode()


class ScatterWithBlockResidual(SIGEModule):
    """Scatter for residual blocks whose shortcut is itself a sparse 1x1 conv: main tiles are added
    to the cached shortcut output, then the shortcut's own tiles are corrected by
    (fresh - cached) (reference scatter.py:66-136)."""

    def __init__(self, main_gather: Gather, shortcut_gather: Gather):
        super().__init__()
        self.main_gather = SIGEModuleWrapper(main_gather)
        self.shortcut_gather = SIGEModuleWrapper(shortcut_gather)
        self.load_runtime("scatter_with_block_residual")
        self.scatter_runtime = None
        self.output_res = None
        self.original_outputs: Dict[int, torch.Tensor] = {}
        self.original_residuals: Dict[int, torch.Tensor] = {}

    def clear_cache(self):
        self.original_outputs = {}
        self.original_residuals = {}

    def forward(self, x: torch.Tensor, residual: torch.Tensor) -> torch.Tensor:
        self.check_dtype(x, residual)
        self.check_dim(x, residual)
        if self.mode == "full":
            out = x + residual
            self.output_res = out.shape[2:]
            self.original_outputs[self.cache_id] = out if ops.layout_of(out) >= 0 else out.contiguous()
            self.original_residuals[self.cache_id] = residual if ops.layout_of(residual) >= 0 else residual.contiguous()
            bump_cache_generation()
            return out
        if self.mode == "sparse":
            mg, sg = self.main_gather.module, self.shortcut_gather.module
            y0, y1 = self.original_outputs[self.cache_id], self.original_residuals[self.cache_id]
            if lazy.is_lazy(x, residual):
                shape = tuple(y0.shape) if mg.num_edits is None else (mg.num_edits, *y0.shape[1:])
                return lazy.record_module_call("sige.scatter_block_residual", self, (x, residual), shape, x if lazy.is_lazy(x) else residual)
            mg._no_batched_edits()
            idx0, idx1 = _on(mg.active_indices, x), _on(sg.active_indices, x)
            out = ops.scatter_with_block_residual(x, y0, residual, y1, mg.offset[0], mg.offset[1], mg.model_stride[0],
                                                  mg.model_stride[1], idx0, idx1)
            if self.sparse_update:
                y0.copy_(out)
                ops.scatter(residual, y1, sg.offset[0], sg.offset[1], sg.model_stride[0], sg.model_stride[1], idx1, None,
                            inplace=True)
            return out
        if self.mode == "profile":
            cached = self.original_outputs[self.cache_id]
            return _dummy_like(x, (cached.size(0), x.shape[1], *self.output_res)) + residual.reshape(-1)[0]
        raise self._unknown_mode()


class ScatterGather(SIGEModule):
    """Between two sparse convs: conceptually scatters conv1's tiles into the cached activation and
    immediately gathers conv2's halo tiles, without materialising the full tensor
    (reference scatter_gather.py:10-117)."""

    def __init__(self, gather: Gather, activation_name: str = "identity", activation_first: bool = False):
        super().__init__()
        self.gather = SIGEModuleWrapper(gather)
        self.activation_name = activation_name
        self.activation_first = activation_first
        self.load_runtime("scatter_gather")
        self.scatter_runtime = self.load_runtime("scatter", {})
        self.get_scatter_map_runtime = self.load_runtime("get_scatter_map", {})
        self.scatter_map = None
        self.output_res = None
        self.original_outputs: Dict[int, torch.Tensor] = {}

    def clear_cache(self):
        self.original_outputs = {}

    def forward(self, x: torch.Tensor, scale: Optional[torch.Tensor] = None, shift: Optional[torch.Tensor] = None) -> torch.Tensor:
        self.check_dtype(x, scale, shift)
        self.check_dim(x, scale, shift)
        g = self.gather.module
        if self.mode == "full":
            self.output_res = x.shape[2:]
            self.original_outputs[self.cache_id] = x if ops.layout_of(x) >= 0 else x.contiguous()
            bump_cache_generation()
            return x
        if self.mode == "sparse":
            cached = self.original_outputs[self.cache_id]
            if lazy.is_lazy(x, scale, shift):
                n = g.active_indices.size(0)
                rows = n if g.tile_images is not None else cached.size(0) * n
                return lazy.record_module_call("sige.scatter_gather", self, (x, scale, shift), (rows, x.shape[1], *g.block_size), x)
            g._no_batched_edits()
            idx = _on(g.active_indices, x)
            self.scatter_map = _on(self.scatter_map, x)
            out = ops.scatter_gather(x, cached, g.block_size[0], g.block_size[1], idx, self.scatter_map, scale, shift,
                                     self.activation_name, self.activation_first)
            if self.sparse_update:
                ops.scatter(x, cached, g.offset[0], g.offset[1], g.model_stride[0], g.model_stride[1], idx, None, inplace=True)
            return out
        if self.mode == "profile":
            cached = self.original_outputs[self.cache_id]
            out = _dummy_like(x, (cached.size(0) * g.active_indices.size(0), x.shape[1], *g.block_size))
            if scale is not None:
                out = out * scale.reshape(-1)[0]
            if shift is not None:
                out = out + shift.reshape(-1)[0]
            return activation(out, self.activation_name)
        raise self._unknown_mode()

    def set_mask(self, masks: Dict, cache: Dict, timestamp: int):
        if self.timestamp == timestamp:
            return
        super().set_mask(masks, cache, timestamp)
        g = self.gather.module
        g.set_mask(masks, cache, timestamp)  # the paired gather owns the index list
        if g.tile_images is not None:         # batch of independent edits: fused step only, which needs no scatter map
            self.scatter_map = None
            return
        h, w = g.mask.shape
        key = ("scatter_map", h, w, *g.block_size, *g.kernel_size, *g.offset, *g.model_stride)
        if key not in cache:
            idx = g.active_indices
            if idx.is_cuda:
                cache[key] = ops.get_scatter_map(h, w, g.block_size[0], g.block_size[1], g.kernel_size[0], g.kernel_size[1],
                                                 g.offset[0], g.offset[1], g.model_stride[0], g.model_stride[1], idx)
            else:
                cache[key] = _scatter_map_host(h, w, g.block_size, g.kernel_size, g.offset, g.model_stride, idx)
        self.scatter_map = cache[key]


def _scatter_map_host(h, w, block, kernel, offset, stride, idx: torch.Tensor) -> torch.Tensor:
    """Host-side scatter map for CPU index lists (set_masks on CPU masks; moved to the GPU lazily).
    Same definition as sige_get_scatter_map: (tile id, r, s) of the output tile covering each pixel, else -1."""
    out = torch.full((h, w, 3), -1, dtype=torch.int32)
    ro, so = (block[0] - kernel[0]) // stride[0] + 1, (block[1] - kernel[1]) // stride[1] + 1
    n = idx.shape[0]
    if n == 0:
        return out
    oy = torch.div(offset[0] + idx[:, 0].long(), stride[0], rounding_mode="trunc")
    ox = torch.div(offset[1] + idx[:, 1].long(), stride[1], rounding_mode="trunc")
    r, s = torch.arange(ro), torch.arange(so)
    hh = (oy[:, None, None] + r[None, :, None]).expand(n, ro, so)
    ww = (ox[:, None, None] + s[None, None, :]).expand(n, ro, so)
    tid = torch.arange(n)[:, None, None].expand(n, ro, so)
    rr, ss = r[None, :, None].expand(n, ro, so), s[None, None, :].expand(n, ro, so)
    ok = (hh >= 0) & (hh < h) & (ww >= 0) & (ww < w)
    vals = torch.stack((tid[ok], rr[ok], ss[ok]), dim=1).to(torch.int32)
    out[hh[ok], ww[ok]] = vals
    return out
