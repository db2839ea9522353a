"""Fused step: an UNMODIFIED model forward, traced once, executed as one fused sm_90a launch per layer.

``FusedStep(model, x, *more)`` runs ``model.forward`` once on lazy handles (``sige_b200.lazy``) in sparse
mode, lowers the recorded tape to a short program of launches and captures it in a CUDA graph.  The model is
any ``sige.nn.SIGEModel`` — the reference's own ``diffusion/models/ddpm_arch/sige_fused_unet.py`` drops in
unmodified (tests/test_gpu_reference_model.py); nothing here looks at model classes, only at the calls the
forward makes.

What the lowering recognises (everything else runs as an eager torch node inside the same graph, so any
traceable forward stays correct):

  Gather -> SIGEConv2d / nn.Conv2d -> Scatter          one ``sige_tile_conv`` launch: gather (+GroupNorm affine,
  (reference sige_fused_unet.py:100-131, 212-248)      +SiLU) -> wgmma conv -> (+bias, +residual) -> in-place
                                                        scatter into a persistent NHWC buffer initialised from the
                                                        module's cache (the reference's sparse_update form,
                                                        sige/nn/scatter.py:59-60: no clone)
  ... -> ScatterGather -> SIGEConv2d                    free: conv2 gathers from the buffer conv1 scattered into
  ScatterWithBlockResidual                              the 1x1 shortcut rides in conv2's launch as extra K chunks
  (sige/cuda/scatter_kernel.cu:46-74)                   (fresh where its own tile is active, cached elsewhere)
  torch.cat / F.interpolate(nearest, x2) / F.pad        folded into the consumer's gather stage (channel segments,
  (sige_fused_unet.py:423, :223, :244)                  half-resolution addressing, zero halo) — never materialised
  x*scale+shift, x*sigmoid(x), F.silu                   folded into the consumer conv's pre-op (written once by the
  (sige_fused_unet.py:112-123)                          PRODUCER's epilogue when it can, else applied in the gather)
  nn.Conv2d on a full tensor (dense low-res blocks)     the same kernel with an all-tiles index list; `+ x` and the
                                                        1x1 shortcut of a dense block join the conv's launch
  split/reshape/bmm/softmax/bmm attention core          ``sige_attention_tokens`` (one launch), c^-0.5 folded into
  (sige_fused_unet.py:185-199)                          the q rows of the qkv weights
  conv on the <=4-channel input image                   ``sige_conv_in_nhwc`` (restricted to the active tiles when
                                                        every reader gathers it through one index set)
  GroupNorm -> SiLU -> conv to <=8 channels             ``sige_group_norm_fold`` + ``sige_conv_out_nhwc``

Numerics: the same formulas as the operator-module path; the only reassociations are fp32 FMA for the affine, the
1x1 shortcut evaluated on every main tile whose shortcut tile is active instead of being patched by (fresh - cached),
and scalar / per-channel affines in front of a 1x1 conv folded exactly into its weights.

The executor is injected: ``CudaExecutor`` (libsige_b200.so through ``sige_b200.ops``) is the product; tests
inject a CPU simulator of the launch descriptors to check the lowering without a GPU.
"""
from __future__ import annotations

import copy
import ctypes
import math
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple

import torch
from torch import nn
from torch.nn import functional as F

from . import lazy
from .lazy import LazyTensor, Node, TraceUnsupported


# =====================================================================================================================
# program objects
# =====================================================================================================================
class Buf:
    """One activation of the step: an NHWC tensor (allocated on first request) plus pre-transformed views
    act(raw*scale+shift) that its PRODUCER writes for each consumer (so that consumers gather plain bytes)."""

    def __init__(self, owner: "Lowering", shape, cached_init: Optional[torch.Tensor] = None, raw: Optional[torch.Tensor] = None):
        self.owner = owner
        self.shape = tuple(int(s) for s in shape)            # (B, C, H, W)
        self.cached_init = cached_init                        # pristine values when only active tiles are rewritten per step
        self._raw = raw
        self.producers: List = []                             # objects with .can_aux() / .add_aux(view, scale, shift, act)
        self.readers: List = []                               # (idx, block, up) of fused launches reading it; None = a dense read
        self.views: Dict = {}
        self.view_inits: List = []                            # (view, scale, shift, act) of the views initialised from the cache

    @property
    def raw(self) -> torch.Tensor:
        if self._raw is None:
            if self.cached_init is not None:
                if self.owner.loads(self) and not self.owner.built:
                    self._raw = self.owner.empty(*self.shape)        # filled when the lowering ends (Lowering.load_caches)
                else:
                    self._raw = self.owner.clone_cache(self.cached_init, self.shape[0])
                self.owner.loader = None
            else:
                self._raw = self.owner.empty(*self.shape)
        return self._raw

    @property
    def has_raw(self) -> bool:
        return self._raw is not None

    def restore(self) -> None:
        """Back to the cached original values (a new edit starts from them): raw copy and every transformed view.  The torch
        restatement of `sige_cache_load`, for executors without it and caches it does not take."""
        if self.cached_init is None:
            return
        if self._raw is not None:
            c = self.cached_init.to(self._raw.device)
            self._raw.copy_(c if c.shape[0] == self.shape[0] else c.expand(self.shape[0], *c.shape[1:]))
        for (v, sc, sh, act) in self.view_inits:
            self.owner.init_view(v, self.cached_init, sc, sh, act)


class Derived:
    """A tensor the program reads that was derived from tensors taken from outside the tape (module caches, dense-pass
    statistics, parameters): ``out = fn(*srcs)``.  `FusedStep.refresh` re-runs ``fn`` on the sources' current values and
    copies the result into ``out``'s storage, which every launch keeps reading.  ``fn`` None: the sources are read as they are."""

    def __init__(self, fn: Optional[Callable], srcs: Sequence, out):
        self.fn, self.srcs, self.out = fn, tuple(srcs), out


class ConvSpec:
    """Everything one fused gather->conv->scatter launch needs, as tensors (the executor turns it into a descriptor)."""

    def __init__(self):
        self.name = ""
        self.srcs: List[Tuple[torch.Tensor, int]] = []       # (NHWC tensor, upsample flag); or the stack when src_is_stack
        self.src_is_stack = False
        self.B = 1
        self.H = self.W = 0
        self.idx: Optional[torch.Tensor] = None
        self.tile_img: Optional[torch.Tensor] = None         # int32 [N]: a batch of independent edits (image of each row of idx)
        self.slot: Optional["IdxSlot"] = None                # fixed-capacity index buffer (N = capacity, or E * capacity for a batch)
        self.N = 0
        self.block = 0
        self.scale: Optional[torch.Tensor] = None            # fp32 [Cin] or [B, Cin]
        self.shift: Optional[torch.Tensor] = None
        self.per_sample_affine = False
        self.act = "identity"
        self.weight: Optional[torch.Tensor] = None           # fp32 OIHW (after exact folds)
        self.bias: Optional[torch.Tensor] = None             # fp32 [Cout] or None
        self.weight_key = None                               # cache key of the packed form
        self.refold = False                                  # weight / bias fold dense-pass statistics (`Lowering.derive`)
        self.out_row_scale: Optional[Tuple[int, float]] = None
        self.k = 1
        self.stride = 1
        self.off = 0
        self.dst: Optional[Buf] = None
        self.dst_stack: Optional[torch.Tensor] = None        # destination is a tile stack (B*N, Cout, Ro, So) NHWC
        self.residual: Optional[torch.Tensor] = None
        self.aux: List[Tuple[torch.Tensor, Optional[torch.Tensor], Optional[torch.Tensor], str]] = []
        self.epilogue_act = "identity"                       # "relu": the destination holds relu(conv + bias [+ residual])
        self.modulation = None                               # (gamma, beta, slope): SPADE's modulation in the gather stage
        self.shortcut = None                                 # (src tensors, weight fp32 OI11, bias fp32, flags uint8 [N] or None)
        self.shortcut_key = None
        self.pdl = False
        self.tc5 = False
        self.ksplit = 0
        self.early = 0                                       # early source groups: SIGE_CONV_EARLY_* >> 4 (Lowering._early_masks)
        self.early_release = False                           # SIGE_CONV_EARLY_RELEASE: the next launch has early source groups

    @property
    def Cin(self) -> int:
        return int(self.weight.shape[1])

    @property
    def Cout(self) -> int:
        return int(self.weight.shape[0])


class FusedConv:
    """One prepared ``sige_tile_conv`` launch (prepared by the executor at finalize time)."""

    trace_hook = None        # development aid (tools/trace_graph.py)

    def __init__(self, spec: ConvSpec):
        self.spec = spec
        self.name = spec.name
        self.launch_fn: Optional[Callable[[int], None]] = None
        self.desc = None
        self.keep: List = []

    def can_aux(self) -> bool:
        # a ReLU epilogue writes its destination through the launch's aux slot, and a view would see the pre-ReLU value
        return len(self.spec.aux) < 2 and self.spec.epilogue_act == "identity"

    def add_aux(self, view: torch.Tensor, scale, shift, act: str) -> None:
        self.spec.aux.append((view, scale, shift, act))

    def launch(self, stream: int) -> None:
        if FusedConv.trace_hook is not None:
            FusedConv.trace_hook(self)
        self.launch_fn(stream)

    # ---- accounting (SURVEY.md §8d: algorithmic bytes / flops of one fused launch)
    @property
    def tiles(self) -> int:
        s = self.spec
        n = s.slot.n if s.slot is not None else s.N
        return n if s.tile_img is not None else s.B * n         # (a batch's lists hold the tiles of every edit)

    @property
    def out_elems(self) -> int:
        s = self.spec
        ro = (s.block - s.k) // s.stride + 1
        return self.tiles * s.Cout * ro * ro

    @property
    def bytes(self) -> int:
        s = self.spec
        n = self.tiles
        dsts = (1 if (s.dst is not None and s.dst.has_raw) or s.dst_stack is not None else 0) + (1 if s.residual is not None else 0) + len(s.aux)
        b = 2 * (n * s.Cin * s.block * s.block + s.k * s.k * s.Cout * s.Cin + self.out_elems * dsts)
        if s.shortcut is not None:
            c2 = int(s.shortcut[1].shape[1])
            b += 2 * (n * c2 * 16 + s.Cout * c2)
        if s.modulation is not None:
            b += 2 * 2 * n * s.Cin * s.block * s.block
        return b

    @property
    def flops(self) -> int:
        s = self.spec
        ro = (s.block - s.k) // s.stride + 1
        f = 2 * self.tiles * ro * ro * s.Cout * s.Cin * s.k * s.k
        if s.shortcut is not None:
            f += 2 * self.tiles * ro * ro * s.Cout * int(s.shortcut[1].shape[1])
        return f


class IdxSlot:
    """A tile list with a fixed capacity: the launches hold this buffer's address and N = capacity; entries beyond the current
    count are SIGE_TILE_NONE origins (such a tile reads zeros and writes nothing, include/sige_b200.h).  A new mask whose lists
    fit is installed by rewriting the buffers in place (`FusedStep.rebind`): no re-trace, no re-capture.

    A batch of E independent edits (the Gather has `tile_images`) gets one list of `cap` rows per edit: `buf` is [E*cap, 2], row
    e*cap + i = tile i of edit e (the per-image layout of sige_tile_conv_t.idx_per_image and of `sige_reduce_mask_batched`), and
    `tile_img` is the constant image index row // cap of every row.  `cap` is the longest list at build time, or with headroom
    that times (1 + headroom) rounded up to a multiple of 8, so that padding fills whole CTAs (SIGE_CONV_PADDED)."""

    def __init__(self, gather, dev, headroom: float = 0.0):
        from ._cabi import TILE_NONE

        self.gather = gather
        self.none = TILE_NONE
        timg = getattr(gather, "tile_images", None)
        self.E = 1 if timg is None else int(gather.num_edits)
        self.tile_img: Optional[torch.Tensor] = None
        if timg is None:
            self.cap = max(8, (int(math.ceil(int(gather.active_indices.shape[0]) * (1.0 + headroom))) + 7) // 8 * 8)
        else:
            top = int(self._counts().max())
            self.cap = top if headroom <= 0 else (int(math.ceil(top * (1.0 + headroom))) + 7) // 8 * 8
            self.tile_img = (torch.arange(self.E * self.cap, dtype=torch.int32) // max(self.cap, 1)).to(dev)
        self.padded = headroom > 0          # batches: whole CTAs of padding may follow each edit's tiles
        self.buf = torch.full((self.E * self.cap, 2), TILE_NONE, dtype=torch.int32, device=dev)
        self.reload()

    def _counts(self) -> torch.Tensor:
        """Tiles per edit of the gather's current lists (a batch)."""
        g = self.gather
        return torch.bincount(g.tile_images.long().cpu(), minlength=int(g.num_edits))

    def fits(self) -> bool:
        g = self.gather
        timg = getattr(g, "tile_images", None)
        if g.active_indices is None or int(g.active_indices.shape[0]) == 0 or (timg is None) != (self.tile_img is None):
            return False
        if timg is None:
            return int(g.active_indices.shape[0]) <= self.cap
        return int(g.num_edits) == self.E and int(self._counts().max()) <= self.cap

    def reload(self) -> None:
        idx = self.gather.active_indices.to(self.buf.device)
        self.n = int(idx.shape[0])
        if self.tile_img is None:
            self.buf[:self.n] = idx
            self.buf[self.n:] = self.none
            return
        img = self.gather.tile_images.to(self.buf.device).long()           # the concatenated lists are in edit order
        counts = torch.bincount(img, minlength=self.E)
        starts = torch.cumsum(counts, 0) - counts
        rows = img * self.cap + (torch.arange(self.n, device=img.device) - starts[img])
        self.buf.fill_(self.none)
        self.buf[rows] = idx

    def install_device(self, out: torch.Tensor, count: torch.Tensor, status: torch.Tensor) -> None:
        """Install the result of `sige_reduce_mask` (`out` [candidates, 2] of which the first `count` rows are real, `count` a
        DEVICE int32) without the host ever learning the count: the first min(count, cap) origins, SIGE_TILE_NONE behind them;
        `status` (device int32) gets bit 0 set if the list did not fit."""
        cap = self.cap
        src = out[:cap]
        if src.shape[0] < cap:
            src = torch.cat([src, torch.full((cap - src.shape[0], 2), self.none, dtype=torch.int32, device=src.device)], 0)
        rows = torch.arange(cap, device=src.device, dtype=torch.int32).view(cap, 1)
        self.buf.copy_(torch.where(rows < count.view(1, 1), src, torch.full_like(src, self.none)))
        status.bitwise_or_((count > cap).to(torch.int32))
        self.n = cap           # the real count is only known on the device: host-side code treats every entry as potentially real

    def install_batched_device(self, masks: torch.Tensor, status: torch.Tensor) -> None:
        """Reduce the [E, H, W] CUDA masks of a batch straight into `buf` (one `sige_reduce_mask_batched` launch): each edit's
        first min(count, cap) origins, SIGE_TILE_NONE behind them; bit 0 of `status` (device int32) if an edit's list did not fit."""
        from . import ops

        g = self.gather
        ops.reduce_mask_batched_cuda(masks, g.block_size, g.block_stride, g.offset, self.cap, out=self.buf, status=status)
        self.n = self.E * self.cap


def _shortcut_flags(ms: IdxSlot, off: int, ss: IdxSlot, soff: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """The fused 1x1 shortcut's flags of a main conv's list `ms` (origin offset `off`) against the shortcut's list `ss`: uint8,
    one per row of ms.buf, 1 where the row is a real tile whose centre 4x4 tile is in the shortcut's list of the same edit; and
    an int32 [1] that is 1 when some shortcut tile is no such centre (it left the main conv's grid).  Device tensor arithmetic
    only, sorted per edit — no host synchronisation (torch.isin would synchronise)."""
    E, width = ms.E, 1 << 16
    mi, si = ms.buf.view(E, ms.cap, 2).long(), ss.buf.view(E, ss.cap, 2).long()
    real_m, real_s = mi[..., 0] > ms.none, si[..., 0] > ss.none
    main_key = torch.where(real_m, (mi[..., 0] + off) * width + (mi[..., 1] + off), torch.full_like(mi[..., 0], -1))
    sc_key = torch.where(real_s, (si[..., 0] + soff) * width + (si[..., 1] + soff), torch.full_like(si[..., 0], -2))

    def member(keys, pool):          # [E, n] keys found in the same edit's row of pool [E, m]
        if pool.shape[1] == 0:
            return torch.zeros_like(keys, dtype=torch.bool)
        srt = torch.sort(pool, dim=1).values
        return srt.gather(1, torch.searchsorted(srt, keys).clamp(max=srt.shape[1] - 1)) == keys

    flags = (member(main_key, sc_key) & real_m).to(torch.uint8).view(-1)
    stray = (~member(sc_key, main_key) & real_s).any().to(torch.int32).view(1)
    return flags, stray


class ConvInRec:
    """conv_in launch record (<=4-channel stem) with up to two transformed extra outputs."""

    def __init__(self, x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], out: Buf):
        self.x, self.weight, self.bias, self.out = x, weight, bias, out
        self.aux: List = []
        self.tiles: Optional[torch.Tensor] = None   # tile origins when every reader gathers the stem through ONE index set
        self.tile_img: Optional[torch.Tensor] = None
        self.tile_size = 6

    def can_aux(self) -> bool:
        return len(self.aux) < 2

    def add_aux(self, view, scale, shift, act) -> None:
        self.aux.append((view, scale, shift, act))


# =====================================================================================================================
# executors
# =====================================================================================================================
# Packed weights survive re-compilation (new masks, same weights).  Keyed by the IDENTITY of the parameter object (held
# weakly and re-checked) + its version counter — never by address: the caching allocator hands a freed model's addresses to
# the next one.
_PACKED: Dict = {}
_SEPARABLE: Dict = {}


class CudaExecutor:
    """The product path: every launch goes through libsige_b200.so (sige_b200.ops).  No fallback."""

    name = "cuda"

    def __init__(self, device: torch.device, dtype: torch.dtype):
        from . import ops

        self.ops, self.device, self.dtype = ops, device, dtype

    def _pack(self, w: torch.Tensor, key, pad_cin: int = 0) -> torch.Tensor:
        """key: None (do not cache) or (parameter object, tag).  pad_cin > Cin: zero input channels appended before packing (the
        layout of a narrow source's launch)."""
        import weakref

        if key is not None:
            param, tag = key
            k = (id(param), tag, pad_cin, self.dtype)
            hit = _PACKED.get(k)
            if hit is not None and hit[0]() is param and hit[1] == param._version and hit[2].device == param.device:
                return hit[2]
        if pad_cin > w.shape[1]:
            w = F.pad(w, (0, 0, 0, 0, 0, pad_cin - w.shape[1]))
        wp = self.ops.pack_conv_weight(w.contiguous(), self.dtype)
        if key is not None:
            for dead in [kk for kk, vv in _PACKED.items() if vv[0]() is None]:
                del _PACKED[dead]
            _PACKED[k] = (weakref.ref(param), param._version, wp)
        return wp

    def prepare_conv(self, fc: FusedConv) -> None:
        ops = self.ops
        from ._cabi import CONV_EARLY_RELEASE, CONV_PADDED, CONV_PDL, CONV_PER_IMAGE_OPERANDS, CONV_TC5

        s = fc.spec
        w, b = s.weight, s.bias
        key = s.weight_key
        if s.out_row_scale is not None:
            rows, f = s.out_row_scale
            w = w.clone()
            w[:rows] *= f
            if b is not None:
                b = b.clone()
                b[:rows] *= f
            key = None
        wp = self._pack(w, key, pad_cin=(s.Cin + 63) // 64 * 64 if s.Cin % 64 else 0)
        b32 = None if b is None else b.float().contiguous()
        d = ops.tile_conv_descriptor()
        d.dtype = ops._DTYPES[self.dtype]
        d.n_src = len(s.srcs)
        for i, (t, up) in enumerate(s.srcs):
            d.src[i].ptr, d.src[i].C, d.src[i].up = t.data_ptr(), t.shape[1], up
        if not s.src_is_stack and len(s.srcs) == 1 and not s.srcs[0][0].is_contiguous(memory_format=torch.channels_last):
            d.src_pixel_stride = ops.channel_window(s.srcs[0][0])[1]        # a channel window of a wider buffer
        d.B, d.H, d.W = s.B, s.H, s.W
        d.src_is_stack = 1 if s.src_is_stack else 0
        idx_t, sc_flags_t = s.idx, (None if s.shortcut is None else s.shortcut[3])
        d.idx_per_image = 0
        d.N = s.N
        if s.tile_img is not None:           # batch of independent edits: the slot's per-image lists, `cap` rows per edit
            d.idx_per_image, d.N = 1, s.slot.cap
        d.idx = None if idx_t is None else idx_t.data_ptr()
        d.R = d.S = s.block
        d.scale = None if s.scale is None else s.scale.data_ptr()
        d.shift = None if s.shift is None else s.shift.data_ptr()
        d.affine_bstride = s.Cin if s.per_sample_affine else 0
        d.act = ops._act(s.act)
        d.w_packed = wp.data_ptr()
        d.bias = None if b32 is None else b32.data_ptr()
        d.Cin, d.Cout, d.kH, d.kW, d.stride = s.Cin, s.Cout, s.k, s.k, s.stride
        if s.dst_stack is not None:
            d.dst, d.dst_is_stack = s.dst_stack.data_ptr(), 1
            d.dH, d.dW, d.dC, d.dst_c0 = s.dst_stack.shape[2], s.dst_stack.shape[3], s.dst_stack.shape[1], 0
        else:
            need_raw = s.dst.has_raw or not s.aux
            d.dst = s.dst.raw.data_ptr() if need_raw else None
            d.dst_is_stack = 0
            d.dH, d.dW, d.dC, d.dst_c0 = s.dst.shape[2], s.dst.shape[3], s.dst.shape[1], 0
        d.offH = d.offW = s.off
        if s.residual is not None:
            d.residual, d.rC, d.res_c0 = s.residual.data_ptr(), s.residual.shape[1], 0
        else:
            d.residual, d.rC, d.res_c0 = None, 0, 0
        d.ksplit = s.ksplit
        d.flags = (CONV_PDL if s.pdl else 0) | (CONV_TC5 if s.tc5 else 0) | (CONV_EARLY_RELEASE if s.early_release else 0) | (s.early << 4)
        if s.slot is not None and (s.slot.padded if s.tile_img is not None else (s.B == 1 and s.slot.cap - s.slot.n >= 8)):
            d.flags |= CONV_PADDED          # whole CTAs of padding exist (capacity headroom): let them exit at once
        d.n_aux = len(s.aux)
        keep = [wp, b32]
        for i, (view, sc, sh, act) in enumerate(s.aux):
            a = d.aux[i]
            a.ptr, a.C, a.c0 = view.data_ptr(), view.shape[1], 0
            a.scale = None if sc is None else sc.data_ptr()
            a.shift = None if sh is None else sh.data_ptr()
            a.act = ops._act(act)
        if s.epilogue_act == "relu":         # the destination becomes the launch's one aux, with no affine
            assert not s.aux and d.dst
            a = d.aux[0]
            a.ptr, a.C, a.c0, a.scale, a.shift, a.act = d.dst, d.dC, d.dst_c0, None, None, ops._cabi.ACT_RELU
            d.dst, d.n_aux = None, 1
        if s.modulation is not None:       # SPADE's modulation in the gather stage
            gamma, beta, slope = s.modulation
            mod = ops.conv_modulation(gamma, beta, slope)
            d.modulation = ctypes.pointer(mod)
            keep.append(mod)
        if s.tile_img is not None and (s.modulation is not None or d.src_pixel_stride):
            d.flags |= CONV_PER_IMAGE_OPERANDS    # a batch's window / gamma / beta: image b of each at b * H * W * (pixel stride)
        d.n_src2 = 0
        if s.shortcut is not None:
            sc_tensors, sc_w, sc_b, sc_flags = s.shortcut
            w2 = self._pack(sc_w, s.shortcut_key)
            b2 = None if sc_b is None else sc_b.float().contiguous()
            d.n_src2 = len(sc_tensors)
            for i, t in enumerate(sc_tensors):
                d.src2[i].ptr, d.src2[i].C, d.src2[i].up = t.data_ptr(), t.shape[1], 0
            d.Cin2 = int(sc_w.shape[1])
            d.w2_packed = w2.data_ptr()
            d.bias2 = None if b2 is None else b2.data_ptr()
            d.sc_flags = None if sc_flags_t is None else sc_flags_t.data_ptr()
            keep += [w2, b2]
        keep += [idx_t, sc_flags_t]
        fc.desc, fc.keep = d, keep
        fc.launch_fn = lambda stream, d=d: ops.launch_tile_conv(d, stream)

    def takes_wgmma(self, fc: FusedConv) -> bool:
        """Whether the prepared launch runs on the wgmma kernel (sige_tile_conv_plan)."""
        pl = self.ops._cabi.TileConvPlan()
        self.ops._cabi.check(self.ops._cabi.lib().sige_tile_conv_plan(ctypes.byref(fc.desc), ctypes.byref(pl)), "sige_tile_conv_plan")
        return pl.path == 1

    def prepare_conv_in(self, rec: ConvInRec) -> Callable[[int], None]:
        ops = self.ops
        w = rec.weight.detach().to(self.dtype).contiguous()
        b = None if rec.bias is None else rec.bias.detach().to(self.dtype).contiguous()
        aux = [ops.conv_aux(v, sc, sh, act) for (v, sc, sh, act) in rec.aux]
        out = rec.out.raw
        tiles, per_image = rec.tiles, rec.tiles is not None and rec.tile_img is not None      # (a batch: a slot's per-image lists)

        def run(_stream):
            ops.conv_in_nhwc(rec.x, w, b, out=out, aux=aux, tiles=tiles, tile_size=rec.tile_size, tiles_per_image=per_image)

        return run

    def prepare_tail(self, x: torch.Tensor, groups: int, eps: float, gamma, beta, act: str, weight, bias, out: torch.Tensor):
        ops = self.ops
        dt = self.dtype
        B, C = x.shape[0], x.shape[1]
        g = None if gamma is None else gamma.detach().to(dt).contiguous()
        bt = None if beta is None else beta.detach().to(dt).contiguous()
        w = weight.detach().to(dt).contiguous()
        b = None if bias is None else bias.detach().to(dt).contiguous()
        scale = torch.empty((B, C), dtype=torch.float32, device=x.device)
        shift = torch.empty((B, C), dtype=torch.float32, device=x.device)
        ws = torch.empty((ops.group_norm_fold_workspace(B, C),), dtype=torch.float32, device=x.device)

        def run(_stream):
            ops.group_norm_fold(x, groups, eps, g, bt, scale=scale, shift=shift, workspace=ws)
            ops.conv_out_nhwc(x, scale, shift, act, w, b, out=out)

        return run

    def attention_supported(self, n_tokens: int, channels: int) -> bool:
        return self.ops.attention_tokens_supported(n_tokens, channels, self.dtype)

    def tail_supported(self, channels: int, cout: int) -> bool:
        """sige_conv_out_nhwc stages a 10 x 34 pixel halo tile and the weights of all channels in shared memory (<= 227 KB)."""
        pitch = channels * 2 + 16
        smem = ((10 * 34 * pitch + 15) & ~15) + 8 * (9 * channels * 2 + 16)      # (CO_TH + 2) x (CO_TW + 2) = 10 x 34 pixels
        return cout <= 8 and channels % 16 == 0 and channels <= 1024 and smem <= 227 * 1024

    def prepare_attention(self, qkv_tokens: torch.Tensor, out_tokens: torch.Tensor, pdl: bool):
        ops = self.ops
        from ._cabi import CONV_PDL

        flags = CONV_PDL if pdl else 0

        def run(_stream):
            ops.attention_tokens(qkv_tokens, out=out_tokens, flags=flags)

        return run

    def spade_supported(self, x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor) -> bool:
        return self.ops.spade_modulate_supported(x, gamma, beta)

    def prepare_spade(self, x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, slope: float, out: torch.Tensor):
        """out = leaky_relu(x * (1 + gamma) + beta, slope) as ONE launch (sige_spade_modulate); slope = 1: no activation."""
        ops = self.ops

        def run(_stream):
            ops.spade_modulate(x, gamma, beta, slope, out=out)

        return run

    def separable_supported(self, cin: int, cout: int) -> bool:
        return self.ops.separable_conv_supported(cin, cout, self.dtype)

    def writeback_supported(self) -> bool:
        """Can the step copy its output tiles into the module caches (sige_tile_writeback: sparse_update on the fused path)?"""
        return True

    def batch_slots_supported(self) -> bool:
        """Can the launches of a batch of edits read its per-edit fixed-capacity lists (`IdxSlot` of a batch: each edit's rows end
        in SIGE_TILE_NONE padding)?  Then a new batch is installed in place (`FusedStep.rebind`); without it a batch's launches get
        the concatenated lists with a per-row image index, and a new batch recompiles."""
        return True

    def per_image_operands_supported(self) -> bool:
        """Can the modulated, windowed and separable launches of a batch of edits read per-edit lists over operands of E images
        (SIGE_CONV_PER_IMAGE_OPERANDS)?  Then the GauGAN generators' SPADE layers lower for a batch as for one edit."""
        return True

    def per_image_stacks_supported(self) -> bool:
        """Can a tile conv of a batch of edits read per-edit lists with a tile stack on one side (sige_tile_conv_t.idx_per_image:
        stack row b*N + i is list row b*N + i)?  Then SIGEAttnBlock's q conv and proj_out, and the sparse attention between
        them, lower for a batch as for one edit."""
        return True

    def prepare_writeback(self, entries) -> Callable[[int], None]:
        """One `sige_tile_writeback` over (src buffer, module cache, tile list, off, stride, output tile) entries."""
        return self.ops.tile_writeback_launcher(entries)

    def cache_load_supported(self, cache: Optional[torch.Tensor] = None) -> bool:
        """Can `sige_cache_load` fill a cached buffer from this module cache (a dense 4-D f32 / f16 / bf16 CUDA tensor, C a
        multiple of 8)?  Without an argument: does the executor have the launch at all?"""
        return cache is None or (cache.is_cuda and cache.dim() == 4 and int(cache.shape[1]) % 8 == 0 and cache.dtype in self.ops._DTYPES
                                 and self.ops.layout_of(cache) >= 0)

    def prepare_cache_load(self, entries) -> Callable[[int], None]:
        """One `sige_cache_load` over (module cache, raw buffer or None, [(view, scale, shift, act)]) entries."""
        return self.ops.cache_load_launcher(entries, self.dtype)

    def repack_conv(self, fc: FusedConv) -> None:
        """Enqueue the packing of a prepared launch's `spec.weight` / `spec.bias`, recomputed in place (`FusedStep.refresh`),
        into the packed buffers its descriptor points at."""
        s = fc.spec
        w, b = s.weight, s.bias
        if s.out_row_scale is not None:
            rows, f = s.out_row_scale
            w = w.clone()
            w[:rows] *= f
            if b is not None:
                b = b.clone()
                b[:rows] *= f
        pad_cin = (s.Cin + 63) // 64 * 64 if s.Cin % 64 else 0
        if pad_cin > w.shape[1]:
            w = F.pad(w, (0, 0, 0, 0, 0, pad_cin - w.shape[1]))
        wp, b32 = fc.keep[0], fc.keep[1]
        self.ops.pack_conv_weight(w.contiguous(), self.dtype, out=wp)
        if b32 is not None and b32 is not b:
            b32.copy_(b)

    def narrow_conv_supported(self, cin: int, cout: int, k: int, stride: int) -> bool:
        """Can sige_tile_conv run a conv whose single source has `cin` channels, a multiple of 8 but not of 64 (the mma.sync
        kernel with a partial last K chunk)?"""
        return cin % 64 != 0 and self.ops.tile_conv_supported(cin, cout, k, stride, self.dtype)

    def modulated_conv_supported(self, cin: int, cout: int, k: int, stride: int) -> bool:
        """Can sige_tile_conv run a conv whose source is SPADE's modulation of `cin` channels?"""
        return self.ops.tile_conv_supported(cin, cout, k, stride, self.dtype)

    def strided_conv_supported(self, cin: int, cout: int, k: int, stride: int) -> bool:
        """Can sige_tile_conv run a conv whose source is a `cin`-channel window of a wider buffer?"""
        return self.ops.tile_conv_supported(cin, cout, k, stride, self.dtype)

    def _separable_weights(self, dw: "DWConv", pw_w: torch.Tensor, pw_b: Optional[torch.Tensor]):
        """(depthwise weight, bias with the affine folded in fp32; 1x1 weight in the step's dtype; fp32 1x1 bias), cached by the
        identity (and version) of the parameters and of the tensors the affine was recorded with."""
        import weakref

        objs = tuple(o for o in (dw.weight, dw.bias, pw_w, pw_b) + tuple(c._base if c._base is not None else c for c in dw.consts) if o is not None)
        k = (tuple(id(o) for o in objs), self.dtype)
        hit = _SEPARABLE.get(k)
        if hit is not None and all(r() is o for r, o in zip(hit[0], objs)) and hit[1] == tuple(o._version for o in objs) and hit[2][2].device == self.device:
            return hit[2]
        w, b = self.ops.separable_fold(dw.weight.to(self.device), None if dw.bias is None else dw.bias.to(self.device), dw.scale, dw.shift)
        packed = (w, b, pw_w.detach().to(self.device, self.dtype).reshape(pw_w.shape[0], -1).contiguous(),
                  None if pw_b is None else pw_b.detach().to(self.device).float().contiguous())
        for dead in [kk for kk, vv in _SEPARABLE.items() if any(r() is None for r in vv[0])]:
            del _SEPARABLE[dead]
        _SEPARABLE[k] = (tuple(weakref.ref(o) for o in objs), tuple(o._version for o in objs), packed)
        return packed

    def prepare_separable(self, rec: "SepLaunch") -> Callable[[int], None]:
        """One sige_separable_conv launch of a SepLaunch record (gamma and beta of one SPADE layer)."""
        from ._cabi import CONV_PDL, CONV_PER_IMAGE_OPERANDS

        branches = [self._separable_weights(dw, pw_w, pw_b) + (dst.raw,) for (dw, pw_w, pw_b, dst) in rec.branches]
        src = rec.src[:, rec.c0:rec.c0 + rec.Cin]
        ops, idx, off, stack, batch, flags = self.ops, rec.idx, rec.off, rec.src_stack, rec.batch, (CONV_PDL if rec.pdl else 0)
        if rec.tile_img is not None:
            flags |= CONV_PER_IMAGE_OPERANDS      # a batch of edits: the slot's per-edit lists

        def run(_stream):
            ops.separable_conv(src, branches, idx, src_stack=stack, offset=off, batch=batch, flags=flags)

        return run

    def sparse_attention_supported(self, head_dim: int) -> bool:
        return self.ops.sparse_attention_supported(head_dim, self.dtype)

    def prepare_sparse_attention(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float, out: torch.Tensor):
        """softmax(scale * q k^T) v of [(b h), n, d] operands as ONE launch of this repo's kernel (sige_sparse_attention)."""
        ops = self.ops

        def run(_stream):
            ops.sparse_attention(q, k, v, scale, out=out)

        return run

    def gather(self, x, block, idx, scale, shift, act, act_first, up=0):
        return self.ops.gather(x, block[0], block[1], idx, scale, shift, act, act_first, up=up)

    def launch_counter(self) -> int:
        return self.ops.launch_count


# =====================================================================================================================
# symbolic values of the lowering
# =====================================================================================================================
class Pre:
    """Pending per-channel pointwise op act(x*scale+shift); scale/shift are fp32 [C] or [B, C] tensors or None.  `mod` = ((gamma Buf,
    first channel), (beta Buf, first channel), slope): SPADE's modulation leaky((x*scale+shift) * (1 + gamma) + beta) after it (a
    ModStack's gather stage)."""

    def __init__(self, scale=None, shift=None, act: Optional[str] = None, mod=None):
        self.scale, self.shift, self.act, self.mod = scale, shift, act, mod

    def copy(self) -> "Pre":
        return Pre(self.scale, self.shift, self.act)


class Full:
    """A (B, C, H, W) activation: channel concat of (Buf, upsample flag) segments + pending pointwise op + pending pad."""

    def __init__(self, segs: List[Tuple[Buf, int]], pre: Optional[Pre] = None, pad: Optional[Tuple[int, int, int, int]] = None):
        self.segs, self.pre, self.pad = segs, pre, pad

    @property
    def plain(self) -> bool:
        return self.pre is None and self.pad is None

    @property
    def single(self) -> Optional[Buf]:
        return self.segs[0][0] if (self.plain and len(self.segs) == 1 and self.segs[0][1] == 0) else None

    @property
    def C(self) -> int:
        return sum(b.shape[1] for b, _ in self.segs)

    @property
    def B(self) -> int:
        return self.segs[0][0].shape[0]

    @property
    def HW(self) -> Tuple[int, int]:
        b, up = self.segs[0]
        return (b.shape[2] << up, b.shape[3] << up)


class Stack:
    """Lazy Gather: halo tiles of `src` (a plain Full) cut by `gather` with the fused pre-op."""

    def __init__(self, src: Full, gather, scale, shift):
        self.src, self.gather, self.scale, self.shift = src, gather, scale, shift


class ModStack(Stack):
    """SPADE's modulation of three lazy Stacks cut with one tile list: the tiles of `src` (with the Gather's scale / shift) times
    (1 + the same tiles of `gamma`) plus those of `beta`, then leaky_relu(slope).  gamma / beta are channels [c0, c0 + C) of their
    buffers (C = the source's channels; c0 > 0: a torch.split window).  Only ever the source of a ConvOut: the conv's launch applies
    it in its gather stage (sige_tile_conv_t.modulation), so none of the stacks is materialised."""

    def __init__(self, x: Stack, gamma: "Buf", beta: "Buf", slope: float, gamma_c0: int = 0, beta_c0: int = 0):
        super().__init__(x.src, x.gather, x.scale, x.shift)
        self.gamma, self.beta, self.slope = gamma, beta, slope
        self.gamma_c0, self.beta_c0 = gamma_c0, beta_c0


class WinStack(Stack):
    """The tiles of channels [c0, c0 + C) of a plain lazy Stack of one buffer (a torch.split part of it: SPADE's actv_0 / actv_1 /
    actv_s).  Only ever the source of a ConvOut: the launch reads the window in place (sige_tile_conv_t.src_pixel_stride)."""

    def __init__(self, st: Stack, c0: int, C: int):
        super().__init__(st.src, st.gather, st.scale, st.shift)
        self.c0, self.C = c0, C


class RealStack:
    """A materialised tile stack (B*N, C, R, S) produced by an eager node, or one row per entry of a fixed-capacity tile list
    (`slot`: the sparse-attention core's output) — scattered through that list."""

    def __init__(self, tensor: torch.Tensor, slot: Optional["IdxSlot"] = None):
        self.tensor, self.slot = tensor, slot


class ConvOut:
    """A conv whose launch has not been emitted yet (its consumer decides destination / residual / shortcut)."""

    def __init__(self, node: Node, src, weight, bias, k: int, stride: int, padding: int, cin_pad: int = 0, act: Optional[str] = None):
        self.node, self.src, self.weight, self.bias, self.k, self.stride, self.padding = node, src, weight, bias, k, stride, padding
        self.cin_pad = cin_pad          # zero input channels appended to the weight (the source is a zero-padded label map)
        self.act = act                  # "relu": epilogue activation of the launch

    @property
    def on_tiles(self) -> bool:
        return isinstance(self.src, (Stack, RealStack))


class RealT:
    """A real tensor at a stable address (static inputs, outputs of eager nodes)."""

    def __init__(self, tensor: torch.Tensor):
        self.tensor = tensor


class Sig:
    def __init__(self, of: LazyTensor):
        self.of = of


class GNVal:
    def __init__(self, src: Buf, groups: int, weight, bias, eps: float, act: Optional[str] = None):
        self.src, self.groups, self.weight, self.bias, self.eps, self.act = src, groups, weight, bias, eps, act


class ChanSlice:
    def __init__(self, buf: Buf, c0: int, c1: int):
        self.buf, self.c0, self.c1 = buf, c0, c1


class Tok:
    def __init__(self, sl: ChanSlice, layout: str):
        self.sl, self.layout = sl, layout            # 'bcn' or 'bnc'


class Scores:
    def __init__(self, q: ChanSlice, k: ChanSlice, scale: float = 1.0):
        self.q, self.k, self.scale = q, k, scale


class Probs:
    def __init__(self, s: Scores, transposed: bool = False):
        self.s, self.transposed = s, transposed


class AttnOut:
    def __init__(self, s: Scores, v: ChanSlice):
        self.s, self.v = s, v


class GScores:
    """q @ k^T (* scale) of generic (batch*heads, tokens, dim) operands — the attention core of the SD transformer blocks
    (reference stable-diffusion/ldm/modules/sige_attention.py:46-60, attention.py CrossAttention)."""

    def __init__(self, q: LazyTensor, k: LazyTensor, scale: float = 1.0, probs: bool = False):
        self.q, self.k, self.scale, self.probs = q, k, scale, probs


class HeadsOut:
    """Result of the sparse-attention kernel, written straight into the "b n (h d)" tensor `full` that the next Linear reads.
    `stage` follows einops' rearrange "(b h) n d -> b n (h d)" (attention.py:93): 0 = the [(b h), n, d] value, 1 = after
    reshape to [b, h, n, d], 2 = after permute to [b, n, h, d]; the closing reshape to [b, n, h*d] IS `full` — no copy."""

    def __init__(self, full: torch.Tensor, b: int, h: int, n: int, d: int, stage: int = 0):
        self.full, self.b, self.h, self.n, self.d, self.stage = full, b, h, n, d, stage

    @property
    def bhnd(self) -> torch.Tensor:
        return self.full.view(self.b, self.n, self.h, self.d).permute(0, 2, 1, 3)


class Spade:
    """SPADE's modulation recognised on the tape (reference gaugan/models/sige_normalization.py:84-86 + the block's leaky_relu):
    stage 1 = `1 + gamma`, 2 = `x * (1 + gamma)`, 3 = `x * (1 + gamma) + beta` (optionally followed by leaky_relu: `slope`).
    Speculative: a consumer that wants an intermediate value simply gets the recorded call evaluated; only stage 3 materialises
    as ONE `sige_spade_modulate` launch."""

    def __init__(self, stage: int, gamma: LazyTensor, x: Optional[LazyTensor] = None, beta: Optional[LazyTensor] = None, slope: Optional[float] = None):
        self.stage, self.gamma, self.x, self.beta, self.slope = stage, gamma, x, beta, slope


class DWConv:
    """Depthwise 3x3 SIGEConv2d (groups = Cin = Cout) on 6x6 halo tiles, with the per-channel affine that follows it in GAN
    Compression's separable conv (the dense pass's instance norm, reference gaugan/models/mobile_modules.py:108-111).  Speculative:
    only a 1x1 SIGEConv2d consumes it (as `SepOut`); any other consumer gets the recorded calls evaluated.
    `src` is a RealStack (NHWC tile stack) or a plain lazy Stack of a buffer; `c0` the start of its channel window."""

    def __init__(self, src, c0: int, weight, bias, scale=None, shift=None, consts: Tuple = ()):
        self.src, self.c0, self.weight, self.bias, self.scale, self.shift, self.consts = src, c0, weight, bias, scale, shift, consts

    @property
    def C(self) -> int:
        return int(self.weight.shape[0])


class SepOut:
    """1x1 conv of a DWConv: a separable conv whose launch waits for its Scatter / ScatterGather (like ConvOut)."""

    def __init__(self, dw: DWConv, weight, bias):
        self.dw, self.weight, self.bias = dw, weight, bias


class SepLaunch:
    """One `sige_separable_conv` launch: up to two branches (gamma and beta of one SPADE layer) on the same source window and
    tile list.  Branch = (DWConv, 1x1 weight, 1x1 bias, destination Buf)."""

    def __init__(self, name: str, src: torch.Tensor, src_stack: bool, c0: int, idx: torch.Tensor, off: int, batch: int, slot: int):
        self.name, self.src, self.src_stack, self.c0, self.idx, self.off, self.batch = name, src, src_stack, c0, idx, off, batch
        self.slot = slot                      # index of the launch in Lowering.steps
        self.tile_img: Optional[torch.Tensor] = None       # a batch of edits: image of each row of idx (the IdxSlot's per-edit lists)
        self.pdl = False
        self.branches: List[Tuple[DWConv, torch.Tensor, Optional[torch.Tensor], Buf]] = []

    @property
    def Cin(self) -> int:
        return self.branches[0][0].C

    @property
    def Cout(self) -> int:
        return int(self.branches[0][1].shape[0])


_POINTWISE = {"add", "mul", "sub", "div", "rsub", "neg", "leaky_relu", "relu", "silu", "gelu", "sigmoid", "tanh", "clamp", "clamp_min", "abs"}
_MATERIAL = (Full, Stack, RealStack, ConvOut, RealT)
_VIEW_OPS = {"reshape", "view", "permute", "transpose", "chunk", "split", "__getitem__", "unsqueeze", "squeeze", "flatten", "unflatten",
             "expand", "narrow", "select", "unbind", "t", "movedim", "swapaxes", "view_as", "reshape_as", "T.__get__", "mT.__get__"}


def _channels(t: torch.Tensor, c0: int, C: int) -> torch.Tensor:
    """Channels [c0, c0 + C) of a (B, C', H, W) buffer: the buffer itself when that is all of it, else the channel-slice view."""
    return t if (c0 == 0 and int(t.shape[1]) == C) else t[:, c0:c0 + C]


def _bits(t: torch.Tensor) -> torch.Tensor:
    """Bit pattern of a tensor (NaN-safe equality)."""
    if t.dtype in (torch.float16, torch.bfloat16):
        return t.contiguous().view(torch.int16)
    if t.dtype == torch.float32:
        return t.contiguous().view(torch.int32)
    return t


def _out_variant(name: str, op):
    """out= form of a recorded torch call: f(args, kwargs, dst) writes the call's result into dst, or None if there is none.
    Only calls whose out= overload computes exactly what the recorded call computes under autocast on 16-bit operands."""
    if name in ("add", "mul") and op in (torch.add, torch.mul, torch.Tensor.add, torch.Tensor.mul, torch.Tensor.__add__, torch.Tensor.__mul__,
                                         torch.Tensor.__radd__, torch.Tensor.__rmul__):
        fn = torch.add if name == "add" else torch.mul
        return lambda args, kwargs, dst: fn(*args, **kwargs, out=dst)
    if name == "linear" and op is F.linear:
        def linear(args, kwargs, dst):
            kw = dict(zip(("input", "weight", "bias"), args))
            kw.update(kwargs)
            x, w, b = kw["input"], kw["weight"], kw.get("bias")
            if not (x.dtype == w.dtype == dst.dtype and x.dtype in (torch.float16, torch.bfloat16) and (b is None or b.dtype == x.dtype)
                    and x.is_contiguous() and dst.is_contiguous()):
                raise TypeError("linear: not the plain 16-bit case")
            x2, d2 = x.view(-1, x.shape[-1]), dst.view(-1, dst.shape[-1])
            if b is None:
                torch.mm(x2, w.t(), out=d2)
            else:
                torch.addmm(b, x2, w.t(), out=d2)
        return linear
    if name == "gelu" and op is F.gelu:
        return lambda args, kwargs, dst: torch._C._nn.gelu(*args, **kwargs, out=dst)
    if name == "silu" and op is F.silu:
        return lambda args, kwargs, dst: torch._C._nn.silu(args[0], out=dst) if not kwargs.get("inplace", False) and len(args) == 1 else (_ for _ in ()).throw(TypeError())
    if name == "leaky_relu" and op is F.leaky_relu:
        def leaky(args, kwargs, dst):
            kw = dict(zip(("input", "negative_slope", "inplace"), args))
            kw.update(kwargs)
            if kw.get("inplace", False):
                raise TypeError("in-place")
            torch._C._nn.leaky_relu(kw["input"], kw.get("negative_slope", 0.01), out=dst)
        return leaky
    return None


def _is_const(o) -> bool:
    return isinstance(o, torch.Tensor) and not isinstance(o, LazyTensor)


def _fold_affine(weight: torch.Tensor, bias: Optional[torch.Tensor], f_scale: Optional[torch.Tensor], f_shift: Optional[torch.Tensor],
                 cin_pad: int) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """fp32 (weight, bias) of a 1x1 conv with the per-input-channel affine x * f_scale + f_shift folded in (exact: no halo),
    `cin_pad` zero input channels appended."""
    w32 = weight.detach().float()
    b32 = None if bias is None else bias.detach().float()
    if f_shift is not None:
        b32 = (torch.zeros(w32.shape[0], device=w32.device) if b32 is None else b32) + (w32[:, :, 0, 0] @ f_shift.to(w32.device))
    if f_scale is not None:
        w32 = w32 * f_scale.to(w32.device).view(1, -1, 1, 1)
    if cin_pad:
        w32 = F.pad(w32, (0, 0, 0, 0, 0, cin_pad))
    return w32, b32


def _pair(v) -> Tuple[int, int]:
    if isinstance(v, (tuple, list)):
        return (int(v[0]), int(v[-1]))
    return (int(v), int(v))


# =====================================================================================================================
# lowering
# =====================================================================================================================
class Lowering:
    def __init__(self, tape: lazy.Tape, outputs, static_inputs: Sequence[torch.Tensor], executor, dtype: torch.dtype, device,
                 pdl: bool = True, tc5: bool = True, producer_preop: bool = True, fuse_shortcut: bool = True,
                 fused_attention: bool = True, sparse_stem: bool = True, ksplit: int = 0, module_names: Optional[Dict[int, str]] = None,
                 headroom: float = 0.0):
        """headroom: extra capacity of the tile-list buffers (0.25 = a later mask may have 25 % more tiles per list and still be
        installed in place by `FusedStep.rebind`; CTAs made only of padding exit at once)."""
        self.tape, self.ex, self.dtype, self.dev = tape, executor, dtype, device
        self.headroom = float(headroom)
        ok = getattr(executor, "batch_slots_supported", None)
        self.batch_slots = ok is not None and ok()
        ok = getattr(executor, "per_image_operands_supported", None)
        self.per_image_ops = self.batch_slots and ok is not None and ok()
        ok = getattr(executor, "per_image_stacks_supported", None)
        self.per_image_stacks = self.batch_slots and ok is not None and ok()
        self.module_names = module_names or {}
        self.pdl, self.tc5, self.producer_preop, self.fuse_shortcut = pdl, tc5, producer_preop, fuse_shortcut
        self.fused_attention, self.sparse_stem, self.ksplit = fused_attention, sparse_stem, ksplit
        self.sparse_attention_calls = 0
        self._consumers: Optional[Dict[int, Node]] = None       # LazyTensor id -> first node that reads it (_sole_consumer)
        self.spade_calls = 0
        self.separable: List[SepLaunch] = []
        self._nhwc_stacks: Dict[int, torch.Tensor] = {}
        self._padded_maps: Dict[int, Full] = {}
        self.steps: List[Tuple[str, Callable[[int], None]]] = []
        self.fused: List[FusedConv] = []
        self.conv_ins: List[ConvInRec] = []
        self.eager_nodes: List[str] = []
        self.slots: Dict[int, IdxSlot] = {}
        self.flag_recipes: List = []       # (flags buffer, main slot, off, shortcut slot, soff) of fused shortcuts
        self.cached_bufs: List[Buf] = []
        # sparse_update: (cached Buf, IdxSlot or None, off, stride, output tile) of every launch that writes a cached buffer, and
        # (name, shortcut source Bufs, weight, bias, skip Buf, IdxSlot, off, conv2's launch) of every shortcut fused into conv2
        self.cache_writers: List[Tuple[Buf, Optional[IdxSlot], int, int, int]] = []
        self.shortcut_relaunches: List = []
        self.epilogue: List[Tuple[str, Callable[[int], None]]] = []
        self.epilogue_fused: List[FusedConv] = []
        self.sparse_update_reason: Optional[str] = "not lowered yet"
        self.view_nodes = 0              # view ops resolved at build time (no run-time work)
        self._all_idx: Dict = {}
        self._vecs: Dict = {}
        self._pending_prepare: List[Callable[[], None]] = []
        self.env: Dict[int, Any] = {}
        self._alias_of: Dict[int, LazyTensor] = {}
        self.uses: Dict[int, int] = {}
        self._keepalive: List = []
        self.derived: List[Derived] = []       # every tensor taken from outside the tape, and what the program made of it
        self.eager_state: List[str] = []       # eager operator-module calls that read module caches themselves
        self.cache_load = getattr(executor, "cache_load_supported", None)
        self.loader = None                     # (prepared sige_cache_load, buffers it does not take) of load_caches
        self.built = False
        for lt, t in zip(tape.inputs, static_inputs):
            self.env[id(lt)] = RealT(t)
        self._count_uses(outputs)
        for node in tape.nodes:
            self._lower(node)
        self.outputs = lazy._tree_map(lambda o: self._output(o) if isinstance(o, LazyTensor) else o, outputs)
        self._post()
        self.built = True
        if self.cache_load is not None:
            self.load_caches(torch.cuda.current_stream(self.dev).cuda_stream if self.dev.type == "cuda" else 0)

    # ------------------------------------------------------------------ helpers: memory
    def empty(self, b: int, c: int, h: int, w: int) -> torch.Tensor:
        return torch.empty((b, c, h, w), dtype=self.dtype, device=self.dev, memory_format=torch.channels_last)

    def clone_cache(self, cache: torch.Tensor, batch: int) -> torch.Tensor:
        c = cache.detach().to(self.dtype)
        if batch != c.shape[0]:            # a batch of edits of ONE original image: every edit starts from the same cached activation
            c = c.expand(batch, *c.shape[1:])
        return c.clone(memory_format=torch.channels_last)

    def fresh(self, b: int, c: int, h: int, w: int) -> Buf:
        """A buffer that is completely rewritten every step (dense layers)."""
        return Buf(self, (b, c, h, w))

    def cached(self, cache: torch.Tensor, batch: Optional[int] = None) -> Buf:
        """A buffer initialised from a module cache; only active tiles are rewritten per step.  The program owns a
        copy (the module's cache stays pristine).  `batch`: number of independent edits sharing the cache."""
        shape = tuple(cache.shape) if batch is None else (batch, *cache.shape[1:])
        b = Buf(self, shape, cached_init=cache.detach())
        self.cached_bufs.append(b)
        return b

    def loads(self, buf: Buf) -> bool:
        """Does the executor's one-launch cache load (`sige_cache_load`) fill this cached buffer?"""
        return self.cache_load is not None and self.cache_load(buf.cached_init)

    def prepared_loader(self):
        """(the prepared `sige_cache_load` or None, the cached buffers it does not take), prepared once per set of caches."""
        if self.loader is None:
            entries, rest = [], []
            for b in self.cached_bufs:
                if not self.loads(b):
                    rest.append(b)
                elif b.has_raw or b.view_inits:
                    entries.append((b.cached_init, b._raw, [(v, sc, sh, act) for (v, sc, sh, act) in b.view_inits]))
            self.loader = (self.ex.prepare_cache_load(entries) if entries else None, rest)
        return self.loader

    def load_caches(self, stream: int) -> None:
        """Every cached buffer (raw copy and transformed views) from its cache, as the step starts a new edit: one
        `sige_cache_load` for the caches the executor takes, the torch chain (`Buf.restore`) for the others."""
        run, rest = self.prepared_loader()
        if run is not None:
            run(stream)
        for b in rest:
            b.restore()

    def derive(self, fn: Optional[Callable], *srcs):
        """``fn(*srcs)`` for a tensor the program reads that is made from tensors taken from outside the tape; ``fn`` None:
        ``srcs`` are read as they are (nothing is returned).  Recorded (`Derived`) so that `FusedStep.refresh` can recompute it
        into the same storage after a dense pass.  A result that aliases a source is copied: the program owns its storage."""
        out = fn(*srcs) if fn is not None else None
        ptrs = {t.untyped_storage().data_ptr() for t in srcs if isinstance(t, torch.Tensor)}

        def own(t):
            return t.clone() if isinstance(t, torch.Tensor) and t.untyped_storage().data_ptr() in ptrs else t

        out = tuple(own(t) for t in out) if isinstance(out, tuple) else own(out)
        self.derived.append(Derived(fn, srcs, out))
        return out

    def vec(self, v: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
        """fp32 contiguous copy of a per-channel vector (kept alive; one copy per distinct source)."""
        if v is None:
            return None
        key = (v.data_ptr(), v.numel(), v._version, tuple(v.shape), tuple(v.stride()))
        if key not in self._vecs:
            dev = self.dev
            self._vecs[key] = (self.derive(lambda t: t.detach().to(dev).reshape(-1).float().contiguous(), v), v)
        return self._vecs[key][0]

    def all_tiles(self, h: int, w: int, off: int) -> torch.Tensor:
        """Index list covering the whole image with stride-4 tiles (dense layers as 'everything active')."""
        key = (h, w, off)
        if key not in self._all_idx:
            ii, jj = torch.meshgrid(torch.arange(0, h, 4), torch.arange(0, w, 4), indexing="ij")
            idx = torch.stack([ii.reshape(-1), jj.reshape(-1)], 1) - off
            self._all_idx[key] = idx.to(torch.int32).to(self.dev).contiguous()
        return self._all_idx[key]

    # ------------------------------------------------------------------ use counts
    def _count_uses(self, outputs) -> None:
        def bump(o):
            if isinstance(o, LazyTensor):
                self.uses[id(o)] = self.uses.get(id(o), 0) + 1
            return o

        for node in self.tape.nodes:
            lazy._tree_map(bump, node.args)
            lazy._tree_map(bump, node.kwargs)
        lazy._tree_map(bump, outputs)

    def n_uses(self, lt: LazyTensor) -> int:
        return self.uses.get(id(lt), 0)

    # ------------------------------------------------------------------ views (producer-side pre-op)
    def view(self, buf: Buf, scale: Optional[torch.Tensor], shift: Optional[torch.Tensor], act: str) -> Optional[torch.Tensor]:
        """Tensor holding act(buf*scale+shift), kept up to date by buf's producer(s); None if not possible.
        scale / shift: fp32 [C] vectors (slices allowed)."""
        if not self.producer_preop or not buf.producers:
            return None
        key = (None if scale is None else (scale.data_ptr(), scale.numel()), None if shift is None else (shift.data_ptr(), shift.numel()), act)
        if key in buf.views:
            return buf.views[key][0]
        if not all(pr.can_aux() for pr in buf.producers):
            return None
        b, c, h, w = buf.shape
        sc = None if scale is None else scale.contiguous()
        sh = None if shift is None else shift.contiguous()
        v = self.empty(b, c, h, w)
        if buf.cached_init is not None:
            if self.built or not self.loads(buf):
                self.init_view(v, buf.cached_init, sc, sh, act)
            buf.view_inits.append((v, sc, sh, act))
            self.loader = None
        else:
            v.zero_()
        for pr in buf.producers:
            pr.add_aux(v, sc, sh, act)
        buf.views[key] = (v, sc, sh)
        return v

    def init_view(self, v: torch.Tensor, cached: torch.Tensor, sc, sh, act: str) -> None:
        z = cached.to(self.dev).float()
        if sc is not None:
            z = z * sc.view(1, -1, 1, 1)
        if sh is not None:
            z = z + sh.view(1, -1, 1, 1)
        if act == "swish":
            z = z * torch.sigmoid(z)
        v.copy_(z)

    def slot(self, g) -> "IdxSlot":
        """The fixed-capacity index buffer of Gather `g`'s tile list (one per distinct list)."""
        key = id(g.active_indices)
        if key not in self.slots:
            self.slots[key] = IdxSlot(getattr(g, "real", g), self.dev, self.headroom)       # (a ScatterGather's geometry stub points at the real Gather)
        return self.slots[key]

    # ------------------------------------------------------------------ emission of one fused launch
    def emit_conv(self, name: str, segs: Sequence[Tuple[Buf, int]], pre: Optional[Pre], hw: Tuple[int, int], idx: torch.Tensor, block: int,
                  weight: torch.Tensor, bias: Optional[torch.Tensor], stride: int, off: int, dst: Optional[Buf], residual: Optional[Buf] = None,
                  shortcut=None, stack_src: Optional[torch.Tensor] = None, dst_stack: Optional[torch.Tensor] = None,
                  weight_fold: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, tile_img: Optional[torch.Tensor] = None,
                  cin_pad: int = 0, epilogue: Optional[str] = None, window: Optional[Tuple[int, int]] = None) -> Optional[FusedConv]:
        """Each source is (buffer, upsample flag); `pre` spans the concatenated channels.  An affine source is read from the
        pre-transformed view its producer maintains, else the gather stage applies the pre-op.  `cin_pad` zero input channels
        are appended to the weight; `epilogue` = "relu" writes relu(out) to the destination.  `window` = (c0, c1): the launch
        reads channels [c0, c1) of its single plain source (the spec holds that channel slice of the buffer)."""
        if stack_src is not None:            # rows are b*N + i (reference sige/cuda/gather_kernel.cu:30)
            B = dst.shape[0] if (dst is not None and idx is not None) else 1
            n = int(stack_src.shape[0]) // (B if tile_img is None else 1)     # (per-image lists: one list row per stack row)
            assert idx is None or int(idx.shape[0]) == n, name
        else:
            B, n = segs[0][0].shape[0], int(idx.shape[0])
        s = ConvSpec()
        s.name = name
        key = (weight, "w")
        if weight_fold is not None:        # exact fold of a per-input-channel affine (no activation) into a 1x1 conv
            assert weight.shape[2] == 1 and weight.shape[3] == 1
            w32, b32 = self.derive(_fold_affine, weight, bias, weight_fold[0], weight_fold[1], cin_pad)
            key = None                      # folded with per-image statistics: never cached
            s.refold = True
            self._keepalive.append(weight_fold)
        else:
            self.derive(None, weight, bias)
            w32 = weight.detach().float()
            b32 = None if bias is None else bias.detach().float()
            if cin_pad:
                w32 = F.pad(w32, (0, 0, 0, 0, 0, cin_pad))
        s.weight, s.bias, s.weight_key = w32, b32, key
        s.epilogue_act = epilogue or "identity"
        s.k, s.stride, s.off, s.block = int(weight.shape[2]), stride, off, block
        s.B, s.H, s.W = B, hw[0], hw[1]
        s.idx, s.N, s.tile_img = idx, n, tile_img
        s.slot = next((sl for sl in self.slots.values() if sl.buf is idx), None)
        s.pdl, s.tc5, s.ksplit = self.pdl, self.tc5, self.ksplit
        if stack_src is not None:
            s.src_is_stack = True
            s.srcs = [(stack_src, 0)]
            s.H, s.W = block, block
        else:
            tensors: List[torch.Tensor] = []
            gather_side = False
            if pre is not None and pre.mod is not None:        # modulated gather: raw x, its affine applied before the modulation
                tensors = [b_.raw for (b_, _) in segs]
                s.scale = None if pre.scale is None else pre.scale.contiguous()
                s.shift = None if pre.shift is None else pre.shift.contiguous()
                s.per_sample_affine = self._per_sample(pre)
                (gamma, g0), (beta, b0), slope = pre.mod
                for b_ in (gamma, beta):
                    b_.readers.append((idx, block, 0, tile_img))
                cin = sum(b_.shape[1] for b_, _ in segs)
                s.modulation = (_channels(gamma.raw, g0, cin), _channels(beta.raw, b0, cin), slope)
            elif pre is not None and (pre.scale is not None or pre.shift is not None or pre.act):
                per_sample = (pre.scale is not None and pre.scale.dim() == 2) or (pre.shift is not None and pre.shift.dim() == 2)
                views, c0 = [], 0
                if not per_sample:
                    for (b_, up_) in segs:
                        c = b_.shape[1]
                        sc = None if pre.scale is None else pre.scale[c0:c0 + c]
                        sh = None if pre.shift is None else pre.shift[c0:c0 + c]
                        views.append(self.view(b_, sc, sh, pre.act or "identity"))
                        c0 += c
                if per_sample or any(v is None for v in views):
                    gather_side = True
                    tensors = [b_.raw for (b_, _) in segs]
                    s.scale = None if pre.scale is None else pre.scale.contiguous()
                    s.shift = None if pre.shift is None else pre.shift.contiguous()
                    s.per_sample_affine = per_sample
                    s.act = pre.act or "identity"
                else:
                    tensors = views
            else:
                tensors = [b_.raw for (b_, _) in segs]
                if window is not None:
                    assert len(segs) == 1, name
                    tensors = [_channels(tensors[0], window[0], window[1] - window[0])]
            for (b_, up_) in segs:
                b_.readers.append((idx, block, up_, tile_img))
            s.srcs = [(t, up) for t, (_, up) in zip(tensors, segs)]
            del gather_side
        if residual is not None:
            residual.readers.append((idx, block, 0, tile_img))
            s.residual = residual.raw
        s.dst, s.dst_stack = dst, dst_stack
        if shortcut is not None:
            sc_bufs, sc_w, sc_b, sc_flags = shortcut
            for b_ in sc_bufs:
                b_.readers.append((idx, block, 0, tile_img))      # the fused shortcut reads the centre 4x4 of conv2's 6x6 tiles
            self.derive(None, sc_w, sc_b)
            s.shortcut = ([b_.raw for b_ in sc_bufs], sc_w.detach().float(), None if sc_b is None else sc_b.detach().float(), sc_flags)
            s.shortcut_key = (sc_w, "w")
        fc = FusedConv(s)
        if n == 0:
            return None
        if dst is not None:
            dst.producers.append(fc)
            if dst.cached_init is not None:
                self.cache_writers.append((dst, s.slot if tile_img is None else None, off, stride, (block - s.k) // stride + 1))
        fc.pos = len(self.steps)
        self.fused.append(fc)
        self.steps.append(("conv", fc.launch))
        return fc

    # ------------------------------------------------------------------ forcing / materialising values
    def sym(self, lt) -> Any:
        v = self.env.get(id(lt))
        if v is None and id(lt) in self._alias_of:        # identity op on a value that has no symbolic form (yet)
            return self.sym(self._alias_of[id(lt)])
        return v

    def as_full(self, lt: LazyTensor) -> Optional[Full]:
        """The value as a Full (emitting a pending conv / evaluating an un-lowered producer eagerly and wrapping its
        result); None if it is not a (B, C, H, W) activation."""
        v = self.sym(lt)
        if isinstance(v, Full):
            return v
        if isinstance(v, ConvOut) and not v.on_tiles:
            buf = self.force_dense(v)
            f = Full([(buf, 0)])
            self.env[id(lt)] = f
            return f
        if isinstance(v, (Stack, RealStack, ConvOut)) or lt.dim() != 4 or lt.shape[1] % 8 != 0:
            return None
        if not isinstance(v, RealT):
            if lt.node is None:
                return None
            t = self.runtime_tensor(lt)    # an island the lowering does not know: its result feeds the fused layers again
            v = self.sym(lt)
            if not isinstance(v, RealT):
                v = RealT(t)
        if isinstance(v, RealT):
            t = v.tensor
            if not t.is_contiguous(memory_format=torch.channels_last):      # the fused kernels read NHWC
                src, t = t, torch.empty(tuple(t.shape), dtype=self.dtype, device=self.dev, memory_format=torch.channels_last)
                self.steps.append(("eager", lambda _s, src=src, t=t: t.copy_(src)))
                self.eager_nodes.append("to_nhwc")
            f = Full([(Buf(self, t.shape, raw=t), 0)])
            self.env[id(lt)] = f
            return f
        return None

    def plain_buf(self, lt: LazyTensor) -> Optional[Buf]:
        """The value as ONE raw buffer (materialising pending cat / upsample / pre-op through an eager node if needed)."""
        f = self.as_full(lt)
        if f is None:
            return None
        if f.single is not None:
            return f.single
        t = self.materialize_full(lt, f)
        return self.sym(lt).single if isinstance(self.sym(lt), Full) else Buf(self, t.shape, raw=t)

    def force_dense(self, co: ConvOut, residual: Optional[Buf] = None, shortcut=None) -> Buf:
        """Emit a dense (all-tiles) conv into a fresh buffer."""
        f: Full = co.src
        h, w = f.HW
        B = f.B
        cout = int(co.weight.shape[0])
        name = "n%d.conv%dx%d" % (co.node.index, co.k, co.k)
        if co.k == 3 and co.stride == 1:
            idx, block, off, dh, dw = self.all_tiles(h, w, 1), 6, 1, h, w
        elif co.k == 1:
            idx, block, off, dh, dw = self.all_tiles(h, w, 0), 4, 0, h, w
        else:       # 3x3 stride 2 on the (0,1,0,1)-padded input: 5x5 tiles overhang the far edges, where the halo is zero
            idx, block, off, dh, dw = self.all_tiles(h, w, 0), 5, 0, h // 2, w // 2
        dst = self.fresh(B, cout, dh, dw)
        pre, fold = f.pre, None
        if pre is not None and co.k == 1 and not pre.act and not self._per_sample(pre):
            fold, pre = (pre.scale, pre.shift), None          # exact: no halo in a 1x1 conv
        self.emit_conv(name, f.segs, pre, (h, w), idx, block, co.weight, co.bias, co.stride, off, dst, residual=residual, shortcut=shortcut,
                       weight_fold=fold)
        return dst

    @staticmethod
    def _per_sample(pre: Pre) -> bool:
        return (pre.scale is not None and pre.scale.dim() == 2) or (pre.shift is not None and pre.shift.dim() == 2)

    def tile_conv_args(self, co: ConvOut, exact: bool = False):
        """(segs, pre, hw, idx, block, off, stack_src, tile_img) of a conv on tiles.  `exact`: the launch's output stays a tile
        stack that recorded torch calls consume — its row count must be the real tile count, not a padded capacity."""
        st = co.src
        if isinstance(st, RealStack):
            t = st.tensor
            return None, None, (t.shape[2], t.shape[3]), None, int(t.shape[2]), 0, t, None
        g = st.gather
        pre = None
        if st.scale is not None or st.shift is not None or g.activation_name != "identity":
            pre = Pre(self._chan_vec(st.scale, st.src), self._chan_vec(st.shift, st.src), None if g.activation_name == "identity" else g.activation_name)
        if isinstance(st, ModStack):
            pre = pre or Pre()
            pre.mod = ((st.gamma, st.gamma_c0), (st.beta, st.beta_c0), st.slope)
        timg = getattr(g, "tile_images", None)
        if int(g.active_indices.shape[0]) > 0 and not exact and (timg is None or self.batch_slots):
            sl = self.slot(g)                 # fixed capacity, padded with SIGE_TILE_NONE (see IdxSlot)
            idx, timg = sl.buf, sl.tile_img
        else:
            idx = g.active_indices.to(self.dev)
            timg = None if timg is None else timg.to(self.dev)
        return (st.src.segs, pre, st.src.HW, idx, int(g.block_size[0]), int(g.offset[0]), None, timg)

    def _chan_vec(self, t: Optional[torch.Tensor], f: Full) -> Optional[torch.Tensor]:
        """(1|B, C, 1, 1) broadcast operand -> fp32 [C] (or [B, C]) vector."""
        if t is None:
            return None
        C = f.C
        if t.numel() == 1:
            return self.derive(lambda u: u.expand(C).contiguous(), self.vec(t))
        if t.dim() == 4 and t.shape[2] == 1 and t.shape[3] == 1 and t.shape[1] == C:
            if t.shape[0] == 1:
                return self.vec(t)
            return self.vec(t).view(t.shape[0], C)
        raise TraceUnsupported("unsupported affine operand shape %s" % (tuple(t.shape),))

    # ---- eager fallback ------------------------------------------------------------------------------------------
    def runtime_tensor(self, lt: LazyTensor) -> Optional[torch.Tensor]:
        """A real tensor, at a stable address, that holds the value when the program reaches this point."""
        v = self.sym(lt)
        if isinstance(v, RealT):
            return v.tensor
        if isinstance(v, RealStack):
            return v.tensor
        if isinstance(v, Full):
            if v.single is not None:
                v.single.readers.append(None)
                return v.single.raw
            return self.materialize_full(lt, v)
        if isinstance(v, ConvOut):
            if v.on_tiles:
                return self.force_stack(lt, v)
            buf = self.force_dense(v)
            self.env[id(lt)] = Full([(buf, 0)])
            buf.readers.append(None)
            return buf.raw
        if isinstance(v, Stack):
            return self.materialize_stack(lt, v)
        if isinstance(v, Spade) and v.stage == 3:
            t = self._materialize_spade(lt, v)
            if t is not None:
                return t
            self.env.pop(id(lt), None)        # operands the kernel does not take: the recorded calls run as they are
            self.eager(lt.node)
            return self.runtime_tensor(lt)
        if isinstance(v, HeadsOut):           # a consumer other than einops' closing rearrange
            if v.stage == 2:
                t = v.full.view(v.b, v.n, v.h, v.d)
            elif v.stage == 1:
                t = v.bhnd
            else:
                t = torch.empty((v.b * v.h, v.n, v.d), dtype=v.full.dtype, device=v.full.device)
                src, dst = v.bhnd, t.view(v.b, v.h, v.n, v.d)
                self.steps.append(("eager", lambda _s, src=src, dst=dst: dst.copy_(src)))
                self.eager_nodes.append("heads_copy")
            self.env[id(lt)] = RealT(t)
            return t
        # speculative symbolic kinds (or nothing yet): evaluate the producing node eagerly
        if v is None and id(lt) in self._alias_of:
            return self.runtime_tensor(self._alias_of[id(lt)])
        if lt.node is None:
            raise TraceUnsupported("input without a binding")
        self.eager(lt.node)
        return self.runtime_tensor(lt)

    def _materialize_spade(self, lt: LazyTensor, v: Spade) -> Optional[torch.Tensor]:
        x, g, b = self.runtime_tensor(v.x), self.runtime_tensor(v.gamma), self.runtime_tensor(v.beta)
        if not (x.dtype == g.dtype == b.dtype == self.dtype and tuple(x.shape) == tuple(g.shape) == tuple(b.shape) == tuple(lt.shape)
                and self.ex.spade_supported(x, g, b)):
            return None
        out = torch.empty(tuple(lt.shape), dtype=self.dtype, device=self.dev, memory_format=torch.channels_last)
        self.steps.append(("spade", self.ex.prepare_spade(x, g, b, 1.0 if v.slope is None else float(v.slope), out)))
        self.spade_calls += 1
        is_stack = isinstance(self.sym(v.x), RealStack)       # pointwise math on a tile stack yields a tile stack
        self.env[id(lt)] = RealStack(out) if is_stack else RealT(out)
        return out

    def materialize_full(self, lt: LazyTensor, f: Full) -> torch.Tensor:
        B, C = f.B, f.C
        h, w = f.HW
        if f.pad is not None:
            l, r, t_, b_ = f.pad
            out = self.empty(B, C, h + t_ + b_, w + l + r)
        else:
            out = self.empty(B, C, h, w)
        raws = []
        for buf, up in f.segs:
            buf.readers.append(None)
            raws.append((buf.raw, up))
        pre, pad = f.pre, f.pad
        dtype = self.dtype

        def run(_stream):
            parts = [F.interpolate(t, scale_factor=2.0, mode="nearest") if up else t for (t, up) in raws]
            z = parts[0] if len(parts) == 1 else torch.cat(parts, dim=1)
            if pre is not None:
                zf = z.float()
                if pre.scale is not None:
                    zf = zf * (pre.scale.view(1, -1, 1, 1) if pre.scale.dim() == 1 else pre.scale.view(pre.scale.shape[0], -1, 1, 1))
                if pre.shift is not None:
                    zf = zf + (pre.shift.view(1, -1, 1, 1) if pre.shift.dim() == 1 else pre.shift.view(pre.shift.shape[0], -1, 1, 1))
                if pre.act == "swish":
                    zf = zf * torch.sigmoid(zf)
                z = zf.to(dtype)
            if pad is not None:
                z = F.pad(z, pad)
            out.copy_(z)

        self.steps.append(("eager", run))
        self.eager_nodes.append("materialize(%s)" % (lt.node.name if (lt is not None and lt.node is not None) else "value"))
        if lt is not None:
            self.env[id(lt)] = Full([(Buf(self, out.shape, raw=out), 0)])
        return out

    def materialize_stack(self, lt: LazyTensor, st: Stack) -> torch.Tensor:
        g = st.gather
        if getattr(g, "tile_images", None) is not None:
            raise TraceUnsupported("foreign ops on the tile stack of a batch of independent edits")
        f = st.src
        up = 0
        if f.pre is None and f.pad is None and len(f.segs) == 1 and f.segs[0][1] == 1:
            src, up = f.segs[0][0], 1        # Gather(F.interpolate(x, x2)): read the half-resolution tensor, never materialise the big one
        else:
            src = self.plain_of_full(f)
        src.readers.append(None)
        x = src.raw
        idx = g.active_indices.to(self.dev)
        n = int(idx.shape[0])
        out = torch.empty((x.shape[0] * n, x.shape[1], g.block_size[0], g.block_size[1]), dtype=self.dtype, device=self.dev, memory_format=torch.channels_last)
        dev = self.dev
        ex = self.ex
        # the gather's broadcast operands (dense-pass statistics, often): owned copies, so that a refresh rewrites what it reads
        scale, shift = (None if v is None else self.derive(lambda u: u.detach().to(dev).clone(), v) for v in (st.scale, st.shift))

        def run(_stream):
            out.copy_(ex.gather(x, g.block_size, idx, scale, shift, g.activation_name, g.activation_first, up))

        self.steps.append(("eager", run))
        self.eager_nodes.append("gather(n%d)" % lt.node.index)
        if out.shape[1] != lt.shape[1]:          # a zero-padded label map: the recorded channels only
            out = out[:, :lt.shape[1]]
        self.env[id(lt)] = RealStack(out)
        return out

    def plain_of_full(self, f: Full) -> Buf:
        if f.single is not None:
            return f.single
        t = self.materialize_full(None, f)         # concatenated / upsampled / pre-op'ed value needed as one tensor
        return Buf(self, t.shape, raw=t)

    def force_stack(self, lt: LazyTensor, co: ConvOut) -> torch.Tensor:
        """Emit a conv on tiles whose result stays a stack (a foreign op consumes it)."""
        segs, pre, hw, idx, block, off, stack_src, timg = self.tile_conv_args(co, exact=True)
        if timg is not None:
            raise TraceUnsupported("foreign ops on the tile stack of a batch of independent edits")
        n = int(idx.shape[0]) if idx is not None else int(stack_src.shape[0])
        B = 1 if stack_src is not None else segs[0][0].shape[0]
        ro = (block - co.k) // co.stride + 1
        out = torch.empty((B * n, int(co.weight.shape[0]), ro, ro), dtype=self.dtype, device=self.dev, memory_format=torch.channels_last)
        self.emit_conv("n%d.conv_stack" % co.node.index, segs, pre, hw, idx, block, co.weight, co.bias, co.stride, off, None, stack_src=stack_src, dst_stack=out,
                       cin_pad=co.cin_pad, epilogue=co.act, window=self._window_of(co))
        self.env[id(lt)] = RealStack(out)
        return out

    def eager(self, node: Node) -> None:
        """Run the recorded call itself (torch op or operator module) on real tensors at this point of the program."""
        if all(isinstance(self.sym(o), (RealT, RealStack)) for o in node.outs) and node.outs:
            return
        getters: Dict[int, torch.Tensor] = {}
        lazy_strides: Dict[int, Tuple[int, ...]] = {}
        stack_shapes = set()

        def bind(o):
            if isinstance(o, LazyTensor):
                getters[id(o)] = self.runtime_tensor(o)
                with torch._C.DisableTorchFunctionSubclass():
                    lazy_strides[id(o)] = tuple(o.stride())
                if isinstance(self.sym(o), RealStack):
                    stack_shapes.add(tuple(o.shape))
            return o

        lazy._tree_map(bind, node.args)
        lazy._tree_map(bind, node.kwargs)
        is_module_call = isinstance(node.op, str)
        consts: List[torch.Tensor] = []

        def const(o):
            if _is_const(o):
                consts.append(o)
            return o

        lazy._tree_map(const, node.args)
        lazy._tree_map(const, node.kwargs)
        self.derive(None, *consts)       # (an eager node's arguments are frozen in the captured graph)
        if is_module_call and node.name not in ("sige.conv", "sige.gather"):
            self.eager_state.append(node.name)
        if not is_module_call and node.name in _VIEW_OPS and self._static_view(node, getters):
            return
        outs = []
        # Pointwise math between fused layers (SPADE's x*(1+gamma)+beta, leaky_relu, ...: GauGAN) keeps the layout of its operands:
        # when every 4-D operand is an NHWC buffer / stack the result is allocated channels-last too, so the fused launch that
        # reads it needs no NCHW -> NHWC copy (53 such copies per full-size GauGAN step).  Ops that depend on the recorded strides
        # (`view`, operator modules) still get their operands in the recorded layout (see `sub`).
        big = [g for g in getters.values() if g.dim() == 4]

        def nhwc_like(g):      # channels innermost (an NHWC buffer / stack, or a channel slice of one: torch.split(gamma_beta, C, dim=1))
            return g.shape[1] > 1 and g.shape[2] * g.shape[3] > 1 and g.stride(1) == 1

        follow_nhwc = (not is_module_call and node.name in _POINTWISE and any(nhwc_like(g) for g in big)
                       and all(nhwc_like(g) or g.shape[1] == 1 or tuple(g.shape[2:]) == (1, 1) for g in big))
        for o in node.outs:
            with torch._C.DisableTorchFunctionSubclass():
                st = tuple(o.stride())
            # the recorded memory layout: later `view`s of this value were validated against exactly these strides
            act_like = o.dtype.is_floating_point and o.dim() >= 3
            if follow_nhwc and o.dim() == 4:
                outs.append(torch.empty(tuple(o.shape), dtype=self.dtype if act_like else o.dtype, device=self.dev, memory_format=torch.channels_last))
            else:
                outs.append(torch.empty_strided(tuple(o.shape), st, dtype=self.dtype if act_like else o.dtype, device=self.dev))

        # Precision of a recorded call (mixed-precision steps: fp32 model, fp16/bf16 step): it runs under autocast — GEMM-like
        # ops on the tensor cores in the step's dtype, softmax / norms / transcendental math in fp32 — on the tensors as they
        # are stored: activation-like values (>= 3-D) in the step's dtype, small ones (time embeddings, statistics) in the
        # dtype the model computed them in.  Constant fp32 operands of GEMM-like ops (weights) are converted once, here.
        gemm_like = node.name in ("linear", "bmm", "matmul", "conv2d", "conv1d", "baddbmm", "addmm", "mm", "einsum")
        half_consts: Dict[int, torch.Tensor] = {}

        def sub(o):
            if not isinstance(o, LazyTensor):
                if gemm_like and _is_const(o) and o.dtype == torch.float32 and self.dtype != torch.float32:
                    if id(o) not in half_consts:
                        half_consts[id(o)] = o.detach().to(self.dtype)
                    return half_consts[id(o)]
                return o
            g = getters[id(o)]
            if casts_to_model_dtype and g.dtype != o.dtype:
                g = g.to(o.dtype)          # an operator module that reads its caches falls back to its eager kernels in the MODEL's dtype
            want = lazy_strides[id(o)]
            if stride_sensitive and g.dim() >= 2 and tuple(g.stride()) != want and g.numel() > 0:
                # `view` was validated against the model's memory layout (NCHW tensors), the buffers are NHWC
                g = torch.empty_strided(tuple(g.shape), want, dtype=g.dtype, device=g.device).copy_(g)
            return g

        stride_sensitive = is_module_call or node.name in ("view", "view_as", "as_strided")
        casts_to_model_dtype = is_module_call and node.name not in ("sige.conv", "sige.gather")     # these two read no cache: the step's dtype
        op, module, multi = node.op, node.module, node.multi
        use_autocast = self.dev.type == "cuda" and self.dtype in (torch.float16, torch.bfloat16) and not is_module_call
        dev_type, ac_dtype = self.dev.type, self.dtype

        # The result of a recorded call has to live at a stable address (fused launches hold raw pointers), so by default it is
        # COPIED into its persistent tensor: one extra launch per recorded call (9 % of the full-size SD step).  The common calls
        # have an out= form that writes there directly; it is adopted per node only after the first (warm-up) run has checked,
        # on the real data, that it reproduces the recorded call bit for bit.
        fast = None if (is_module_call or multi or len(outs) != 1) else _out_variant(node.name, op)
        state = {"mode": 0 if fast is not None else 2}        # 0 undecided, 1 out= form, 2 call + copy

        def run(_stream):
            args = lazy._tree_map(sub, node.args)
            kwargs = lazy._tree_map(sub, node.kwargs)
            if state["mode"] == 1:
                fast(args, kwargs, outs[0])
                return
            with torch.autocast(device_type=dev_type, dtype=ac_dtype, enabled=use_autocast):
                if isinstance(op, str):
                    res = module(*args)
                else:
                    res = op(*args, **kwargs)
            res = list(res) if multi else [res]
            for dst, r in zip(outs, [r for r in res if isinstance(r, torch.Tensor)]):
                dst.copy_(r)
            if state["mode"] == 0:
                ok = False
                if not (dev_type == "cuda" and torch.cuda.is_current_stream_capturing()):
                    try:
                        tmp = torch.empty_strided(tuple(outs[0].shape), tuple(outs[0].stride()), dtype=outs[0].dtype, device=outs[0].device)
                        fast(args, kwargs, tmp)
                        ok = tmp.dtype == outs[0].dtype and bool(torch.equal(_bits(tmp), _bits(outs[0])))
                    except Exception:  # noqa: BLE001  (dtype promotion the out= form refuses, unsupported overload, ...)
                        ok = False
                state["mode"] = 1 if ok else 2

        self.steps.append(("eager", run))
        self.eager_nodes.append(node.name)
        is_stack_op = node.name in ("sige.gather", "sige.conv", "sige.scatter_gather")
        for o, t in zip(node.outs, outs):
            # pointwise math on a tile stack yields a tile stack (GauGAN's SPADE modulation between Gather and the conv)
            self.env[id(o)] = RealStack(t) if (is_stack_op or (not isinstance(node.op, str) and tuple(o.shape) in stack_shapes)) else RealT(t)

    def _static_view(self, node: Node, getters: Dict[int, torch.Tensor]) -> bool:
        """A pure view op (reshape / permute / split / indexing ...) of persistent tensors is evaluated ONCE, here: its result
        aliases the persistent buffer, which every replay refreshes in place — no kernel, no copy at run time."""
        def sub(o):
            return getters[id(o)] if isinstance(o, LazyTensor) else o

        try:
            with torch.no_grad():
                res = node.op(*lazy._tree_map(sub, node.args), **lazy._tree_map(sub, node.kwargs))
        except Exception:  # noqa: BLE001  (e.g. `view` on a layout it was not recorded on: the run-time path fixes the strides)
            return False
        res = list(res) if node.multi else [res]
        tensors = [r for r in res if isinstance(r, torch.Tensor)]
        bases = {g.untyped_storage().data_ptr() for g in getters.values()}
        if len(tensors) != len(node.outs) or not all(r.untyped_storage().data_ptr() in bases and tuple(r.shape) == tuple(o.shape)
                                                     for r, o in zip(tensors, node.outs)):
            return False           # the op had to copy (or is not a view): evaluate it at run time
        for o, r in zip(node.outs, tensors):
            self.env[id(o)] = RealT(r)
        self.view_nodes += 1
        return True

    # ------------------------------------------------------------------ node handlers
    def _lower(self, node: Node) -> None:
        h = getattr(self, "_h_" + node.name.replace(".", "_").strip("_"), None)
        done = False
        if h is not None:
            done = h(node) is not False
        if not done:
            # unknown op: decide later (evaluated eagerly if and when a consumer needs its value)
            pass

    @staticmethod
    def _bind(node: Node, names: Sequence[str], defaults: Dict[str, Any]):
        vals = dict(defaults)
        for n_, a in zip(names, node.args):
            vals[n_] = a
        vals.update(node.kwargs)
        return vals

    # ---- convolutions
    def _conv_common(self, node: Node, x, weight, bias, stride, padding, dilation, groups, src: Optional[Stack] = None) -> bool:
        """`src`: the conv's source when it is not x's symbolic value (a ModStack)."""
        if not (_is_const(weight) and (bias is None or _is_const(bias))) or weight.dim() != 4:
            return False
        self.derive(None, weight, bias)
        k, s, p = _pair(weight.shape[2:]), _pair(stride), (_pair(padding) if not isinstance(padding, str) else None)
        if p is None or k[0] != k[1] or s[0] != s[1] or p[0] != p[1] or _pair(dilation) != (1, 1) or groups != 1:
            return False
        k, s, p = k[0], s[0], p[0]
        cout, cin = int(weight.shape[0]), int(weight.shape[1])
        out = node.outs[0]
        v = self.sym(x) if src is None else src
        if isinstance(v, GNVal):
            if k == 3 and s == 1 and p == 1 and cout <= 8 and cin % 16 == 0 and v.act in (None, "swish") and self.ex.tail_supported(cin, cout):
                res = torch.empty((v.src.shape[0], cout, v.src.shape[2], v.src.shape[3]), dtype=self.dtype, device=self.dev)
                v.src.readers.append(None)
                x_raw = v.src.raw
                slot = len(self.steps)
                self.steps.append(("tail", None))
                ex = self.ex

                def prep(slot=slot, v=v, x_raw=x_raw, res=res):
                    self.steps[slot] = ("tail", ex.prepare_tail(x_raw, v.groups, v.eps, v.weight, v.bias, v.act or "identity", weight, bias, res))

                self._pending_prepare.append(prep)
                self.env[id(out)] = RealT(res)
                return True
            return False
        if isinstance(v, (Stack, RealStack)):
            src_c = v.C if isinstance(v, WinStack) else (v.src.C if isinstance(v, Stack) else int(v.tensor.shape[1]))
            nsegs = len(v.src.segs) if isinstance(v, Stack) else 1
            if p != 0 or cout % 8 != 0 or not (cin % 64 == 0 or self._narrow(cin, src_c, nsegs, cout, k, s)):
                return False
            if isinstance(v, Stack) and (v.gather.activation_first and v.gather.activation_name != "identity"):
                return False
            block = int(v.gather.block_size[0]) if isinstance(v, Stack) else int(v.tensor.shape[2])
            if isinstance(v, Stack) and v.gather.block_size[0] != v.gather.block_size[1]:
                return False
            if block < k or (block - k) % s != 0:
                return False
            self.env[id(out)] = ConvOut(node, v, weight, bias, k, s, 0, cin_pad=src_c - cin)
            return True
        if isinstance(v, RealT) and v.tensor.dim() == 4 and cin <= 4 and k == 3 and s == 1 and p == 1 and cout % 8 == 0 and v.tensor.shape[1] == cin:
            t = v.tensor
            if not t.is_contiguous(memory_format=torch.channels_last):
                return False
            dst = self.fresh(t.shape[0], cout, t.shape[2], t.shape[3])
            rec = ConvInRec(t, weight, bias, dst)
            dst.producers.append(rec)
            self.conv_ins.append(rec)
            slot = len(self.steps)
            self.steps.append(("conv_in", None))

            def prep(slot=slot, rec=rec):
                self.steps[slot] = ("conv_in", self.ex.prepare_conv_in(rec))

            self._pending_prepare.append(prep)
            self.env[id(out)] = Full([(dst, 0)])
            return True
        f = self.as_full(x)
        if f is None or cout % 8 != 0 or len(f.segs) > 2:
            return False
        if (cin % 64 != 0 or any(b.shape[1] % 64 for b, _ in f.segs)) and not (f.C == cin and self._narrow(cin, cin, len(f.segs), cout, k, s)):
            return False
        h, w = f.HW
        if h % 4 or w % 4:
            return False
        if f.pad is not None:
            if not (f.pad == (0, 1, 0, 1) and k == 3 and s == 2 and p == 0):
                return False
        elif not ((k == 3 and s == 1 and p == 1) or (k == 1 and s == 1 and p == 0)):
            return False
        if f.pre is not None and f.pre.act not in (None, "swish"):
            return False
        self.env[id(out)] = ConvOut(node, f, weight, bias, k, s, p)
        return True

    def _narrow(self, cin: int, src_c: int, nsegs: int, cout: int, k: int, stride: int) -> bool:
        """A conv whose input width is a multiple of 8 but not of 64 (the narrow layers of pruned / compressed models) is one
        tile-conv launch on a single source when the executor runs such launches.  src_c > cin: the source is a label map
        zero-padded to round_up(cin, 8) channels, and the weight is padded to match."""
        ok = getattr(self.ex, "narrow_conv_supported", None)
        return (ok is not None and nsegs == 1 and src_c % 8 == 0 and src_c in (cin, (cin + 7) // 8 * 8)
                and ok(src_c, cout, k, stride))

    @staticmethod
    def _narrow_dense(v) -> bool:
        """A dense conv of a narrow input (the dense sub-mobile SPADE's 1x1 gamma conv): SPADE's modulation reads its buffer, as it
        read the result of the eager conv before such convs were lowered."""
        return isinstance(v, ConvOut) and not v.on_tiles and int(v.weight.shape[1]) % 64 != 0

    def _padded_map(self, x) -> Optional[Full]:
        """A map whose channel count is not a multiple of 8 (GauGAN's 36-channel label map), for a Gather when the executor runs
        narrow tile convs: written once per step into a channels-last buffer of round_up(C, 8) channels in the step's dtype, the
        channels behind C zero.  That copy is the layout copy the map needs anyway."""
        if (getattr(self.ex, "narrow_conv_supported", None) is None or not isinstance(x, LazyTensor) or x.dim() != 4 or x.shape[1] % 8 == 0
                or not x.dtype.is_floating_point):
            return None
        if id(x) not in self._padded_maps:
            src = self.runtime_tensor(x)
            B, C, H, W = (int(d) for d in src.shape)
            t = self.empty(B, (C + 7) // 8 * 8, H, W)
            t.zero_()
            self.steps.append(("eager", lambda _s, src=src, dst=t[:, :C]: dst.copy_(src)))
            self.eager_nodes.append("to_nhwc")
            self._padded_maps[id(x)] = Full([(Buf(self, t.shape, raw=t), 0)])
        return self._padded_maps[id(x)]

    def _h_conv2d(self, node: Node):
        a = self._bind(node, ("input", "weight", "bias", "stride", "padding", "dilation", "groups"),
                       {"bias": None, "stride": 1, "padding": 0, "dilation": 1, "groups": 1})
        return self._conv_common(node, a["input"], a["weight"], a["bias"], a["stride"], a["padding"], a["dilation"], a["groups"])

    def _h_sige_conv(self, node: Node):
        m = node.module
        if isinstance(m.padding, str) or m.padding_mode != "zeros":
            return False
        x = node.args[0]
        if self._separable_conv(node, m, x):
            return True
        mod = self._modulated(x, m.weight, m.stride)
        if mod is None:
            mod = self._windowed(x, m.weight, m.stride)
        if mod is None and not isinstance(self.sym(x), (Stack, RealStack)) and x.dim() == 4:      # SIGEConv2d in sparse mode always sees a tile stack
            t = self.runtime_tensor(x)
            if not t.is_contiguous(memory_format=torch.channels_last):
                src, t = t, torch.empty(tuple(t.shape), dtype=self.dtype, device=self.dev, memory_format=torch.channels_last)
                self.steps.append(("eager", lambda _s, src=src, t=t: t.copy_(src)))
                self.eager_nodes.append("to_nhwc")
            self.env[id(x)] = RealStack(t)
        return self._conv_common(node, node.args[0], m.weight, m.bias, m.stride, 0, m.dilation, m.groups, src=mod)

    def _modulated(self, x, weight, stride) -> Optional[ModStack]:
        """The source of a conv that reads SPADE's modulation `leaky((x*scale+shift) * (1 + gamma) + beta)` (Spade stage 3) of three lazy
        Stacks of single buffers cut with ONE tile list (reference gaugan/models/sige_normalization.py:84-86: x from the block's
        Gather with the batch norm folded in, gamma / beta re-gathered from the separable launches' buffers), when the executor
        runs such launches; None otherwise (the modulation is then evaluated on its own).  When the executor also runs strided
        launches, gamma and beta may be torch.split windows of one such Stack (the full SPADE's `gamma, beta = torch.split(
        gamma_beta, norm_nc)`, reference gaugan/models/sige_normalization.py:80)."""
        ok = getattr(self.ex, "modulated_conv_supported", None)
        v = self.sym(x) if isinstance(x, LazyTensor) else None
        if ok is None or not isinstance(v, Spade) or v.stage != 3 or (v.slope is not None and not math.isfinite(v.slope)):
            return None
        sx = self.sym(v.x)
        if not isinstance(sx, Stack) or isinstance(sx, (ModStack, WinStack)):
            return None
        g, f = sx.gather, sx.src
        if (not self._batch_ok(g) or g.activation_name != "identity" or g.block_size[0] != g.block_size[1]
                or int(g.active_indices.shape[0]) == 0 or not f.plain or len(f.segs) != 1):
            return None
        windows = getattr(self.ex, "strided_conv_supported", None) is not None
        parts = []
        for lt in (v.gamma, v.beta):
            t = self.sym(lt)
            if isinstance(t, Stack) and not isinstance(t, (ModStack, WinStack)):
                win = (t, 0, t.src.C)
            elif t is None and windows and isinstance(lt, LazyTensor):
                win = self._stack_window(lt)
            else:
                return None
            if win is None:
                return None
            t, c0, C = win
            buf = t.src.single
            if (buf is None or t.scale is not None or t.shift is not None or t.gather.activation_name != "identity"
                    or not self._same_gather(t.gather, g) or (buf.shape[0], *buf.shape[2:]) != (f.B, *f.HW) or C != f.C or c0 % 8):
                return None
            parts.append((buf, c0))
        k, s = _pair(weight.shape[2:]), _pair(stride)
        if k[0] != k[1] or s[0] != s[1] or not ok(f.C, int(weight.shape[0]), k[0], s[0]):
            return None
        (gb, g0), (bb, b0) = parts
        return ModStack(sx, gb, bb, 1.0 if v.slope is None else float(v.slope), gamma_c0=g0, beta_c0=b0)

    def _stack_window(self, lt: LazyTensor) -> Optional[Tuple[Stack, int, int]]:
        """(Stack, first channel, channels) of a torch.split part along dim 1 of a lazy Stack that has no other symbolic form (SPADE's
        actv_0 / actv_1 / actv_s, and gamma / beta of gamma_beta); None otherwise."""
        if self.sym(lt) is not None or lt.node is None or lt.node.name != "split":
            return None
        a = self._bind(lt.node, ("tensor", "split_size_or_sections", "dim"), {"dim": 0})
        st = self.sym(a["tensor"]) if isinstance(a["tensor"], LazyTensor) else None
        if not (isinstance(st, Stack) and not isinstance(st, (ModStack, WinStack)) and a["dim"] == 1
                and isinstance(a["split_size_or_sections"], int)):
            return None
        return st, lt.slot * a["split_size_or_sections"], int(lt.shape[1])

    def _windowed(self, x, weight, stride) -> Optional[WinStack]:
        """The source of a conv on a torch.split window of a lazy Stack of one buffer (no pre-op), read in place by a strided
        launch when the executor runs such launches; None otherwise (the split is then evaluated on its own)."""
        ok = getattr(self.ex, "strided_conv_supported", None)
        if ok is None or not isinstance(x, LazyTensor):
            return None
        win = self._stack_window(x)
        if win is None:
            return None
        st, c0, C = win
        g = st.gather
        if (st.src.single is None or st.scale is not None or st.shift is not None or g.activation_name != "identity"
                or g.block_size[0] != g.block_size[1] or not self._batch_ok(g) or c0 % 8 or C % 8):
            return None
        k, s = _pair(weight.shape[2:]), _pair(stride)
        if k[0] != k[1] or s[0] != s[1] or not ok(C, int(weight.shape[0]), k[0], s[0]):
            return None
        return WinStack(st, c0, C)

    # ---- GAN Compression's separable conv: depthwise 3x3 -> per-channel affine -> 1x1, one launch per SPADE layer
    def _separable_conv(self, node: Node, m, x) -> bool:
        """Depthwise 3x3 SIGEConv2d on a tile stack (or a channel window of one) -> DWConv; 1x1 SIGEConv2d on a DWConv -> SepOut."""
        supported = getattr(self.ex, "separable_supported", None)
        if supported is None or not isinstance(x, LazyTensor) or _pair(m.stride) != (1, 1) or _pair(m.dilation) != (1, 1):
            return False
        w, b = m.weight, m.bias
        cout, cin_g = int(w.shape[0]), int(w.shape[1])
        v = self.sym(x)
        if isinstance(v, DWConv):
            if (tuple(w.shape[2:]) != (1, 1) or m.groups != 1 or cin_g != v.C or self.n_uses(x) != 1
                    or not supported(v.C, cout)):
                return False
            self.env[id(node.outs[0])] = SepOut(v, w, b)
            return True
        cin = int(x.shape[1])
        if tuple(w.shape[2:]) != (3, 3) or m.groups != cin or cout != cin or cin_g != 1 or tuple(x.shape[2:]) != (6, 6) or not supported(cin, cin):
            return False
        src = self._separable_source(x)
        if src is None:
            return False
        self.env[id(node.outs[0])] = DWConv(src[0], src[1], w, b)
        return True

    def _separable_source(self, x: LazyTensor):
        """(RealStack with an NHWC tensor | plain lazy Stack, channel offset) of a depthwise conv's input: a 6x6 tile stack or a
        torch.split channel slice of one (SPADE's actv_0 / actv_1 / actv_s, reference
        gaugan/models/sub_mobile_spade_generators/sige_fused_sub_mobile_spade_generator.py:158-169); None otherwise.  (A
        SIGEConv2d in sparse mode only ever reads tile stacks, so a 6x6 "image" here is one.)"""
        v = self.sym(x)
        c0 = 0
        win = self._stack_window(x)
        if win is not None:
            # torch.split of the lazy re-gather of a buffer a fused launch wrote (actvs after a fused mlp_shared): the window is
            # read in place through the tile list
            v, c0 = win[0], win[1]
        if v is None and x.node is not None:
            self.runtime_tensor(x)               # a stack from a call the lowering does not know (the eager scatter_gather)
            v = self.sym(x)
        if isinstance(v, Stack):
            g = v.gather
            if (v.src.single is None or v.scale is not None or v.shift is not None or g.activation_name != "identity"
                    or tuple(g.block_size) != (6, 6) or not self._batch_ok(g) or c0 % 8):
                return None
            return v, c0
        if isinstance(v, ChanSlice):             # torch.split of a stack: the whole stack became one NHWC buffer
            v.buf.readers.append(None)
            t, c0 = v.buf.raw, v.c0
        elif isinstance(v, Full) and v.single is not None:
            v.single.readers.append(None)
            t = v.single.raw
        elif isinstance(v, (RealStack, RealT)):
            t = v.tensor
        else:
            return None
        if t.dim() != 4 or tuple(t.shape[2:]) != (6, 6) or t.shape[1] % 8 or c0 % 8:
            return None
        if not t.is_contiguous(memory_format=torch.channels_last):
            if id(t) not in self._nhwc_stacks:       # one copy per stack, shared by every slice that reads it
                nhwc = torch.empty(tuple(t.shape), dtype=self.dtype, device=self.dev, memory_format=torch.channels_last)
                self.steps.append(("eager", lambda _s, src=t, dst=nhwc: dst.copy_(src)))
                self.eager_nodes.append("to_nhwc")
                self._nhwc_stacks[id(t)] = nhwc
            t = self._nhwc_stacks[id(t)]
        return RealStack(t), c0

    def _sep_affine(self, node: Node, is_mul: bool) -> bool:
        """`x * scale` / `x + shift` by a constant per-channel [1, C, 1, 1] (or scalar) tensor on a DWConv."""
        a, b = node.args[0], node.args[1]
        x, c = (a, b) if isinstance(a, LazyTensor) else (b, a)
        v = self.sym(x) if isinstance(x, LazyTensor) else None
        if not isinstance(v, DWConv) or not _is_const(c) or self.n_uses(x) != 1 or tuple(node.outs[0].shape) != tuple(x.shape):
            return False
        if not (c.numel() == 1 or (c.dim() == 4 and tuple(c.shape) == (1, v.C, 1, 1))):
            return False
        self.derive(None, c)            # (folded into the separable launch's weights by the executor)
        cv = self.vec(c).expand(v.C) if c.numel() == 1 else self.vec(c)
        if is_mul:
            scale = cv if v.scale is None else self.derive(torch.mul, v.scale, cv)
            shift = None if v.shift is None else self.derive(torch.mul, v.shift, cv)
        else:
            scale, shift = v.scale, (cv if v.shift is None else self.derive(torch.add, v.shift, cv))
        self.env[id(node.outs[0])] = DWConv(v.src, v.c0, v.weight, v.bias, scale, shift, v.consts + (c,))
        return True

    def _sep_stack(self, v) -> bool:
        """Is `v` the lazy re-gather of a buffer a separable launch writes?"""
        return isinstance(v, Stack) and v.src.single is not None and any(v.src.single is br[3] for r in self.separable for br in r.branches)

    def _sep_fits(self, so: SepOut, g) -> bool:
        """Can the launch scatter through Gather `g`'s tile set?"""
        if not self._batch_ok(g) or tuple(g.block_size) != (6, 6) or tuple(g.offset)[0] != tuple(g.offset)[1]:
            return False
        src = so.dw.src
        if isinstance(src, Stack):
            return self._same_gather(src.gather, g)
        if getattr(g, "tile_images", None) is not None:      # a materialised stack has no per-edit lists
            return False
        return int(src.tensor.shape[0]) % max(1, int(g.active_indices.shape[0])) == 0 and int(g.active_indices.shape[0]) > 0

    def _sep_emit(self, node: Node, so: SepOut, dst: Buf, g) -> None:
        """Add the branch to the previous launch if that one is the other branch of the same SPADE layer (same source window,
        same tile set, emitted just before), else open a new launch."""
        dw = so.dw
        timg = None
        if isinstance(dw.src, Stack):
            f = dw.src.src
            sl = self.slot(g)
            src, src_stack, idx, timg = f.single.raw, False, sl.buf, sl.tile_img
            f.single.readers.append((idx, 6, 0, timg))
        else:
            src, src_stack, idx = dw.src.tensor, True, g.active_indices.to(self.dev)
        last = self.separable[-1] if self.separable else None
        if (last is not None and len(last.branches) == 1 and last.slot == len(self.steps) - 1 and last.src is src and last.c0 == dw.c0
                and last.idx is idx and last.Cin == dw.C and last.Cout == int(so.weight.shape[0]) and last.batch == dst.shape[0]):
            last.branches.append((dw, so.weight, so.bias, dst))
            last.name += "+" + self._module_name(node)
        else:
            rec = SepLaunch(self._module_name(node), src, src_stack, dw.c0, idx, int(g.offset[0]), dst.shape[0], len(self.steps))
            rec.pdl, rec.tile_img = self.pdl, timg
            rec.branches.append((dw, so.weight, so.bias, dst))
            self.separable.append(rec)
            self.steps.append(("separable", None))
            ex = self.ex

            def prep(rec=rec):
                self.steps[rec.slot] = ("separable", ex.prepare_separable(rec))

            self._pending_prepare.append(prep)
        slot = next((sl for sl in self.slots.values() if sl.buf is idx and timg is None), None)
        self.cache_writers.append((dst, slot, int(g.offset[0]), 1, 4))
        _ = dst.raw               # written in place every step: the buffer must exist (initialised from the module's cache)

    # ---- operator modules
    def _h_sige_gather(self, node: Node):
        x, scale, shift = node.args
        g = node.module
        if not (scale is None or _is_const(scale)) or not (shift is None or _is_const(shift)):
            return False
        f = self.as_full(x)
        if f is None and scale is None and shift is None and g.activation_name == "identity":
            f = self._padded_map(x)
        if f is None or f.pre is not None or f.pad is not None:
            return False
        self.env[id(node.outs[0])] = Stack(f, g, scale, shift)
        return True

    def _tile_emit(self, node: Node, co: ConvOut, dst: Buf, residual: Optional[Buf] = None, shortcut=None, name: str = "", gather=None) -> None:
        segs, pre, hw, idx, block, off, stack_src, timg = self.tile_conv_args(co)
        if stack_src is not None and gather is not None:      # a materialised stack scattered through `gather`'s tile set
            idx, off = co.src.slot.buf if co.src.slot is not None else gather.active_indices.to(self.dev), int(gather.offset[0])
            if co.src.slot is not None:
                timg = co.src.slot.tile_img        # (a batch: the slot's per-edit lists, one per E * cap stack row)
        self.emit_conv(name or ("n%d" % node.index), segs, pre, hw, idx, block, co.weight, co.bias, co.stride, off, dst, residual=residual,
                       shortcut=shortcut, stack_src=stack_src, tile_img=timg, cin_pad=co.cin_pad, epilogue=co.act, window=self._window_of(co))

    @staticmethod
    def _window_of(co: ConvOut) -> Optional[Tuple[int, int]]:
        return (co.src.c0, co.src.c0 + co.src.C) if isinstance(co.src, WinStack) else None

    def _module_name(self, node: Node) -> str:
        return self.module_names.get(id(node.module), "n%d" % node.index)

    def _batch_ok(self, g) -> bool:
        """Can the SPADE launches (modulated, windowed, separable) read Gather `g`'s tile set?  One edit always; a batch of edits
        when the executor runs them on per-edit lists over operands of E images."""
        return getattr(g, "tile_images", None) is None or self.per_image_ops

    @staticmethod
    def _same_gather(a, g) -> bool:
        """Is `a` (a Gather, or the geometry stub a ScatterGather hands on) the tile set of Gather `g`?"""
        return a is g or (getattr(a, "active_indices", None) is g.active_indices and tuple(a.block_size) == tuple(g.block_size)
                          and tuple(a.offset) == tuple(g.offset))

    def _h_sige_scatter(self, node: Node):
        x, residual = node.args
        m = node.module
        co = self.sym(x)
        if isinstance(co, SepOut):         # the shortcut SPADE's gamma / beta: Scatter, then a Gather of its own geometry
            g = m.gather.module
            if residual is not None or self.n_uses(x) != 1 or not self._sep_fits(co, g):
                return False
            dst = self.cached(m.original_outputs[m.cache_id], g.num_edits)
            self._sep_emit(node, co, dst, g)
            self.env[id(node.outs[0])] = Full([(dst, 0)])
            return True
        if not (isinstance(co, ConvOut) and co.on_tiles):
            return False
        # (a conv output that is ALSO consumed as a stack — SD's transformer scatters proj_in's tiles and keeps them as
        #  tokens, sige_attention.py:153-160 — is launched once per form: scatter form here, stack form at its other consumer)
        g = m.gather.module
        if isinstance(co.src, Stack) and not self._same_gather(co.src.gather, g):
            return False
        if isinstance(co.src, RealStack) and (int(co.src.tensor.shape[2]) != int(g.block_size[0]) or g.block_size[0] != g.block_size[1]
                                              or (co.src.slot is not None and co.src.slot is not self.slots.get(id(g.active_indices)))):
            return False
        res_buf = None
        if residual is not None:
            if _is_const(residual) or co.act is not None:      # (the model adds the residual AFTER the activation)
                return False
            res_buf = self.plain_buf(residual)
            if res_buf is None:
                return False
        cache = m.original_outputs[m.cache_id]
        dst = self.cached(cache, g.num_edits)
        if res_buf is not None and tuple(res_buf.shape) != tuple(dst.shape):
            return False
        self._tile_emit(node, co, dst, residual=res_buf, name=self._module_name(node), gather=g)
        self.env[id(node.outs[0])] = Full([(dst, 0)])
        return True

    def _h_sige_scatter_gather(self, node: Node):
        x, scale, shift = node.args
        m = node.module
        co = self.sym(x)
        sep = isinstance(co, SepOut)
        if not ((sep or (isinstance(co, ConvOut) and co.on_tiles)) and self.n_uses(x) == 1):
            return False
        if not (scale is None or _is_const(scale)) or not (shift is None or _is_const(shift)):
            return False
        g = m.gather.module
        if sep:
            if not self._sep_fits(co, g):
                return False
        elif isinstance(co.src, Stack) and not self._same_gather(co.src.gather, g):
            return False
        elif isinstance(co.src, RealStack) and (int(co.src.tensor.shape[2]) != int(g.block_size[0]) or g.block_size[0] != g.block_size[1] or g.tile_images is not None):
            return False          # (a materialised stack — GauGAN's SPADE convs read torch math on the tiles — scatters through g's tile set)
        dst = self.cached(m.original_outputs[m.cache_id], g.num_edits)
        if sep:
            self._sep_emit(node, co, dst, g)
        else:
            self._tile_emit(node, co, dst, name=self._module_name(node), gather=g)

        class _G:        # the second gather re-uses the paired gather's geometry with this module's activation
            pass

        g2 = _G()
        g2.active_indices, g2.block_size, g2.offset, g2.tile_images = g.active_indices, g.block_size, g.offset, g.tile_images
        g2.real = g
        g2.activation_name, g2.activation_first = m.activation_name, m.activation_first
        self.env[id(node.outs[0])] = Stack(Full([(dst, 0)]), g2, scale, shift)
        return True

    def _h_sige_scatter_block_residual(self, node: Node):
        x, residual = node.args
        m = node.module
        co, sc = self.sym(x), self.sym(residual)
        if not (isinstance(co, ConvOut) and isinstance(sc, ConvOut) and co.on_tiles and sc.on_tiles and self.n_uses(x) == 1 and self.n_uses(residual) == 1
                and co.act is None and sc.act is None):
            return False
        # sources: lazy gathers (DDPM) or materialised stacks (GauGAN: SPADE's torch math sits between the Gather and the conv —
        # reference gaugan/models/spade_generators/sige_fused_spade_generator.py:160-198 — such a launch scatters through the
        # module's own tile sets and always takes the un-fused form below)
        main_real, sc_real = isinstance(co.src, RealStack), isinstance(sc.src, RealStack)
        # (the fused shortcut reads its source raw and whole)
        modulated = isinstance(co.src, (ModStack, WinStack)) or isinstance(sc.src, (ModStack, WinStack))
        if not ((isinstance(co.src, Stack) or main_real) and (isinstance(sc.src, Stack) or sc_real)):
            return False
        mg, sg = m.main_gather.module, m.shortcut_gather.module

        def real_ok(c, g):
            return int(c.src.tensor.shape[2]) == int(g.block_size[0]) and g.block_size[0] == g.block_size[1] and g.tile_images is None

        if (main_real and not real_ok(co, mg)) or (not main_real and not self._same_gather(co.src.gather, mg)):
            return False
        if sc_real:
            if not real_ok(sc, sg):
                return False
        elif sc.src.gather is not sg or sc.k != 1 or ((sc.src.scale is not None or sc.src.shift is not None) and not isinstance(sc.src, ModStack)) \
                or sg.activation_name != "identity":
            return False
        cid = m.cache_id
        dst = self.cached(m.original_outputs[cid], mg.num_edits)
        skip = self.cached(m.original_residuals[cid], mg.num_edits)
        idx, off = mg.active_indices.to(self.dev), int(mg.offset[0])
        sidx, soff = sg.active_indices.to(self.dev), int(sg.offset[0])
        sc_full: Optional[Full] = None if sc_real else sc.src.src
        # the shortcut's active tiles must sit on the main conv's output-tile grid and be a subset of it: then evaluating the
        # shortcut on those main tiles (and adding the cached shortcut output elsewhere) IS the reference's
        # `out += fresh - cached` patch (sige/cuda/scatter_kernel.cu:46-74)
        width = 1 << 16
        main_key = (idx[:, 0].long() + off) * width + (idx[:, 1].long() + off)
        sc_key = (sidx[:, 0].long() + soff) * width + (sidx[:, 1].long() + soff)
        if mg.tile_images is not None:         # batch of edits: a tile is (image, origin)
            main_key = main_key + mg.tile_images.to(self.dev).long() * (width * width)
            sc_key = sc_key + sg.tile_images.to(self.dev).long() * (width * width)
        subset = bool(torch.isin(sc_key, main_key).all()) and tuple(mg.block_stride) == tuple(sg.block_stride) == (4, 4) \
            and int(sg.block_size[0]) == 4 and int(mg.block_size[0]) == 6
        fuse = (not main_real and not sc_real and not modulated and self.fuse_shortcut and self.tc5 and self.producer_preop and subset and co.k == 3 and co.stride == 1
                and all(up == 0 for _, up in sc_full.segs) and len(sc_full.segs) <= 2 and sc_full.plain
                and int(sc.weight.shape[1]) % 64 == 0 and int(co.weight.shape[1]) % 64 == 0)
        name = self._module_name(node)
        if fuse:
            if mg.tile_images is None or self.batch_slots:
                ms, ss = self.slot(mg), self.slot(sg)      # one flag per row of the main conv's list; padding rows carry flag 0
                flags = _shortcut_flags(ms, off, ss, soff)[0].contiguous()
                self.flag_recipes.append((flags, ms, off, ss, soff))
            else:                                      # one flag per row of the concatenated lists of a batch
                flags = torch.isin(main_key, sc_key).to(torch.uint8).contiguous()
            shortcut = ([b for b, _ in sc_full.segs], sc.weight, sc.bias, flags)
            n_fused = len(self.fused)
            self._tile_emit(node, co, dst, residual=skip, shortcut=shortcut, name=name)
            if len(self.fused) > n_fused and mg.tile_images is None:
                # the shortcut's output exists only inside conv2's launch: sparse_update relaunches it into `skip` (the un-fused form)
                self.shortcut_relaunches.append((name + ".shortcut", shortcut[0], sc.weight, sc.bias, skip, ss, soff, self.fused[-1]))
                self.cache_writers.append((skip, ss, soff, 1, 4))
        else:
            if not subset:
                return False
            # un-fused: the shortcut's own launch refreshes its tiles of `skip`, then conv2 adds `skip` as the residual
            self._tile_emit(node, sc, skip, name=name + ".shortcut", gather=sg if sc_real else None)
            self._tile_emit(node, co, dst, residual=skip, name=name, gather=mg if main_real else None)
        self.env[id(node.outs[0])] = Full([(dst, 0)])
        return True

    # ---- pointwise algebra
    def _affine(self, node: Node, a, b, is_mul: bool):
        x, c = (a, b) if isinstance(a, LazyTensor) else (b, a)
        if isinstance(c, LazyTensor):
            return None
        v = self.sym(x)
        if isinstance(v, ConvOut) and not v.on_tiles:
            v = self.as_full(x)
        if not isinstance(v, Full) or v.pad is not None:
            return None
        if isinstance(c, (int, float)):
            cv = torch.full((v.C,), float(c), dtype=torch.float32, device=self.dev)
            self._keepalive.append(cv)
        elif _is_const(c):
            try:
                cv = self._chan_vec(c, v)
            except TraceUnsupported:
                return None
        else:
            return None
        pre = v.pre.copy() if v.pre is not None else Pre()
        if pre.act:
            return None
        if is_mul:
            pre.scale = cv if pre.scale is None else self.derive(torch.mul, pre.scale, cv)
            pre.shift = None if pre.shift is None else self.derive(torch.mul, pre.shift, cv)
        else:
            pre.shift = cv if pre.shift is None else self.derive(torch.add, pre.shift, cv)
        return Full(list(v.segs), pre, None)

    def _h_mul(self, node: Node):
        a, b = node.args[0], node.args[1]
        out = node.outs[0]
        if len(node.args) == 2 and not node.kwargs and self._sep_affine(node, True):
            return True
        sa, sb = (self.sym(a) if isinstance(a, LazyTensor) else None), (self.sym(b) if isinstance(b, LazyTensor) else None)
        # x * sigmoid(x)
        for x, s_ in ((a, sb), (b, sa)):
            if isinstance(s_, Sig) and isinstance(x, LazyTensor) and s_.of is x:
                v = self.sym(x)
                if isinstance(v, ConvOut) and not v.on_tiles:
                    v = self.as_full(x)
                if isinstance(v, Full) and v.pad is None and not (v.pre and v.pre.act):
                    pre = v.pre.copy() if v.pre is not None else Pre()
                    pre.act = "swish"
                    self.env[id(out)] = Full(list(v.segs), pre)
                    return True
                if isinstance(v, GNVal) and v.act is None:
                    self.env[id(out)] = GNVal(v.src, v.groups, v.weight, v.bias, v.eps, "swish")
                    return True
                return False
        for x_lt, s_ in ((a, sb), (b, sa)):       # x * (1 + gamma)
            if (isinstance(s_, Spade) and s_.stage == 1 and isinstance(x_lt, LazyTensor) and x_lt.dim() == 4
                    and tuple(x_lt.shape) == tuple(s_.gamma.shape) == tuple(out.shape)):
                self.env[id(out)] = Spade(2, s_.gamma, x=x_lt)
                return True
        for x, c in ((sa, b), (sb, a)):
            if isinstance(x, Scores) and isinstance(c, (int, float)):
                self.env[id(out)] = Scores(x.q, x.k, x.scale * float(c))
                return True
            if isinstance(x, GScores) and not x.probs and isinstance(c, (int, float)):
                self.env[id(out)] = GScores(x.q, x.k, x.scale * float(c))
                return True
        r = self._affine(node, a, b, True)
        if r is None:
            return False
        self.env[id(out)] = r
        return True

    _h_rmul = _h_mul

    def _h_add(self, node: Node):
        a, b = node.args[0], node.args[1]
        if node.kwargs.get("alpha", 1) != 1 or len(node.args) > 2:
            return False
        if self._sep_affine(node, False):
            return True
        out = node.outs[0]
        for t_, c_ in ((a, b), (b, a)):        # 1 + gamma on a value that has no symbolic form (a slice of a tile stack), or on the
            # re-gathered tiles of a separable launch's destination (the sub-mobile SPADE's gamma)
            if (isinstance(t_, LazyTensor) and isinstance(c_, (int, float)) and float(c_) == 1.0 and t_.dim() == 4
                    and (self.sym(t_) is None or self._sep_stack(self.sym(t_)) or self._narrow_dense(self.sym(t_)))
                    and tuple(t_.shape) == tuple(out.shape) and t_.dtype.is_floating_point):
                self.env[id(out)] = Spade(1, t_)
                return True
        if isinstance(a, LazyTensor) and isinstance(b, LazyTensor):
            for m_lt, b_lt in ((a, b), (b, a)):       # x * (1 + gamma) + beta
                sm = self.sym(m_lt)
                if isinstance(sm, Spade) and sm.stage == 2 and b_lt.dim() == 4 and tuple(b_lt.shape) == tuple(out.shape) == tuple(m_lt.shape):
                    self.env[id(out)] = Spade(3, sm.gamma, x=sm.x, beta=b_lt)
                    return True
        if isinstance(a, LazyTensor) and isinstance(b, LazyTensor):
            for x, r in ((a, b), (b, a)):
                co = self.sym(x)
                if not (isinstance(co, ConvOut) and not co.on_tiles and self.n_uses(x) == 1):
                    continue
                ro = self.sym(r)
                src: Full = co.src
                shortcut = None
                res_buf = None
                if (isinstance(ro, ConvOut) and not ro.on_tiles and ro.k == 1 and self.n_uses(r) == 1 and co.k == 3 and co.stride == 1
                        and self.fuse_shortcut and self.tc5 and self.producer_preop and ro.src.plain and all(up == 0 for _, up in ro.src.segs) and len(ro.src.segs) <= 2
                        and ro.src.HW == src.HW and int(ro.weight.shape[0]) == int(co.weight.shape[0]) and int(ro.weight.shape[1]) % 64 == 0
                        and int(co.weight.shape[1]) % 64 == 0):
                    shortcut = ([b_ for b_, _ in ro.src.segs], ro.weight, ro.bias, None)     # dense block: the 1x1 shortcut on every tile
                else:
                    res_buf = self.plain_buf(r)
                    if res_buf is None:
                        continue
                    h, w = src.HW
                    oh, ow = (h // 2, w // 2) if co.stride == 2 else (h, w)
                    if tuple(res_buf.shape) != (src.B, int(co.weight.shape[0]), oh, ow):
                        continue
                dst = self.force_dense(co, residual=res_buf, shortcut=shortcut)
                self.env[id(out)] = Full([(dst, 0)])
                return True
            return False
        r = self._affine(node, a, b, False)
        if r is None:
            return False
        self.env[id(out)] = r
        return True

    _h_radd = _h_add

    def _h_leaky_relu(self, node: Node):
        a = self._bind(node, ("input", "negative_slope", "inplace"), {"negative_slope": 0.01, "inplace": False})
        v = self.sym(a["input"]) if isinstance(a["input"], LazyTensor) else None
        if isinstance(v, Spade) and v.stage == 3 and v.slope is None and not a["inplace"] and self.n_uses(a["input"]) == 1:
            self.env[id(node.outs[0])] = Spade(3, v.gamma, x=v.x, beta=v.beta, slope=float(a["negative_slope"]))
            return True
        return False

    def _h_relu(self, node: Node):
        """ReLU of a conv on tiles that nothing else reads (GauGAN's mlp_shared = conv -> nn.ReLU): the launch's epilogue."""
        a = self._bind(node, ("input", "inplace"), {"inplace": False})
        x = a["input"]
        co = self.sym(x) if isinstance(x, LazyTensor) else None
        if (getattr(self.ex, "narrow_conv_supported", None) is None or a["inplace"] or not isinstance(co, ConvOut) or not co.on_tiles
                or co.act is not None or self.n_uses(x) != 1):
            return False
        self.env[id(node.outs[0])] = ConvOut(co.node, co.src, co.weight, co.bias, co.k, co.stride, co.padding, cin_pad=co.cin_pad, act="relu")
        return True

    def _h_sigmoid(self, node: Node):
        x = node.args[0]
        if isinstance(self.sym(x), (Full, ConvOut, GNVal)):
            self.env[id(node.outs[0])] = Sig(x)
            return True
        return False

    def _h_silu(self, node: Node):
        x = node.args[0]
        v = self.sym(x)
        if isinstance(v, ConvOut) and not v.on_tiles:
            v = self.as_full(x)
        if isinstance(v, Full) and v.pad is None and not (v.pre and v.pre.act):
            pre = v.pre.copy() if v.pre is not None else Pre()
            pre.act = "swish"
            self.env[id(node.outs[0])] = Full(list(v.segs), pre)
            return True
        if isinstance(v, GNVal) and v.act is None:
            self.env[id(node.outs[0])] = GNVal(v.src, v.groups, v.weight, v.bias, v.eps, "swish")
            return True
        return False

    # ---- identities in inference / in the step's single compute dtype
    def _alias(self, node: Node, x) -> bool:
        if not isinstance(x, LazyTensor):
            return False
        v = self.sym(x)
        if isinstance(v, (Sig,)):
            return False
        out = node.outs[0]
        if v is None:
            self._alias_of[id(out)] = x
        else:
            self.env[id(out)] = v
        self.uses[id(out)] = self.uses.get(id(out), 0) + self.uses.get(id(x), 1) - 1
        return True

    def _h_dropout(self, node: Node):
        a = self._bind(node, ("input", "p", "training", "inplace"), {"p": 0.5, "training": True, "inplace": False})
        return (not a["training"] or a["p"] == 0) and not a["inplace"] and self._alias(node, a["input"])

    def _h_float(self, node: Node):        # GroupNorm32 of the SD code: `super().forward(x.float()).type(x.dtype)`
        x = node.args[0]
        return isinstance(x, LazyTensor) and x.dtype.is_floating_point and self._alias(node, x)

    _h_half = _h_float
    _h_contiguous = _h_float

    def _h_type(self, node: Node):
        a = self._bind(node, ("input", "dtype"), {"dtype": None})
        x = a["input"]
        return (isinstance(a["dtype"], torch.dtype) and a["dtype"].is_floating_point and isinstance(x, LazyTensor) and x.dtype.is_floating_point
                and self._alias(node, x))

    def _h_to(self, node: Node):
        if (len(node.args) == 2 and isinstance(node.args[1], torch.dtype) and node.args[1].is_floating_point and not node.kwargs
                and isinstance(node.args[0], LazyTensor) and node.args[0].dtype.is_floating_point):
            return self._alias(node, node.args[0])
        return False

    # ---- structural glue
    def _h_cat(self, node: Node):
        a = self._bind(node, ("tensors", "dim"), {"dim": 0})
        if a["dim"] != 1:
            return False
        segs: List[Tuple[Buf, int]] = []
        for t in a["tensors"]:
            if not isinstance(t, LazyTensor):
                return False
            f = self.as_full(t)
            if f is None or not f.plain:
                return False
            segs += f.segs
        if len({(b.shape[0], b.shape[2] << up, b.shape[3] << up) for b, up in segs}) != 1:
            return False
        self.env[id(node.outs[0])] = Full(segs)
        return True

    _h_concat = _h_cat

    def _h_interpolate(self, node: Node):
        a = self._bind(node, ("input", "size", "scale_factor", "mode"), {"size": None, "scale_factor": None, "mode": "nearest"})
        sf = a["scale_factor"]
        if a["mode"] != "nearest" or a["size"] is not None or sf is None or any(float(s) != 2.0 for s in (sf if isinstance(sf, (tuple, list)) else (sf,))):
            return False
        f = self.as_full(a["input"])
        if f is None or f.pad is not None or any(up for _, up in f.segs):
            return False
        self.env[id(node.outs[0])] = Full([(b, 1) for b, _ in f.segs], f.pre)
        return True

    def _h_pad(self, node: Node):
        a = self._bind(node, ("input", "pad", "mode", "value"), {"mode": "constant", "value": None})
        if a["mode"] != "constant" or a["value"] not in (None, 0, 0.0) or tuple(a["pad"]) != (0, 1, 0, 1):
            return False
        f = self.as_full(a["input"])
        if f is None or f.pad is not None:
            return False
        self.env[id(node.outs[0])] = Full(list(f.segs), f.pre, (0, 1, 0, 1))
        return True

    def _h_group_norm(self, node: Node):
        a = self._bind(node, ("input", "num_groups", "weight", "bias", "eps"), {"weight": None, "bias": None, "eps": 1e-5})
        buf = None
        f = self.as_full(a["input"])
        if f is not None:
            buf = f.single
        if buf is None or not (a["weight"] is None or _is_const(a["weight"])) or not (a["bias"] is None or _is_const(a["bias"])):
            return False
        self.derive(None, a["weight"], a["bias"])
        self.env[id(node.outs[0])] = GNVal(buf, int(a["num_groups"]), a["weight"], a["bias"], float(a["eps"]))
        return True

    # ---- attention core: split -> reshape/permute -> bmm -> *scale -> softmax -> permute -> bmm -> reshape
    def _h_split(self, node: Node):
        a = self._bind(node, ("tensor", "split_size_or_sections", "dim"), {"dim": 0})
        sz = a["split_size_or_sections"]
        if a["dim"] != 1 or not isinstance(sz, int):
            return False
        f = self.as_full(a["tensor"])
        buf = f.single if f is not None else None
        if buf is None or buf.shape[1] % sz:
            return False
        for i, o in enumerate(node.outs):
            self.env[id(o)] = ChanSlice(buf, i * sz, (i + 1) * sz)
        return True

    def _h_reshape(self, node: Node):
        x = node.args[0]
        shape = node.args[1:] if not isinstance(node.args[1], (tuple, list, torch.Size)) else tuple(node.args[1])
        shape = tuple(int(s) for s in shape)
        v = self.sym(x)
        out = node.outs[0]
        if isinstance(v, HeadsOut):
            if v.stage == 0 and shape == (v.b, v.h, v.n, v.d):
                self.env[id(out)] = HeadsOut(v.full, v.b, v.h, v.n, v.d, 1)
                return True
            if v.stage == 2 and shape == (v.b, v.n, v.h * v.d):
                self.env[id(out)] = RealT(v.full)
                return True
            return False
        if isinstance(v, ChanSlice):
            B, _, H, W = v.buf.shape
            if tuple(out.shape) == (B, v.c1 - v.c0, H * W):
                self.env[id(out)] = Tok(v, "bcn")
                return True
            return False
        if isinstance(v, AttnOut):
            B, _, H, W = v.v.buf.shape
            C = v.v.c1 - v.v.c0
            if tuple(out.shape) == (B, C, H, W) and self._emit_attention(out, v):
                return True
            return False
        return False

    _h_view = _h_reshape

    def _h_permute(self, node: Node):
        x = node.args[0]
        dims = node.args[1:] if not isinstance(node.args[1], (tuple, list)) else tuple(node.args[1])
        v = self.sym(x)
        if isinstance(v, HeadsOut):
            if v.stage == 1 and tuple(int(d) for d in dims) == (0, 2, 1, 3):
                self.env[id(node.outs[0])] = HeadsOut(v.full, v.b, v.h, v.n, v.d, 2)
                return True
            return False
        if tuple(dims) != (0, 2, 1):
            return False
        if isinstance(v, Tok):
            self.env[id(node.outs[0])] = Tok(v.sl, "bnc" if v.layout == "bcn" else "bcn")
            return True
        if isinstance(v, Probs):
            self.env[id(node.outs[0])] = Probs(v.s, not v.transposed)
            return True
        return False

    def _h_bmm(self, node: Node):
        if self._tile_attention(node):
            return True
        a, b = self.sym(node.args[0]), self.sym(node.args[1])
        if isinstance(a, Tok) and isinstance(b, Tok) and a.layout == "bnc" and b.layout == "bcn":
            self.env[id(node.outs[0])] = Scores(a.sl, b.sl)
            return True
        if isinstance(a, Tok) and a.layout == "bcn" and isinstance(b, Probs) and b.transposed:
            self.env[id(node.outs[0])] = AttnOut(b.s, a.sl)
            return True
        # generic core: bmm(q, k.permute(0, 2, 1)) [* scale] -> softmax(-1) -> bmm(., v)  ==  one fused attention call
        qa, kb = node.args[0], node.args[1]
        if (a is None and isinstance(kb, LazyTensor) and kb.node is not None and kb.node.name in ("permute", "transpose") and self.n_uses(kb) == 1
                and qa.dim() == 3 and kb.dim() == 3):
            pn = kb.node
            dims = tuple(pn.args[1:]) if not isinstance(pn.args[1], (tuple, list)) else tuple(pn.args[1])
            if (pn.name == "permute" and dims == (0, 2, 1)) or (pn.name == "transpose" and set(int(d) % 3 for d in dims) == {1, 2}):
                self.env[id(node.outs[0])] = GScores(qa, pn.args[0])
                return True
        if a is None and isinstance(qa, LazyTensor) and _is_const(kb) and qa.dim() == 3 and kb.dim() == 3:
            # cross-attention against CACHED keys (sige_attention.py:35-42): k^T is a constant computed in the dense pass
            self.env[id(node.outs[0])] = GScores(qa, kb.transpose(1, 2))
            return True
        if isinstance(a, GScores) and a.probs and self.n_uses(node.args[0]) == 1 and node.args[1].dim() == 3:
            return self._emit_sdpa(node, a, node.args[1])
        return False

    def _sole_consumer(self, lt: LazyTensor, name: Tuple[str, ...]) -> Optional[Node]:
        """The one node that reads `lt`, if it is one of `name`."""
        if self._consumers is None:
            self._consumers = {}

            def note(o, n):
                if isinstance(o, LazyTensor):
                    self._consumers.setdefault(id(o), n)
                return o

            for n in self.tape.nodes:
                lazy._tree_map(lambda o, n=n: note(o, n), n.args)
                lazy._tree_map(lambda o, n=n: note(o, n), n.kwargs)
        n = self._consumers.get(id(lt)) if self.n_uses(lt) == 1 else None
        return n if n is not None and n.name in name else None

    def _tile_attention(self, node: Node) -> bool:
        """SIGEAttnBlock's core in sparse mode (reference stable-diffusion/ldm/modules/diffusionmodules/model.py:180-252, the VAE's
        mid block): the queries are the q conv's tile stack as tokens (reshape -> permute -> reshape: tile-major, then pixel order),
        the keys and values the full k / v maps that k_scatter / v_scatter paste together:
            bmm(q, k.reshape(b, c, hw)) * c^-0.5 -> softmax(2) -> bmm(v.reshape(b, c, hw), . .permute(0, 2, 1))
            -> reshape(b, c, tiles, bs, bs) -> permute(0, 2, 1, 3, 4) -> reshape(-1, c, bs, bs) -> proj_out -> out_scatter.
        Recognised at the first bmm, with every later node of the chain checked on the tape; then ONE `sige_sparse_attention`
        launch reads the q stack (written by the q conv's launch over the fixed-capacity tile list) and the k / v buffers in place
        (token stride C) and writes the NHWC tile stack that proj_out reads — padding tiles' rows are computed and never scattered.
        A batch of E independent edits records every tile as a batch row of its own (b = tiles) against k[tile_images] /
        v[tile_images], its edit's maps; it lowers, when the executor takes per-edit lists with a tile stack on one side
        (`per_image_stacks_supported`), to the q conv over the slot's per-edit lists into an [E * cap] stack, one launch at B = E
        (queries cap * bs * bs tokens of each edit's stack rows, keys and values its maps) and proj_out from that stack.
        Anything else keeps the recorded calls."""
        qa, kb = node.args[0], node.args[1]
        if not (isinstance(qa, LazyTensor) and isinstance(kb, LazyTensor) and qa.dim() == 3 and kb.dim() == 3):
            return False
        # queries: reshape(b, tiles / b * bs * bs, c) <- permute(0, 1, 3, 2) <- reshape(b, tiles / b, c, bs * bs) <- 1x1 conv on the tiles
        q3 = qa
        p3 = q3.node.args[0] if q3.node is not None and q3.node.name in ("reshape", "view") else None
        r4 = p3.node.args[0] if isinstance(p3, LazyTensor) and p3.node is not None and p3.node.name == "permute" else None
        qc = r4.node.args[0] if isinstance(r4, LazyTensor) and r4.node is not None and r4.node.name in ("reshape", "view") else None
        co = self.sym(qc) if isinstance(qc, LazyTensor) else None
        if not (isinstance(co, ConvOut) and isinstance(co.src, Stack) and not isinstance(co.src, (ModStack, WinStack)) and co.k == 1
                and co.stride == 1 and co.act is None and co.cin_pad == 0 and all(self.n_uses(t) == 1 for t in (q3, p3, r4, qc))):
            return False
        g = co.src.gather
        timg = getattr(g, "tile_images", None)
        if timg is not None and not self.per_image_stacks:
            return False
        bs = int(g.block_size[0])
        nt, C = int(qc.shape[0]), int(qc.shape[1])
        b = 1 if timg is None else nt            # bmm batch rows: the one image, or every tile of a batch of edits
        per = nt // b
        if (tuple(g.block_size) != (bs, bs) or tuple(qc.shape[2:]) != (bs, bs) or tuple(r4.shape) != (b, per, C, bs * bs)
                or tuple(int(d) for d in p3.node.args[1:]) != (0, 1, 3, 2) or tuple(q3.shape) != (b, per * bs * bs, C)
                or int(g.active_indices.shape[0]) != nt or nt == 0):
            return False
        E = 1 if timg is None else int(g.num_edits)

        def full_tokens(t):          # reshape(b, c, h * w) of a plain single-buffer map of E images (a batch: indexed by tile_images)
            if not (t.node is not None and t.node.name in ("reshape", "view") and self.n_uses(t) == 1):
                return None
            m = t.node.args[0]
            if timg is not None:
                if not (isinstance(m, LazyTensor) and m.node is not None and m.node.name == "__getitem__" and self.n_uses(m) == 1
                        and len(m.node.args) == 2 and m.node.args[1] is timg and not m.node.kwargs):
                    return None
                m = m.node.args[0]
            f = self.sym(m)
            buf = f.single if isinstance(f, Full) else None
            if buf is None or tuple(buf.shape[:2]) != (E, C) or tuple(t.shape) != (b, C, buf.shape[2] * buf.shape[3]):
                return None
            return buf

        kbuf = full_tokens(kb)
        # the rest of the chain
        mul = self._sole_consumer(node.outs[0], ("mul",))
        scale = mul.args[1] if mul is not None and len(mul.args) == 2 and mul.args[0] is node.outs[0] and not mul.kwargs else None
        sm = self._sole_consumer(mul.outs[0], ("softmax",)) if isinstance(scale, (int, float)) else None
        if sm is None:
            return False
        a = self._bind(sm, ("input", "dim"), {"dim": None})
        pt = self._sole_consumer(sm.outs[0], ("permute",)) if a["dim"] in (2, -1) and a.get("dtype") is None else None
        bmm2 = self._sole_consumer(pt.outs[0], ("bmm",)) if pt is not None and tuple(int(d) for d in pt.args[1:]) == (0, 2, 1) else None
        vbuf = full_tokens(bmm2.args[0]) if bmm2 is not None and bmm2.args[1] is pt.outs[0] else None
        o5 = self._sole_consumer(bmm2.outs[0], ("reshape", "view")) if vbuf is not None else None
        o5p = self._sole_consumer(o5.outs[0], ("permute",)) if o5 is not None and tuple(o5.outs[0].shape) == (b, C, per, bs, bs) else None
        o4 = (self._sole_consumer(o5p.outs[0], ("reshape", "view"))
              if o5p is not None and tuple(int(d) for d in o5p.args[1:]) == (0, 2, 1, 3, 4) else None)
        if (o4 is None or tuple(o4.outs[0].shape) != (nt, C, bs, bs) or kbuf is None or tuple(vbuf.shape) != tuple(kbuf.shape)
                or not (float(scale) > 0 and self.ex.sparse_attention_supported(C))):
            return False
        # q: the conv's launch over the fixed-capacity list(s) writes a capacity-row NHWC stack (E * cap rows for a batch)
        segs, pre, hw, idx, block, off, stack_src, qimg = self.tile_conv_args(co)
        sl = self.slots.get(id(g.active_indices))
        if (stack_src is not None or sl is None or idx is not sl.buf or segs[0][0].shape[0] != E or sl.E != E
                or (qimg is None) != (timg is None)):
            return False
        rows = int(idx.shape[0])
        # (zeros: the rows of padding tiles, which the q conv never writes, hold finite values for the attention to compute on)
        q_st = torch.empty((rows, C, bs, bs), dtype=self.dtype, device=self.dev, memory_format=torch.channels_last).zero_()
        self.emit_conv("n%d.q_stack" % co.node.index, segs, pre, hw, idx, block, co.weight, co.bias, co.stride, off, None, dst_stack=q_st,
                       tile_img=qimg)
        o_st = torch.empty_like(q_st)

        def tokens(t):               # [E, 1, tokens, C] view of an NHWC map or stack of E images (a stack: its rows in edit order)
            return t.permute(0, 2, 3, 1).reshape(E, -1, C).unsqueeze(1)

        for buf in (kbuf, vbuf):
            buf.readers.append(None)
        self.steps.append(("sparse_attention", self.ex.prepare_sparse_attention(tokens(q_st), tokens(kbuf.raw), tokens(vbuf.raw), float(scale),
                                                                                 tokens(o_st))))
        self.sparse_attention_calls += 1
        self.env[id(o4.outs[0])] = RealStack(o_st, slot=sl)
        return True

    def _emit_sdpa(self, node: Node, g: GScores, v: LazyTensor) -> bool:
        def rt(t):
            if isinstance(t, LazyTensor):
                return self.runtime_tensor(t)
            dev, dt = self.dev, self.dtype
            c = self.derive(lambda u: u.detach().to(dev).to(dt).contiguous(), t)       # cached keys / values: constants of this step
            self._keepalive.append(c)
            return c

        o = node.outs[0]
        scale = float(g.scale)
        D = int(o.shape[2])
        ours = scale > 0 and self.ex.sparse_attention_supported(D)

        def operand(t):
            """The [(b h), n, d] operand — or, when it is einops' copy of a "b n (h d)" tensor (reshape -> permute -> reshape,
            attention.py:81) that nothing else reads, the strided [b, h, n, d] VIEW of that tensor: the kernel takes explicit
            (batch, head, token) strides, so the three rearrange copies per attention call disappear."""
            if (ours and isinstance(t, LazyTensor) and t.node is not None and t.node.name in ("reshape", "view") and self.sym(t) is None
                    and self.n_uses(t) == 1):
                src = t.node.args[0]
                if isinstance(src, LazyTensor) and src.dim() == 4 and tuple(t.shape) == (src.shape[0] * src.shape[1], src.shape[2], src.shape[3]):
                    r = self.runtime_tensor(src)
                    if r.dtype == self.dtype and r.stride(3) == 1 and all(int(r.stride(i)) % 8 == 0 for i in range(3)) and r.data_ptr() % 16 == 0:
                        return r
            return rt(t)

        q, k, vv = operand(g.q), operand(g.k), operand(v)
        if not (q.dtype == k.dtype == vv.dtype):
            return False
        out = torch.empty(tuple(o.shape), dtype=q.dtype, device=self.dev)
        if ours:
            heads = {int(t.shape[1]) for t in (q, k, vv) if t.dim() == 4}
            ho = None
            if len(heads) == 1:       # mixed 3-D / 4-D operands: present every one as [b, h, n, d]
                hh = heads.pop()
                q, k, vv = (t if t.dim() == 4 else t.view(t.shape[0] // hh, hh, t.shape[1], t.shape[2]) for t in (q, k, vv))
                # ... and write the result in the "b n (h d)" layout its consumer (to_out's Linear) reads: see HeadsOut
                ho = HeadsOut(torch.empty((out.shape[0] // hh, out.shape[1], hh * D), dtype=out.dtype, device=self.dev), out.shape[0] // hh, hh,
                              int(out.shape[1]), D)
                out_arg = ho.bhnd
            else:
                out_arg = out
            ok = (len(heads) == 0 and q.dim() == k.dim() == vv.dim() and k.shape == vv.shape and k.shape[:-2] == q.shape[:-2] and k.shape[-1] == D
                  and all(t.stride(-1) == 1 and all(int(st) % 8 == 0 for st in t.stride()[:-1]) for t in (q, k, vv)))
            if ok:
                # this repo's flash-style kernel: sparse queries against all keys / the cached text keys, one launch
                self.steps.append(("sparse_attention", self.ex.prepare_sparse_attention(q, k, vv, scale, out_arg)))
                self.sparse_attention_calls += 1
                self.env[id(o)] = ho if ho is not None else RealT(out)
                return True
        if not (q.dim() == k.dim() == vv.dim() == 3):
            return False            # (strided operands the kernel refused: the recorded bmm / softmax / bmm run as they are)

        q4, k4, v4 = q.unsqueeze(0), k.unsqueeze(0), vv.unsqueeze(0)      # 4-D: with 3-D operands torch falls to its fp32 math path (40x slower)

        def run(_stream):
            out.copy_(F.scaled_dot_product_attention(q4, k4, v4, scale=scale)[0])

        self.steps.append(("eager", run))
        self.eager_nodes.append("sdpa")
        self.env[id(o)] = RealT(out)
        return True

    def _h_softmax(self, node: Node):
        a = self._bind(node, ("input", "dim"), {"dim": None})
        v = self.sym(a["input"])
        if isinstance(v, Scores) and a["dim"] in (2, -1) and a.get("dtype") is None:
            self.env[id(node.outs[0])] = Probs(v)
            return True
        if isinstance(v, GScores) and not v.probs and a["dim"] in (2, -1) and a.get("dtype") is None and self.n_uses(a["input"]) == 1:
            self.env[id(node.outs[0])] = GScores(v.q, v.k, v.scale, probs=True)
            return True
        return False

    def _emit_attention(self, out: LazyTensor, v: AttnOut) -> bool:
        q, k, vv = v.s.q, v.s.k, v.v
        buf = q.buf
        B, C3, H, W = buf.shape
        C = q.c1 - q.c0
        if not self.fused_attention:
            return False
        cluster_ok = (k.buf is buf and vv.buf is buf and (q.c0, k.c0, vv.c0) == (0, C, 2 * C) and C3 == 3 * C
                      and self.ex.attention_supported(H * W, C) and len(buf.producers) == 1 and isinstance(buf.producers[0], FusedConv))
        if not cluster_ok:
            return self._emit_attention_generic(out, v)
        prod: FusedConv = buf.producers[0]
        if prod.spec.out_row_scale is not None or prod.spec.aux or any(r is None for r in buf.readers):
            return False
        # q <- q * scale: folded into the q rows of the producing 1x1 conv (the kernel takes pre-scaled q)
        if v.s.scale != 1.0:
            prod.spec.out_row_scale = (C, float(v.s.scale))
        buf.readers.append(None)
        dst = self.fresh(B, C, H, W)
        tok = buf.raw.permute(0, 2, 3, 1).reshape(B, H * W, 3 * C)
        o_tok = dst.raw.permute(0, 2, 3, 1).reshape(B, H * W, C)
        self.steps.append(("attention", self.ex.prepare_attention(tok, o_tok, self.pdl)))
        self.env[id(out)] = Full([(dst, 0)])
        return True

    def _emit_attention_generic(self, out: LazyTensor, v: AttnOut) -> bool:
        """Single-head attention core outside the cluster kernel's range (token count / channel count): the flash-style
        `sige_sparse_attention` on the channel slices of the NHWC buffers, addressed in place — q, k, v = [B, 1, H*W, C] views with
        the token stride of their buffer, the result written as NHWC tokens of a fresh buffer."""
        q, k, vv = v.s.q, v.s.k, v.v
        C = q.c1 - q.c0
        B, _, H, W = q.buf.shape
        if not (k.c1 - k.c0 == C and vv.c1 - vv.c0 == C and k.buf.shape[0] == B and vv.buf.shape[0] == B
                and tuple(k.buf.shape[2:]) == tuple(vv.buf.shape[2:]) and v.s.scale > 0 and self.ex.sparse_attention_supported(C)
                and all(sl.c0 % 8 == 0 and sl.buf.shape[1] % 8 == 0 for sl in (q, k, vv))):
            return False

        def tokens(sl):
            sl.buf.readers.append(None)
            b, ct, h, w = sl.buf.shape
            return sl.buf.raw.permute(0, 2, 3, 1).reshape(b, h * w, ct)[:, :, sl.c0:sl.c1].unsqueeze(1)        # [B, 1, N, C], strided view

        dst = self.fresh(B, C, H, W)
        o_tok = dst.raw.permute(0, 2, 3, 1).reshape(B, H * W, C).unsqueeze(1)
        self.steps.append(("sparse_attention", self.ex.prepare_sparse_attention(tokens(q), tokens(k), tokens(vv), float(v.s.scale), o_tok)))
        self.sparse_attention_calls += 1
        self.env[id(out)] = Full([(dst, 0)])
        return True

    # ------------------------------------------------------------------ outputs / post-pass
    def _output(self, lt: LazyTensor) -> torch.Tensor:
        return self.runtime_tensor(lt)

    def _post(self) -> None:
        # the stem only has to exist where it is read: if every reader gathers it through one index set, restrict it
        for rec in self.conv_ins:
            rd = rec.out.readers
            def same_img(a, b):
                return (a is None and b is None) or (a is not None and b is not None and torch.equal(a, b))

            if (self.sparse_stem and rd and all(r is not None for r in rd)
                    and all(up_ == 0 and blk_ <= 6 and i_ is not None and torch.equal(i_, rd[0][0]) and same_img(ti_, rd[0][3]) for (i_, blk_, up_, ti_) in rd)):
                rec.tiles, rec.tile_size, rec.tile_img = rd[0][0].contiguous(), max(r[1] for r in rd), rd[0][3]
                for t_ in ([rec.out._raw] if rec.out.has_raw else []) + [v[0] for v in rec.out.views.values()]:
                    t_.zero_()          # never read outside the tiles; defined contents all the same
        for fc in self.fused:
            s = fc.spec
            if s.dst is not None and not s.aux:
                _ = s.dst.raw             # a value nobody transformed: keep the raw destination
        self._early_masks()
        for fc in self.fused:
            self.ex.prepare_conv(fc)
        takes_wgmma = getattr(self.ex, "takes_wgmma", None)
        if takes_wgmma is not None:
            for fc in self.fused:
                prev = self._conv_at.get(fc.pos - 1)
                if fc.spec.early and not takes_wgmma(prev):          # (the mma.sync kernel releases before it waits)
                    fc.spec.early, prev.spec.early_release = 0, False
                    fc.desc.flags &= ~(7 << 4)
                    prev.desc.flags &= ~self.ex.ops._cabi.CONV_EARLY_RELEASE
        for prep in self._pending_prepare:
            prep()
        self._build_sparse_update()

    def _early_masks(self) -> None:
        """The early source groups of every launch (SIGE_CONV_EARLY_SRC0 / _SRC1 / _SHORTCUT, kept as bits 0..2 in ConvSpec.early):
        the source groups that the immediately preceding step does not write.  Only when that step is a tile conv meant for the wgmma kernel
        (it waits for its own predecessor before it releases this launch; the attention, glue and mma.sync kernels release first)
        and both launches use programmatic dependent launch.  The predecessor of a launch with a mask releases it as soon as its
        own dependency has resolved (SIGE_CONV_EARLY_RELEASE).  Masks depend on buffers and launch order only, not on tiles, so
        `rebind` keeps them; the sparse_update epilogue leaves them 0."""
        self._conv_at = {fc.pos: fc for fc in self.fused}

        def key(t):
            return t.untyped_storage().data_ptr()

        for fc in self.fused:
            s = fc.spec
            prev = self._conv_at.get(fc.pos - 1)
            if not (s.pdl and s.tc5 and prev is not None and prev.spec.pdl and prev.spec.tc5):
                continue
            p = prev.spec
            written = {key(v) for (v, _, _, _) in p.aux}
            if p.dst_stack is not None:
                written.add(key(p.dst_stack))
            if p.dst is not None and p.dst.has_raw:
                written.add(key(p.dst.raw))
            pre = [t for t in (s.scale, s.shift) if t is not None] + (list(s.modulation[:2]) if s.modulation is not None else [])
            groups = [[t] + pre for t, _ in s.srcs[:2]]
            if s.shortcut is not None:
                groups += [[]] * (2 - len(groups)) + [list(s.shortcut[0])]
            mask = 0
            for g, reads in enumerate(groups):
                if reads and not any(key(t) in written for t in reads):
                    mask |= 1 << g
            if mask:
                s.early, p.early_release = mask, True

    # ------------------------------------------------------------------ sparse_update epilogue
    def _sparse_update_refusal(self) -> Optional[str]:
        """Why this step cannot write its results back into the module caches (None: it can)."""
        ok = getattr(self.ex, "writeback_supported", None)
        if ok is None or not ok():
            return "the executor has no tile write-back"
        if any(b.shape[0] != b.cached_init.shape[0] for b in self.cached_bufs) or any(f.spec.tile_img is not None for f in self.fused):
            return "a batch of edits (a cache holds one image)"
        eager = [n for n in self.eager_nodes if n.startswith("sige.scatter")]
        if eager:
            return "eager operator-module scatters in the step (%s)" % ", ".join(eager)
        for (buf, slot, _off, _st, _ro) in self.cache_writers:
            if slot is None:
                return "a cached %s buffer is written through a tile list without a fixed-capacity buffer" % (buf.shape,)
        for buf in self.cached_bufs:
            c = buf.cached_init
            if c.dtype not in (torch.float32, self.dtype):
                return "a %s cache cannot take %s tiles exactly" % (c.dtype, self.dtype)
            if c.dim() != 4 or tuple(c.shape) != buf.shape or c.shape[1] % 8 or not (c.is_contiguous() or c.is_contiguous(memory_format=torch.channels_last)):
                return "a cache of shape %s is not a dense [B, C, H, W] tensor with C a multiple of 8" % (tuple(c.shape),)
        return None

    def _relaunch(self, spec: ConvSpec, name: str) -> FusedConv:
        spec.name, spec.pdl = name, False          # (the epilogue's first launch follows another graph)
        spec.early, spec.early_release = 0, False
        fc = FusedConv(spec)
        self.ex.prepare_conv(fc)
        self.epilogue_fused.append(fc)
        self.epilogue.append(("conv", fc.launch))
        return fc

    def _build_sparse_update(self) -> None:
        """The program `FusedStep.sparse_update()` runs after the main program: (1) every shortcut fused into a conv2 launch as its own
        1x1 tile conv into `skip` (its tiles of the reference's `original_residuals`), (2) every launch whose cached destination
        only exists as producer-written views again, writing the raw values, (3) one `sige_tile_writeback` of the output tiles of
        every cached buffer into its module cache.  The main program is not touched: its launches were prepared before this runs."""
        self.sparse_update_reason = self._sparse_update_refusal()
        if self.sparse_update_reason is not None:
            return
        plan: List[Tuple[ConvSpec, str, int]] = []
        for (name, sc_bufs, w, b, skip, slot, soff, conv2) in self.shortcut_relaunches:
            s = ConvSpec()
            s.srcs = [(sb.raw, 0) for sb in sc_bufs]
            s.B, s.H, s.W = skip.shape[0], sc_bufs[0].shape[2], sc_bufs[0].shape[3]
            s.idx, s.N, s.slot, s.block, s.k, s.stride, s.off = slot.buf, slot.cap, slot, 4, 1, 1, soff
            s.weight, s.bias, s.weight_key = w.detach().float(), None if b is None else b.detach().float(), (w, "w")
            s.tc5, s.ksplit, s.dst = self.tc5, self.ksplit, skip
            plan.append((s, name, conv2.pos))
        raw_less = {id(b) for b in self.cached_bufs if not b.has_raw}
        for fc in self.fused:
            if fc.spec.dst is not None and id(fc.spec.dst) in raw_less:
                s = copy.copy(fc.spec)
                s.aux = []                # the launch wrote only transformed views of its destination: write the raw values
                plan.append((s, fc.name + ".raw", fc.pos))
        # the relaunched launches read their sources after the whole main program: nothing may rewrite them after the launch
        # they repeat, nor in the epilogue
        writes: List[Tuple[int, int]] = []       # (storage, position)
        for fc in self.fused:
            s = fc.spec
            outs = [v for (v, _, _, _) in s.aux] + ([s.dst_stack] if s.dst_stack is not None else []) + ([s.dst.raw] if s.dst is not None and s.dst.has_raw else [])
            writes += [(t.untyped_storage().data_ptr(), fc.pos) for t in outs]
        for rec in self.separable:
            writes += [(br[3].raw.untyped_storage().data_ptr(), rec.slot) for br in rec.branches]
        writes += [(s.dst.raw.untyped_storage().data_ptr(), len(self.steps)) for (s, _, _) in plan]

        def sources(s: ConvSpec) -> List[torch.Tensor]:
            out = [t for t, _ in s.srcs] + ([s.residual] if s.residual is not None else [])
            if s.shortcut is not None:
                out += list(s.shortcut[0])
            if s.modulation is not None:
                out += [s.modulation[0], s.modulation[1]]
            return out

        for (s, name, pos) in plan:
            for t in sources(s):
                key = t.untyped_storage().data_ptr()
                if any(k == key and p > pos for (k, p) in writes):
                    self.sparse_update_reason = "%s: a source is rewritten after the launch the epilogue repeats" % name
                    return
        for (s, name, _pos) in plan:
            self._relaunch(s, name)
        entries = []
        for (buf, slot, off, stride, ro) in self.cache_writers:
            entries.append((buf.raw, buf.cached_init, slot.buf, off, stride, ro))
        if entries:
            self.epilogue.append(("writeback", self.ex.prepare_writeback(entries)))


# =====================================================================================================================
# public object
# =====================================================================================================================
class FusedStep:
    """Traced + fused + graph-captured sparse forward of ``model`` for inputs shaped like ``args``.

    ``step(*args)`` copies the tensor arguments into the static inputs, replays the program and returns the static
    output tensor(s) (valid until the next call).  ``replay()`` skips the input copy."""

    def __init__(self, model: nn.Module, *args, use_graph: bool = True, executor=None, dtype: Optional[torch.dtype] = None,
                 call_kwargs: Optional[Dict[str, Any]] = None, **options):
        """``dtype``: arithmetic / storage type of the fused step (fp16 or bf16).  Defaults to the input's dtype; an fp32
        model (the reference's own precision: its dense pass then stays exactly the reference's) runs its sparse steps on
        the tensor cores with ``dtype=torch.float16`` — activations, caches and weights are converted once at build."""
        if getattr(model, "mode", "sparse") != "sparse":
            raise RuntimeError("FusedStep: run the dense pass, set_masks() and set_mode('sparse') first")
        call_kwargs = dict(call_kwargs or {})         # keyword arguments of the model call (SD: model(x, t, context=c))
        self._kw_names = sorted(call_kwargs)
        kw_values = [call_kwargs[k] for k in self._kw_names]
        self._n_pos = len(args)
        args = tuple(args) + tuple(kw_values)
        tensors = [a for a in args if isinstance(a, torch.Tensor)]
        if not tensors:
            raise TraceUnsupported("no tensor argument")
        x = tensors[0]
        self.dev, self.dtype = x.device, (dtype or x.dtype)
        if executor is None:
            if not x.is_cuda or self.dtype not in (torch.float16, torch.bfloat16):
                raise TraceUnsupported("the fused step needs CUDA tensors and an fp16/bf16 compute dtype (tensor-core path); got %s %s" % (x.device, self.dtype))
            executor = CudaExecutor(x.device, self.dtype)
        self.ex = executor
        self.model = model
        self.static_inputs: List[torch.Tensor] = []
        self._arg_dtypes = [t.dtype for t in tensors]
        for t in tensors:
            dt = self.dtype if (t.dtype.is_floating_point and t.dim() == 4) else t.dtype
            if t.dim() == 4:
                s = torch.empty(t.shape, dtype=dt, device=t.device, memory_format=torch.channels_last)
            else:
                s = torch.empty_like(t)
            s.copy_(t)
            self.static_inputs.append(s)
        self._arg_template = [a if not isinstance(a, torch.Tensor) else None for a in args]
        names = {id(m): n for n, m in model.named_modules()}
        with torch.no_grad(), lazy.tracing() as tape:
            it = iter(lazy.make_input(s, tape, dtype=dt) for s, dt in zip(self.static_inputs, self._arg_dtypes))
            largs = [next(it) if a is None else a for a in self._arg_template]
            outs = nn.Module.__call__(model, *largs[:self._n_pos], **dict(zip(self._kw_names, largs[self._n_pos:])))
        self.tape = tape
        with torch.no_grad():
            self.low = Lowering(tape, outs, self.static_inputs, executor, self.dtype, self.dev, module_names=names, **options)
        self.steps = self.low.steps
        self.fused = self.low.fused
        self.outputs = self.low.outputs
        self.output = self.outputs if isinstance(self.outputs, torch.Tensor) else None
        self.eager_nodes = self.low.eager_nodes
        # sparse_update (the reference's apply step): whether this step can write its results back into the module caches
        self.sparse_update_reason: Optional[str] = self.low.sparse_update_reason
        self.sparse_update_supported = self.sparse_update_reason is None
        # refresh (a new dense pass taken in place): why this step cannot (None: it can), and where the model keeps the current value
        # of every tensor the program took from outside the tape
        self.refresh_reason: Optional[str] = None
        self.locations: Dict[int, Tuple] = {}
        self._locate()
        self.graph = None
        self.epilogue_graph = None
        self.launches_per_step = 0
        self._finalize(use_graph)

    # ------------------------------------------------------------------ execution
    def run_eager(self):
        self._run(self.steps)
        return self.outputs

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.dev).cuda_stream if self.dev.type == "cuda" else 0

    def _run(self, steps) -> None:
        stream = self._stream()
        with torch.no_grad():
            for _kind, fn in steps:
                fn(stream)

    def sparse_update(self) -> None:
        """After a call: write its results into the module caches, as the reference's modules do with ``sparse_update=True``
        (sige/nn/scatter.py:59-60,114-129, scatter_gather.py:65-77) — only the output tiles of the current tile lists.  Runs the
        epilogue program the lowering built (`Lowering._build_sparse_update`); the first call runs it eagerly and captures it in
        a second CUDA graph, later calls replay that graph.  The main program and its graph are not involved."""
        if not self.sparse_update_supported:
            raise RuntimeError("this fused step cannot write back into the module caches: %s" % self.sparse_update_reason)
        if self.epilogue_graph is not None:
            self.epilogue_graph.replay()
            return
        self._run(self.low.epilogue)
        if self.graph is not None:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._run(self.low.epilogue)
            self.epilogue_graph = g

    def _finalize(self, use_graph: bool) -> None:
        if self.dev.type != "cuda":
            self.run_eager()
            return
        side = torch.cuda.Stream(device=self.dev)
        side.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(side):
            for _ in range(3):
                self.run_eager()
        torch.cuda.current_stream(self.dev).wait_stream(side)
        torch.cuda.synchronize(self.dev)
        before = self.ex.launch_counter()
        if use_graph:
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self.run_eager()
        else:
            self.run_eager()
        self.launches_per_step = self.ex.launch_counter() - before

    def replay(self):
        if self.graph is not None:
            self.graph.replay()
            return self.outputs
        return self.run_eager()

    def rebind(self) -> bool:
        """Install the model's CURRENT tile lists (after a new ``set_masks``) into this compiled step without re-tracing or
        re-capturing: possible when every list fits the capacity it was built with and nothing outside the fused launches
        holds a tile list (no eager operator-module fallbacks).  A batch of edits takes a new batch of the same size whose every
        per-edit list fits.  Index buffers and shortcut flags are rewritten in place and every cached buffer goes back to the
        original activations; the CUDA graph stays valid."""
        low = self.low
        if any(n.startswith(("sige.", "gather(")) for n in self.eager_nodes) or not low.slots:
            return False
        if not all(sl.fits() for sl in low.slots.values()):
            return False
        with torch.no_grad():
            for sl in low.slots.values():
                sl.reload()
            for (fbuf, ms, off, ss, soff) in low.flag_recipes:
                flags, stray = _shortcut_flags(ms, off, ss, soff)
                if bool(stray):
                    return False            # the shortcut's tiles left the main conv's grid: a different program
                fbuf.copy_(flags)
            low.load_caches(self._stream())
        return True

    def rebind_device(self, masks) -> bool:
        """`rebind` without a host synchronisation (SURVEY section 8f-4): the mask reductions (`sige_reduce_mask`, or one
        `sige_reduce_mask_batched` per geometry for the [E, H, W] masks of a batch of edits) run on the device and their results
        go straight into the fixed-capacity tile lists the captured launches read — counts and all stay in HBM, nothing is copied
        back, so the call only ENQUEUES work (a handful of small kernels) and the next replay sees the new edit.
        Whether every list fit its capacity is recorded in `self.async_status` (device int32: bit 0 = a list overflowed and was
        truncated, bit 1 = a fused shortcut's tiles left the main conv's grid); `async_ok()` reads it (that one does synchronise).
        Returns False — nothing changed — when this step cannot be re-bound in place at all (a batch of another size included)."""
        from . import ops

        low = self.low
        if any(n.startswith(("sige.", "gather(")) for n in self.eager_nodes) or not low.slots:
            return False
        for sl in low.slots.values():
            g = sl.gather
            m = masks.get(tuple(g.input_res)) if g.input_res is not None else None
            want = 2 if sl.tile_img is None else 3
            if m is None or not m.is_cuda or m.dim() != want or (want == 3 and int(m.shape[0]) != sl.E):
                return False
        with torch.no_grad():
            if getattr(self, "async_status", None) is None:
                self.async_status = torch.zeros((1,), dtype=torch.int32, device=self.dev)
            self.async_status.zero_()
            memo: Dict = {}
            for sl in low.slots.values():
                g = sl.gather
                res = tuple(g.input_res)
                key = (res, tuple(g.block_size), tuple(g.block_stride), tuple(g.offset))
                m = masks[res]
                if sl.tile_img is not None:
                    key = key + (sl.cap,)
                    if key in memo:
                        sl.buf.copy_(memo[key].buf)
                        sl.n = memo[key].n
                    else:
                        sl.install_batched_device((m > 0.5) if m.is_floating_point() else (m != 0), self.async_status)
                        memo[key] = sl
                    continue
                if key not in memo:
                    m = (m > 0.5) if m.is_floating_point() else (m != 0)          # same binarisation as masks.reduce_mask
                    memo[key] = ops.reduce_mask_cuda_launch(m, g.block_size, g.block_stride, g.offset)
                sl.install_device(*memo[key], self.async_status)
            for (fbuf, ms, off, ss, soff) in low.flag_recipes:
                flags, stray = _shortcut_flags(ms, off, ss, soff)
                fbuf.copy_(flags)
                self.async_status.bitwise_or_(stray * 2)
            low.load_caches(self._stream())
        return True

    def _locate(self) -> None:
        """Find, for every tensor the program took from outside the tape (module caches, dense-pass statistics, the sources of
        `Lowering.derive`), the module attribute that holds it: a tensor, or a dict / list of tensors one level deep
        (``scale1s[cache_id]``, ``original_outputs[cache_id]``), matched by storage.  Parameters and registered buffers need no
        location.  Sets `refresh_reason` when the step cannot be refreshed."""
        low, model = self.low, self.model
        if low.eager_state:
            self.refresh_reason = "eager operator modules read their caches inside the captured graph (%s)" % ", ".join(low.eager_state)
            return
        fixed = {t.untyped_storage().data_ptr() for t in list(model.parameters()) + list(model.buffers())}
        made = {id(t) for d in low.derived for t in (d.out if isinstance(d.out, tuple) else (d.out,)) if isinstance(t, torch.Tensor)}
        holders: Dict[int, List] = {}
        for name, m in model.named_modules():
            for attr, val in vars(m).items():
                if attr in ("_parameters", "_buffers", "_modules"):
                    continue
                items = ([(None, val)] if isinstance(val, torch.Tensor) else list(val.items()) if isinstance(val, dict)
                         else list(enumerate(val)) if isinstance(val, list) else [])
                for key, t in items:
                    if isinstance(t, torch.Tensor) and not isinstance(t, LazyTensor):
                        holders.setdefault(t.untyped_storage().data_ptr(), []).append((name, attr, key, t))

        def locate(t: torch.Tensor) -> Optional[str]:
            if id(t) in self.locations:
                return None
            lo, hi = t.storage_offset(), t.storage_offset() + sum((n - 1) * st for n, st in zip(t.shape, t.stride()))
            for (name, attr, key, base) in holders.get(t.untyped_storage().data_ptr(), []):
                blo = base.storage_offset()
                bhi = blo + sum((n - 1) * st for n, st in zip(base.shape, base.stride()))
                if base.dtype == t.dtype and blo <= lo and hi <= bhi:
                    self.locations[id(t)] = (name, attr, key, base.dtype, base.device, tuple(base.shape), tuple(base.stride()),
                                             lo - blo, tuple(t.shape), tuple(t.stride()))
                    return None
            return "a %s tensor the forward read is held by no module" % (tuple(t.shape),)

        reasons = [locate(b.cached_init) for b in low.cached_bufs]
        for d in low.derived:
            for t in d.srcs:
                if not isinstance(t, torch.Tensor) or id(t) in made or t.untyped_storage().data_ptr() in fixed:
                    continue
                reasons.append("a %s tensor taken from outside the tape is read as it is" % (tuple(t.shape),) if d.fn is None else locate(t))
        if any(f.spec.refold for f in low.fused) and getattr(self.ex, "repack_conv", None) is None:
            reasons.append("the executor cannot re-pack folded weights")
        self.refresh_reason = next((r for r in reasons if r is not None), None)
        if self.refresh_reason is not None:
            self.locations = {}
        low._vecs.clear()         # (the memo of the lowering held the sources)

    def _resolve(self) -> Tuple[Optional[Dict[int, torch.Tensor]], Optional[str]]:
        """(the model's current tensor at every location, None) when each has the recorded dtype, device, shape, stride and view
        geometry; else (None, why not)."""
        mods = dict(self.model.named_modules())
        new: Dict[int, torch.Tensor] = {}
        for tid, (name, attr, key, dt, dev, shape, stride, rel, vshape, vstride) in self.locations.items():
            m = mods.get(name)
            c = None if m is None else vars(m).get(attr)
            where = "%s.%s%s" % (name, attr, "" if key is None else "[%r]" % (key,))
            try:
                base = c if key is None else c[key]
            except (KeyError, IndexError, TypeError):
                return None, "%s is gone" % where
            if not isinstance(base, torch.Tensor) or isinstance(base, LazyTensor):
                return None, "%s is no longer a tensor" % where
            if base.dtype != dt or base.device != dev or tuple(base.shape) != shape or tuple(base.stride()) != stride:
                return None, "%s is now a %s %s tensor of shape %s, stride %s (the step was built for %s %s, %s, %s)" % (
                    where, base.dtype, base.device, tuple(base.shape), tuple(base.stride()), dt, dev, shape, stride)
            new[tid] = base.as_strided(vshape, vstride, base.storage_offset() + rel)
        return new, None

    def refresh(self, load: bool = True) -> bool:
        """Take the model's CURRENT caches and dense-pass statistics (after a new ``full``-mode pass on an original image) into
        this compiled step in place, without re-tracing or re-capturing: every recorded derivation is recomputed into the
        storage the launches read (per-channel vectors, weights with statistics folded in, re-packed), every cached buffer is
        reloaded from its new cache (one `sige_cache_load`) and the write-back targets the new caches.  Only enqueued work: no
        host synchronisation.  The CUDA graph, descriptors and split-K plans stay as captured.  Returns False — nothing
        changed — when `refresh_reason` is set, when a location no longer holds a tensor of the recorded geometry, or when the
        step writes back and the new caches cannot take its tiles; the last two set `refresh_reason` too (the caller recompiles).
        ``load`` False: the cached buffers are left for the caller to reload (`rebind` follows, which reloads them)."""
        if self.refresh_reason is not None:
            return False
        new, why = self._resolve()
        if new is None:
            self.refresh_reason = why
            return False
        low = self.low
        old = [b.cached_init for b in low.cached_bufs]
        for b in low.cached_bufs:
            b.cached_init = new[id(b.cached_init)]
        refusal = low._sparse_update_refusal() if self.sparse_update_supported else None
        if refusal is not None:
            for b, c in zip(low.cached_bufs, old):
                b.cached_init = c
            self.refresh_reason = "the new caches cannot take the write-back: %s" % refusal
            return False
        with torch.no_grad():
            live = set(new)
            for d in low.derived:
                if d.fn is None or not any(isinstance(t, torch.Tensor) and id(t) in live for t in d.srcs):
                    continue
                srcs = tuple(new.get(id(t), t) if isinstance(t, torch.Tensor) else t for t in d.srcs)
                val = d.fn(*srcs)
                outs, vals = (d.out, val) if isinstance(d.out, tuple) else ((d.out,), (val,))
                for o, v in zip(outs, vals):
                    if o is not None:
                        o.copy_(v)
                        live.add(id(o))
                d.srcs = srcs
            for fc in low.fused + low.epilogue_fused:
                if fc.spec.refold and id(fc.spec.weight) in live:
                    self.ex.repack_conv(fc)
            low.loader = None
            if load:
                low.load_caches(self._stream())
            if self.sparse_update_supported:
                low.epilogue = [e for e in low.epilogue if e[0] != "writeback"]
                entries = [(buf.raw, buf.cached_init, slot.buf, off, stride, ro) for (buf, slot, off, stride, ro) in low.cache_writers]
                if entries:
                    low.epilogue.append(("writeback", self.ex.prepare_writeback(entries)))
                self.epilogue_graph = None
        self.locations = {id(new[k]): loc for k, loc in self.locations.items()}
        return True

    def async_ok(self) -> bool:
        """True if the lists installed by the last `rebind_device` all fit (synchronises)."""
        st = getattr(self, "async_status", None)
        return st is None or int(st.item()) == 0

    def __call__(self, *args, **kwargs):
        args = tuple(args) + tuple(kwargs[k] for k in self._kw_names)
        tensors = [a for a in args if isinstance(a, torch.Tensor)]
        for s, t in zip(self.static_inputs, tensors):
            s.copy_(t, non_blocking=True)
        return self.replay()

    def matches(self, args) -> bool:
        tensors = [a for a in args if isinstance(a, torch.Tensor)]
        if len(tensors) != len(self.static_inputs) or len(args) != len(self._arg_template):
            return False
        for s, t, dt in zip(self.static_inputs, tensors, self._arg_dtypes):
            if s.shape != t.shape or dt != t.dtype or s.device != t.device:
                return False
        return all((a is None and isinstance(b, torch.Tensor)) or (a is not None and not isinstance(b, torch.Tensor) and a == b)
                   for a, b in zip(self._arg_template, args))

    # ------------------------------------------------------------------ accounting
    def algorithmic_bytes(self) -> int:
        return sum(f.bytes for f in self.fused)

    def algorithmic_flops(self) -> int:
        return sum(f.flops for f in self.fused)
