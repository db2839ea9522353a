"""torch-facing wrappers of the C-ABI ops: same names, argument order and return convention as
the reference's pybind module ``sige.cuda`` (reference sige/cuda/pybind_cuda.cpp:5-12), so the
operator modules in ``sige_b200.nn`` call them exactly as the reference's modules call theirs.

PyTorch is plumbing here: it owns device memory (outputs are allocated with ``torch.empty``) and
the current stream; every byte of work is done by libsige_b200.so.  CUDA tensors only — a CPU or
MPS tensor raises (north-star: no multi-backend dispatch, no CPU fallback).

Extensions over the reference:
  * dtypes fp32 / fp16 / bf16 (the reference is fp32-only, sige/nn/base.py:15);
  * memory layout: NCHW-contiguous (the reference's) or channels-last; the stack a call returns
    follows the layout of its input;
  * ``out=`` / in-place forms used by the step engine (no per-call clone).
"""
from __future__ import annotations

from ctypes import byref
from typing import Optional, Tuple

import torch

from . import _cabi
from ._cabi import BF16, F16, F32, NCHW, NHWC, Bcast, ConvSrc, TileConv

_DTYPES = {torch.float32: F32, torch.float16: F16, torch.bfloat16: BF16}
_ACTS = {"identity": _cabi.ACT_IDENTITY, "swish": _cabi.ACT_SWISH}

# launch counter: bench.py reports it as `gpu_launches` (kernels of OUR library only)
launch_count = 0


def _act(name: str) -> int:
    try:
        return _ACTS[name]
    except KeyError:
        # the reference hits __builtin_unreachable() here (sige/common.cpp:22)
        raise ValueError("Unknown activation: [%s]!!!" % name) from None


def _dt(t: torch.Tensor) -> int:
    try:
        return _DTYPES[t.dtype]
    except KeyError:
        raise NotImplementedError("sige_b200 does not support dtype [%s]" % t.dtype) from None


def _require_cuda(*ts) -> None:
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError(
                "sige_b200 runs on CUDA (sm_90a) only; got a tensor on '%s'. "
                "There is no CPU/MPS backend and no fallback." % t.device
            )


def _stream(t: torch.Tensor) -> int:
    return torch.cuda.current_stream(t.device).cuda_stream


def layout_of(t: torch.Tensor) -> int:
    """NHWC if the 4-D tensor is densely channels-last (and not also NCHW-dense)."""
    if t.is_contiguous():
        return NCHW
    if t.is_contiguous(memory_format=torch.channels_last):
        return NHWC
    return -1


def _dense(t: torch.Tensor, layout: Optional[int] = None) -> Tuple[torch.Tensor, int]:
    """Return (tensor, layout) with the tensor dense in `layout` (or in its own dense layout)."""
    lo = layout_of(t)
    if layout is None:
        if lo >= 0:
            return t, lo
        return t.contiguous(), NCHW
    if lo == layout:
        return t, layout
    if layout == NCHW:
        return t.contiguous(), NCHW
    # NHWC requested.  A tensor that is NCHW-dense with C == 1 or H == W == 1 is also NHWC-dense
    if t.is_contiguous(memory_format=torch.channels_last):
        return t, NHWC
    return t.contiguous(memory_format=torch.channels_last), NHWC


def _empty_like_layout(shape, ref: torch.Tensor, layout: int) -> torch.Tensor:
    fmt = torch.channels_last if layout == NHWC else torch.contiguous_format
    return torch.empty(shape, dtype=ref.dtype, device=ref.device, memory_format=fmt)


def _bcast(t: Optional[torch.Tensor]) -> Optional[Bcast]:
    if t is None:
        return None
    if t.dim() != 4:
        raise NotImplementedError("broadcast operand must be 4-D, got %d-D" % t.dim())
    b = Bcast()
    b.ptr = t.data_ptr()
    for d in range(4):
        b.dims[d] = t.shape[d]
        b.stride[d] = t.stride(d)
    b.dtype = _dt(t)
    return b


def _bref(b: Optional[Bcast]):
    return None if b is None else byref(b)


def _idx(active_indices: torch.Tensor) -> torch.Tensor:
    if active_indices.dtype != torch.int32:
        raise TypeError("active_indices must be int32 [N,2]")
    return active_indices if active_indices.is_contiguous() else active_indices.contiguous()


def _same_dtype(what: str, ref: torch.Tensor, **tensors) -> None:
    """The kernels take ONE dtype per call from `ref`; a mismatch (e.g. an fp16 stack under autocast against an fp32 cache)
    would reinterpret memory."""
    for name, t in tensors.items():
        if t is not None and t.dtype != ref.dtype:
            raise TypeError("%s: %s is %s but the cached tensor is %s" % (what, name, t.dtype, ref.dtype))


def _bump(n: int = 1) -> None:
    global launch_count
    launch_count += n


# --------------------------------------------------------------------------------------
# a1: reduce_mask on device          (reference sige/utils.py:8-37)
# --------------------------------------------------------------------------------------
def reduce_mask_cuda_launch(mask: torch.Tensor, block_size, stride, padding):
    """Enqueue the ordered-compaction kernel; returns (idx buffer [capacity, 2], device count [1]) WITHOUT synchronising."""
    _require_cuda(mask)
    H, W = mask.shape
    cap = _cabi.lib().sige_reduce_mask_capacity(H, W, block_size[0], block_size[1], stride[0], stride[1], padding[0], padding[1])
    _cabi.check(cap < 0, "sige_reduce_mask_capacity")
    m8 = mask.to(torch.uint8) if mask.dtype != torch.uint8 else mask
    m8 = m8.contiguous()
    out = torch.empty((cap, 2), dtype=torch.int32, device=mask.device)
    count = torch.empty((1,), dtype=torch.int32, device=mask.device)
    with torch.cuda.device(mask.device):
        _cabi.check(
            _cabi.lib().sige_reduce_mask(m8.data_ptr(), H, W, block_size[0], block_size[1], stride[0], stride[1],
                                         padding[0], padding[1], out.data_ptr(), cap, count.data_ptr(), _stream(mask)),
            "sige_reduce_mask",
        )
    _bump()
    return out, count


def reduce_mask_batched_cuda(masks: torch.Tensor, block_size, stride, padding, cap: int, out: Optional[torch.Tensor] = None,
                             status: Optional[torch.Tensor] = None):
    """bool/uint8 [E, H, W] CUDA masks of one geometry -> (int32 [E*cap, 2] per-image tile lists, row e*cap + i = tile i of
    edit e, SIGE_TILE_NONE behind each edit's tiles; int32 [E] device counts; int32 [1] device status, bit 0 = some edit had
    more than `cap` tiles and was truncated), as ONE launch of `sige_reduce_mask_batched`, without synchronising.  `out` and
    `status` may be given (the status word is OR-ed into, not cleared)."""
    _require_cuda(masks, out, status)
    if masks.dim() != 3:
        raise ValueError("reduce_mask_batched_cuda expects [E, H, W] masks")
    E, H, W = masks.shape
    m8 = (masks.to(torch.uint8) if masks.dtype != torch.uint8 else masks).contiguous()
    if out is None:
        out = torch.empty((E * cap, 2), dtype=torch.int32, device=masks.device)
    if out.dtype != torch.int32 or tuple(out.shape) != (E * cap, 2) or not out.is_contiguous():
        raise ValueError("reduce_mask_batched_cuda: out must be a contiguous int32 [E*cap, 2] tensor")
    if status is None:
        status = torch.zeros((1,), dtype=torch.int32, device=masks.device)
    counts = torch.empty((E,), dtype=torch.int32, device=masks.device)
    with torch.cuda.device(masks.device):
        _cabi.check(
            _cabi.lib().sige_reduce_mask_batched(m8.data_ptr(), E, H, W, block_size[0], block_size[1], stride[0], stride[1],
                                                 padding[0], padding[1], out.data_ptr(), cap, counts.data_ptr(), status.data_ptr(),
                                                 _stream(masks)),
            "sige_reduce_mask_batched",
        )
    _bump()
    return out, counts, status


def reduce_mask_cuda(mask: torch.Tensor, block_size, stride, padding) -> torch.Tensor:
    """bool/uint8 [H,W] CUDA mask -> int32 [N,2] active tile origins, row-major, bit-exact."""
    out, count = reduce_mask_cuda_launch(mask, block_size, stride, padding)
    n = int(count.item())  # one host sync (the reference's torch.nonzero syncs too); SIGEModel.set_masks batches all geometries into one
    return out[:n].contiguous()


# --------------------------------------------------------------------------------------
# a2: gather                          (reference sige/cuda/gather_kernel.cu:69-124)
# --------------------------------------------------------------------------------------
def gather(x, bsize_h: int, bsize_w: int, active_indices, scale=None, shift=None, activation_name: str = "identity",
           activation_first: bool = False, out: Optional[torch.Tensor] = None, up: int = 0) -> torch.Tensor:
    """``up=1``: x holds (H/2, W/2) pixels and is read through nearest x2 up-sampling (tile origins refer to (H, W))."""
    _require_cuda(x, active_indices, scale, shift)
    x, layout = _dense(x)
    idx = _idx(active_indices)
    B, C, H, W = x.shape
    H, W = H << up, W << up
    N = idx.shape[0]
    if out is None:
        out = _empty_like_layout((B * N, C, bsize_h, bsize_w), x, layout)
    if N == 0:
        return out
    sc, sh = _bcast(scale), _bcast(shift)
    with torch.cuda.device(x.device):
        _cabi.check(
            _cabi.lib().sige_gather_upsampled(x.data_ptr(), _dt(x), layout, B, C, H, W, int(up), bsize_h, bsize_w, idx.data_ptr(), N,
                                              _bref(sc), _bref(sh), _act(activation_name), int(activation_first), out.data_ptr(), _stream(x)),
            "sige_gather",
        )
    _bump()
    return out


# --------------------------------------------------------------------------------------
# a6: scatter                         (reference sige/cuda/scatter_kernel.cu:76-117)
# --------------------------------------------------------------------------------------
def scatter(x, y, offset_h: int, offset_w: int, stride_h: int, stride_w: int, active_indices, residual=None,
            out: Optional[torch.Tensor] = None, inplace: bool = False) -> torch.Tensor:
    """out = copy(y) with the tiles of x pasted (+ residual).  ``inplace=True`` pastes into y itself
    (the step engine's no-clone form; equals the reference's sparse_update, sige/nn/scatter.py:59-60)."""
    _require_cuda(x, y, active_indices, residual)
    y, layout = _dense(y)
    x, _ = _dense(x, layout)
    idx = _idx(active_indices)
    B, C, H, W = y.shape
    _, Cx, Ro, So = x.shape
    if Cx != C:
        raise ValueError("scatter: channel mismatch %d vs %d" % (Cx, C))
    N = idx.shape[0]
    _same_dtype("scatter", y, x=x)
    if x.shape[0] != B * N:
        raise ValueError("scatter: the stack has %d rows, expected B*N = %d*%d" % (x.shape[0], B, N))
    if inplace:
        out, y_ptr = y, None
    else:
        if out is None:
            out = _empty_like_layout(y.shape, y, layout)
        y_ptr = y.data_ptr()
    res = _bcast(residual)
    with torch.cuda.device(y.device):
        _cabi.check(
            _cabi.lib().sige_scatter(x.data_ptr() if N else None, y_ptr, out.data_ptr(), _dt(y), layout, B, C, H, W, Ro, So,
                                     offset_h, offset_w, stride_h, stride_w, idx.data_ptr() if N else None, N, _bref(res),
                                     _stream(y)),
            "sige_scatter",
        )
    _bump(1 if inplace else 2)
    return out


# --------------------------------------------------------------------------------------
# a7: scatter_with_block_residual     (reference sige/cuda/scatter_kernel.cu:119-146)
# --------------------------------------------------------------------------------------
def scatter_with_block_residual(x0, y0, x1, y1, offset_h: int, offset_w: int, stride_h: int, stride_w: int,
                                active_indices0, active_indices1, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _require_cuda(x0, y0, x1, y1, active_indices0, active_indices1)
    y0, layout = _dense(y0)
    x0, _ = _dense(x0, layout)
    x1, _ = _dense(x1, layout)
    y1, _ = _dense(y1, layout)
    idx0, idx1 = _idx(active_indices0), _idx(active_indices1)
    B, C, H, W = y0.shape
    if out is None:
        out = _empty_like_layout(y0.shape, y0, layout)
    N0, N1 = idx0.shape[0], idx1.shape[0]
    _same_dtype("scatter_with_block_residual", y0, x0=x0, x1=x1, y1=y1)
    if x0.shape[0] != B * N0 or x1.shape[0] != B * N1 or x0.shape[1] != C or x1.shape[1] != C or tuple(y1.shape) != tuple(y0.shape):
        raise ValueError("scatter_with_block_residual: stack / cache shapes do not match the index lists")
    with torch.cuda.device(y0.device):
        _cabi.check(
            _cabi.lib().sige_scatter_with_block_residual(
                x0.data_ptr() if N0 else None, y0.data_ptr(), x1.data_ptr() if N1 else None, y1.data_ptr(), out.data_ptr(),
                _dt(y0), layout, B, C, H, W, x0.shape[2], x0.shape[3], x1.shape[2], x1.shape[3], offset_h, offset_w,
                stride_h, stride_w, idx0.data_ptr() if N0 else None, N0, idx1.data_ptr() if N1 else None, N1, _stream(y0)),
            "sige_scatter_with_block_residual",
        )
    _bump(3)
    return out


# --------------------------------------------------------------------------------------
# a5: get_scatter_map                 (reference sige/cuda/scatter_gather_kernel.cu:164-188)
# --------------------------------------------------------------------------------------
def get_scatter_map(H: int, W: int, bsize_h: int, bsize_w: int, ksize_h: int, ksize_w: int, offset_h: int, offset_w: int,
                    stride_h: int, stride_w: int, active_indices) -> torch.Tensor:
    _require_cuda(active_indices)
    idx = _idx(active_indices)
    out = torch.empty((H, W, 3), dtype=torch.int32, device=idx.device)
    N = idx.shape[0]
    with torch.cuda.device(idx.device):
        _cabi.check(
            _cabi.lib().sige_get_scatter_map(H, W, bsize_h, bsize_w, ksize_h, ksize_w, offset_h, offset_w, stride_h, stride_w,
                                             idx.data_ptr() if N else None, N, out.data_ptr(), _stream(idx)),
            "sige_get_scatter_map",
        )
    _bump(2)
    return out


# --------------------------------------------------------------------------------------
# a4: scatter_gather                  (reference sige/cuda/scatter_gather_kernel.cu:100-162)
# --------------------------------------------------------------------------------------
def scatter_gather(x, y, bsize_h: int, bsize_w: int, active_indices, scatter_map, scale=None, shift=None,
                   activation_name: str = "identity", activation_first: bool = False,
                   out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _require_cuda(x, y, active_indices, scatter_map, scale, shift)
    y, layout = _dense(y)
    x, _ = _dense(x, layout)
    idx = _idx(active_indices)
    B, C, H, W = y.shape
    N = idx.shape[0]
    if out is None:
        out = _empty_like_layout((B * N, C, bsize_h, bsize_w), y, layout)
    if N == 0:
        return out
    if x.shape[1] != C:
        raise ValueError("scatter_gather: channel mismatch %d vs %d" % (x.shape[1], C))
    _same_dtype("scatter_gather", y, x=x)
    if tuple(scatter_map.shape) != (H, W, 3) or scatter_map.dtype != torch.int32:
        raise ValueError("scatter_gather: scatter_map must be int32 [H, W, 3] = [%d, %d, 3]" % (H, W))
    smap = scatter_map if scatter_map.is_contiguous() else scatter_map.contiguous()
    sc, sh = _bcast(scale), _bcast(shift)
    with torch.cuda.device(y.device):
        _cabi.check(
            _cabi.lib().sige_scatter_gather(x.data_ptr(), y.data_ptr(), _dt(y), layout, B, C, H, W, x.shape[2], x.shape[3],
                                            bsize_h, bsize_w, idx.data_ptr(), N, smap.data_ptr(), _bref(sc), _bref(sh),
                                            _act(activation_name), int(activation_first), out.data_ptr(), _stream(y)),
            "sige_scatter_gather",
        )
    _bump()
    return out


# --------------------------------------------------------------------------------------
# a3: tile convolution
# --------------------------------------------------------------------------------------
def pack_conv_weight(weight: torch.Tensor, dtype: torch.dtype, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """OIHW -> packed weights in `dtype` (f16/bf16) for the tensor-core kernels.  The returned tensor has the
    bookkeeping shape (kH*kW, Cout, Cin); its memory order is [tap][Cin/64][Cout][64] (contiguous slabs per
    (tap, 64-channel chunk)) when Cin % 64 == 0.  `out`: an earlier result of the same shape and dtype, overwritten in place."""
    _require_cuda(weight)
    w = weight.detach().contiguous()
    Cout, Cin, kH, kW = w.shape
    if out is None:
        out = torch.empty((kH * kW, Cout, Cin), dtype=dtype, device=w.device)
    elif tuple(out.shape) != (kH * kW, Cout, Cin) or out.dtype != dtype or not out.is_contiguous() or out.device != w.device:
        raise ValueError("pack_conv_weight: out must be a contiguous %s tensor of shape %s" % (dtype, (kH * kW, Cout, Cin)))
    with torch.cuda.device(w.device):
        _cabi.check(
            _cabi.lib().sige_pack_conv_weight(w.data_ptr(), _dt(w), Cout, Cin, kH, kW, out.data_ptr(), _DTYPES[dtype], _stream(w)),
            "sige_pack_conv_weight",
        )
    _bump()
    return out


def tile_conv_tc_supported(x: torch.Tensor, weight: torch.Tensor, stride, dilation, groups, ignore_cin: bool = False) -> bool:
    """Can the tensor-core kernel take this stack convolution?  (north-star: tensor cores where
    channels >= 64, CUDA-core kernel otherwise.)"""
    return (
        x.dtype in (torch.float16, torch.bfloat16)
        and groups == 1
        and tuple(dilation) == (1, 1)
        and stride[0] == stride[1]
        and (ignore_cin or weight.shape[1] % 64 == 0)
        and weight.shape[0] % 8 == 0
        and x.shape[2] >= weight.shape[2] and x.shape[3] >= weight.shape[3]
        and ((x.shape[2] - weight.shape[2]) // stride[0] + 1) * ((x.shape[3] - weight.shape[3]) // stride[1] + 1) <= 128
        and x.shape[2] * x.shape[3] <= 288
    )


def tile_conv_supported(cin: int, cout: int, k: int, stride: int, dtype: torch.dtype) -> bool:
    """Does ``sige_tile_conv`` take a conv of `cin` -> `cout` channels with a single source, whatever the source is: a narrow one
    (cin a multiple of 8 but not of 64: the mma.sync kernel with a partial last K chunk, the weight packed zero-padded to
    round_up(cin, 64) input channels), a channel window of a wider buffer, or SPADE's modulation in the gather stage?  With the wgmma
    flag, the wgmma kernel runs the geometries it takes; the mma.sync kernel runs the rest."""
    return dtype in (torch.float16, torch.bfloat16) and cin > 0 and cin % 8 == 0 and cout > 0 and cout % 8 == 0 and k >= 1 and stride >= 1


def tile_conv_descriptor() -> TileConv:
    return TileConv()


def launch_tile_conv(desc: TileConv, stream: int) -> None:
    _cabi.check(_cabi.lib().sige_tile_conv(byref(desc), stream), "sige_tile_conv")
    _bump()


def channel_window(t: torch.Tensor) -> Tuple[int, int, int]:
    """(address of channel 0 of pixel 0, channels per pixel, first channel) of a [B, C, H, W] tensor that is a whole channels-last
    buffer or a channel slice of one (``buf[:, c0:c1]``, a torch.split part)."""
    if t.dim() != 4 or t.stride(1) != 1:
        raise ValueError("channel_window: not a channel window of a channels-last 4-D tensor")
    B, C, H, W = (int(d) for d in t.shape)
    pitch = int(t.stride(3)) if W > 1 else (int(t.stride(2)) if H > 1 else C)
    if pitch < C or (H > 1 and t.stride(2) != W * pitch) or (B > 1 and t.stride(0) != H * W * pitch):
        raise ValueError("channel_window: pixels are not evenly spaced")
    c0 = int(t.storage_offset()) % pitch
    return t.data_ptr() - c0 * t.element_size(), pitch, c0


def conv_modulation(gamma: torch.Tensor, beta: torch.Tensor, negative_slope: float, gamma_c0: int = 0, beta_c0: int = 0) -> "_cabi.ConvModulation":
    """sige_conv_modulation_t of [B, C, H, W] gamma / beta read from channel gamma_c0 / beta_c0 on: channels-last buffers or channel
    windows of such buffers (the two torch.split halves of SPADE's gamma_beta, one buffer)."""
    m = _cabi.ConvModulation()
    g, gC, gc0 = channel_window(gamma)
    b, bC, bc0 = channel_window(beta)
    m.gamma, m.gamma_C, m.gamma_c0 = g, gC, gc0 + int(gamma_c0)
    m.beta, m.beta_C, m.beta_c0 = b, bC, bc0 + int(beta_c0)
    m.negative_slope = float(negative_slope)
    return m


def tile_conv_stack(x: torch.Tensor, w_packed: torch.Tensor, bias_f32: Optional[torch.Tensor], ksize: Tuple[int, int],
                    stride: int, out: Optional[torch.Tensor] = None, flags: int = 0, ksplit: int = 0) -> torch.Tensor:
    """Tensor-core conv on a stack: x (M, Cin, R, S) channels-last -> (M, Cout, Ro, So) channels-last.
    Equivalent of F.conv2d(x, w, b, stride, padding=0) (reference sige/nn/base.py:88-89)."""
    _require_cuda(x, w_packed, bias_f32)
    x, _ = _dense(x, NHWC)
    M, Cin, R, S = x.shape
    taps, Cout, Cin_w = w_packed.shape
    kH, kW = ksize
    if Cin_w != Cin or taps != kH * kW:
        raise ValueError("tile_conv_stack: weight does not match input")
    Ro, So = (R - kH) // stride + 1, (S - kW) // stride + 1
    if out is None:
        out = _empty_like_layout((M, Cout, Ro, So), x, NHWC)
    if M == 0:
        return out
    d = TileConv()
    d.dtype = _dt(x)
    d.n_src = 1
    d.src[0].ptr = x.data_ptr(); d.src[0].C = Cin; d.src[0].up = 0
    d.B, d.H, d.W = 1, R, S
    d.src_is_stack = 1
    d.idx = None
    d.N = M
    d.R, d.S = R, S
    d.scale = None; d.shift = None; d.affine_bstride = 0; d.act = 0
    d.w_packed = w_packed.data_ptr()
    d.bias = None if bias_f32 is None else bias_f32.data_ptr()
    d.Cin, d.Cout, d.kH, d.kW, d.stride = Cin, Cout, kH, kW, stride
    d.dst = out.data_ptr()
    d.dst_is_stack = 1
    d.dH, d.dW, d.dC, d.dst_c0 = Ro, So, Cout, 0
    d.offH = d.offW = 0
    d.residual = None; d.rC = 0; d.res_c0 = 0
    d.flags, d.ksplit = flags, ksplit
    with torch.cuda.device(x.device):
        launch_tile_conv(d, _stream(x))
    return out


def tile_conv_generic(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], stride, dilation, groups: int,
                      out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """CUDA-core conv on a stack, any dtype/shape; fp32 accumulate (F.conv2d(..., padding=0))."""
    _require_cuda(x, weight, bias)
    x, layout = _dense(x)
    w = weight.detach()
    if w.dtype != x.dtype:
        w = w.to(x.dtype)
    w = w.contiguous()
    b = None
    if bias is not None:
        b = bias.detach()
        if b.dtype != x.dtype:
            b = b.to(x.dtype)
        b = b.contiguous()
    M, Cin, R, S = x.shape
    Cout, _, kH, kW = w.shape
    Ro = (R - dilation[0] * (kH - 1) - 1) // stride[0] + 1
    So = (S - dilation[1] * (kW - 1) - 1) // stride[1] + 1
    if out is None:
        out = _empty_like_layout((M, Cout, Ro, So), x, layout)
    if M == 0:
        return out
    with torch.cuda.device(x.device):
        _cabi.check(
            _cabi.lib().sige_tile_conv_generic(x.data_ptr(), w.data_ptr(), None if b is None else b.data_ptr(), out.data_ptr(),
                                               _dt(x), layout, M, Cin, R, S, Cout, kH, kW, stride[0], stride[1], dilation[0],
                                               dilation[1], groups, _stream(x)),
            "sige_tile_conv_generic",
        )
    _bump()
    return out


# --------------------------------------------------------------------------------------
# dense glue of a step (conv_in / GroupNorm fold / conv_out), NHWC f16/bf16
# --------------------------------------------------------------------------------------
def conv_aux(view: torch.Tensor, scale: Optional[torch.Tensor], shift: Optional[torch.Tensor], activation_name: str):
    """Descriptor of an extra producer-side output: view = act(out*scale + shift), NHWC with the producer's channels;
    scale / shift fp32 [C] (kept alive by the caller)."""
    a = _cabi.ConvAux()
    a.ptr, a.C, a.c0 = view.data_ptr(), view.shape[1], 0
    a.scale = None if scale is None else scale.data_ptr()
    a.shift = None if shift is None else shift.data_ptr()
    a.act = _act(activation_name)
    return a


def conv_in_nhwc(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], out: Optional[torch.Tensor] = None,
                 aux=None, tiles: Optional[torch.Tensor] = None, tile_size: int = 6, tiles_per_image: bool = False) -> torch.Tensor:
    """3x3 pad-1 conv with Cin <= 4 on a channels-last image (reference sige_fused_unet.py:395).  With ``tiles`` (int32
    [N, 2] tile origins) only the pixels inside those tile_size x tile_size tiles of ``out`` are written."""
    _require_cuda(x, weight, bias, tiles)
    x, _ = _dense(x, NHWC)
    B, Cin, H, W = x.shape
    w = weight.detach().to(x.dtype).contiguous()
    b = None if bias is None else bias.detach().to(x.dtype).contiguous()
    Cout = w.shape[0]
    if out is None:
        out = _empty_like_layout((B, Cout, H, W), x, NHWC)
    with torch.cuda.device(x.device):
        n_aux = 0 if aux is None else len(aux)
        arr = (_cabi.ConvAux * 2)()
        for i in range(n_aux):
            arr[i] = aux[i]
        if tiles is not None:
            assert tiles.dtype == torch.int32 and tiles.dim() == 2 and tiles.shape[1] == 2 and tiles.is_contiguous()
            n_tiles = int(tiles.shape[0]) // B if tiles_per_image else int(tiles.shape[0])
            _cabi.check(_cabi.lib().sige_conv_in_nhwc_tiles(x.data_ptr(), w.data_ptr(), None if b is None else b.data_ptr(), out.data_ptr(), _dt(x),
                                                           B, H, W, Cin, Cout, tiles.data_ptr(), n_tiles, int(tile_size), int(tile_size),
                                                           int(bool(tiles_per_image)), n_aux, arr, _stream(x)), "sige_conv_in_nhwc_tiles")
        else:
            _cabi.check(_cabi.lib().sige_conv_in_nhwc(x.data_ptr(), w.data_ptr(), None if b is None else b.data_ptr(), out.data_ptr(), _dt(x), B, H, W,
                                                     Cin, Cout, n_aux, arr, _stream(x)), "sige_conv_in_nhwc")
    _bump()
    return out


def group_norm_fold_workspace(B: int, C: int) -> int:
    """Floats of workspace sige_group_norm_fold needs for B images of C channels on the current device."""
    need = _cabi.lib().sige_group_norm_fold_workspace(B, C)
    _cabi.check(need < 0, "sige_group_norm_fold_workspace")
    return need


def group_norm_fold(x: torch.Tensor, groups: int, eps: float, gamma: Optional[torch.Tensor], beta: Optional[torch.Tensor],
                    scale: Optional[torch.Tensor] = None, shift: Optional[torch.Tensor] = None, workspace: Optional[torch.Tensor] = None):
    """(scale, shift) fp32 [B, C] with GroupNorm(x) == x*scale + shift (reference models/common.py:37-57)."""
    _require_cuda(x, gamma, beta)
    x, _ = _dense(x, NHWC)
    B, C, H, W = x.shape
    g = None if gamma is None else gamma.detach().to(x.dtype).contiguous()
    bt = None if beta is None else beta.detach().to(x.dtype).contiguous()
    if scale is None:
        scale = torch.empty((B, C), dtype=torch.float32, device=x.device)
    if shift is None:
        shift = torch.empty((B, C), dtype=torch.float32, device=x.device)
    need = group_norm_fold_workspace(B, C)
    if workspace is None:
        workspace = torch.empty((need,), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _cabi.check(_cabi.lib().sige_group_norm_fold(x.data_ptr(), _dt(x), B, H, W, C, groups, float(eps), None if g is None else g.data_ptr(),
                                                    None if bt is None else bt.data_ptr(), scale.data_ptr(), shift.data_ptr(),
                                                    workspace.data_ptr(), workspace.numel(), _stream(x)), "sige_group_norm_fold")
    _bump(2)
    return scale, shift


def conv_out_nhwc(x: torch.Tensor, scale: Optional[torch.Tensor], shift: Optional[torch.Tensor], activation_name: str, weight: torch.Tensor,
                  bias: Optional[torch.Tensor], out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """NCHW out = conv3x3_pad1(act(x*scale+shift)), Cout <= 4 (reference sige_fused_unet.py:431-433)."""
    _require_cuda(x, scale, shift, weight, bias)
    x, _ = _dense(x, NHWC)
    B, C, H, W = x.shape
    w = weight.detach().to(x.dtype).contiguous()
    b = None if bias is None else bias.detach().to(x.dtype).contiguous()
    Cout = w.shape[0]
    if out is None:
        out = torch.empty((B, Cout, H, W), dtype=x.dtype, device=x.device)
    with torch.cuda.device(x.device):
        _cabi.check(_cabi.lib().sige_conv_out_nhwc(x.data_ptr(), None if scale is None else scale.data_ptr(), None if shift is None else shift.data_ptr(),
                                                  _act(activation_name), w.data_ptr(), None if b is None else b.data_ptr(), out.data_ptr(), _dt(x), B,
                                                  H, W, C, Cout, _stream(x)), "sige_conv_out_nhwc")
    _bump()
    return out


def attention_tokens_supported(n_tokens: int, channels: int, dtype: torch.dtype) -> bool:
    code = {torch.float16: _cabi.F16, torch.bfloat16: _cabi.BF16}.get(dtype)
    return code is not None and bool(_cabi.lib().sige_attention_tokens_supported(int(n_tokens), int(channels), code))


def attention_tokens(qkv: torch.Tensor, out: Optional[torch.Tensor] = None, flags: int = 0) -> torch.Tensor:
    """softmax(q k^T) v on tokens: qkv [B, N, 3C] contiguous = per token [q | k | v] with q pre-scaled by C^-0.5
    (reference sige_fused_unet.py:185-199); returns [B, N, C]."""
    _require_cuda(qkv, out)
    assert qkv.dim() == 3 and qkv.is_contiguous() and qkv.shape[2] % 3 == 0
    B, N, C3 = qkv.shape
    C = C3 // 3
    if out is None:
        out = torch.empty((B, N, C), dtype=qkv.dtype, device=qkv.device)
    assert out.is_contiguous() and out.shape == (B, N, C) and out.dtype == qkv.dtype
    with torch.cuda.device(qkv.device):
        _cabi.check(_cabi.lib().sige_attention_tokens(qkv.data_ptr(), out.data_ptr(), B, N, C, _dt(qkv), int(flags), _stream(qkv)),
                    "sige_attention_tokens")
    _bump()
    return out


def sparse_attention_supported(head_dim: int, dtype: torch.dtype) -> bool:
    code = {torch.float16: _cabi.F16, torch.bfloat16: _cabi.BF16}.get(dtype)
    return code is not None and bool(_cabi.lib().sige_sparse_attention_supported(int(head_dim), code))


def sparse_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """softmax(scale * q k^T) v for sparse queries against all keys (reference stable-diffusion/ldm/modules/attention.py:81-93,
    sige_attention.py:44-58).  Operands are [BH, N, D] (the reference's "(b h) n d") or [B, heads, N, D]; any strides whose
    last dim is contiguous and which are multiples of 8 elements — a permuted view of the Linear output "b n (h d)" works
    without a copy.  Returns a tensor shaped like q."""
    _require_cuda(q, k, v, out)
    if q.dim() == 3:
        q4, k4, v4 = q.unsqueeze(1), k.unsqueeze(1), v.unsqueeze(1)
    else:
        q4, k4, v4 = q, k, v
    if not (q4.dim() == k4.dim() == v4.dim() == 4):
        raise ValueError("sparse_attention: q, k, v must all be [BH, N, D] or all [B, heads, N, D]")
    B, Hh, Nq, D = q4.shape
    Nk = k4.shape[2]
    if tuple(k4.shape) != (B, Hh, Nk, D) or tuple(v4.shape) != (B, Hh, Nk, D):
        raise ValueError("sparse_attention: shapes q %s, k %s, v %s do not match" % (tuple(q.shape), tuple(k.shape), tuple(v.shape)))
    if not (q.dtype == k.dtype == v.dtype):
        raise TypeError("sparse_attention: dtypes differ (%s, %s, %s)" % (q.dtype, k.dtype, v.dtype))
    if not scale > 0:
        raise ValueError("sparse_attention: scale must be positive")
    if out is None:
        out = torch.empty(tuple(q.shape), dtype=q.dtype, device=q.device)
    if tuple(out.shape) != tuple(q.shape) or out.dtype != q.dtype:
        raise ValueError("sparse_attention: out must have q's shape and dtype")
    o4 = out.unsqueeze(1) if out.dim() == 3 else out
    d = _cabi.SparseAttention()
    d.q, d.k, d.v, d.out = q4.data_ptr(), k4.data_ptr(), v4.data_ptr(), o4.data_ptr()
    d.B, d.heads, d.Nq, d.Nk, d.D = int(B), int(Hh), int(Nq), int(Nk), int(D)
    for name, t in (("q_stride", q4), ("k_stride", k4), ("v_stride", v4), ("out_stride", o4)):
        if t.numel() and t.stride(3) != 1:
            raise ValueError("sparse_attention: the head dim must be contiguous")
        st = getattr(d, name)
        for i in range(3):
            st[i] = int(t.stride(i)) if t.shape[i] > 1 else 0
    d.scale = float(scale)
    d.dtype = _dt(q)
    d.flags = 0
    with torch.cuda.device(q.device):
        _cabi.check(_cabi.lib().sige_sparse_attention(byref(d), _stream(q)), "sige_sparse_attention")
    _bump()
    return out


def _pixel_rows(t: torch.Tensor):
    """(pixels, C, pixel stride) of a channels-innermost 4-D tensor whose pixels are uniformly strided (an NHWC buffer / stack or a
    channel slice of one); None otherwise."""
    if t.dim() != 4 or t.numel() == 0 or t.stride(1) != 1:
        return None
    n, c, h, w = t.shape
    ps = t.stride(3) if w > 1 else (t.stride(2) if h > 1 else t.stride(0))
    if (w > 1 and h > 1 and t.stride(2) != ps * w) or ((h > 1 or w > 1) and n > 1 and t.stride(0) != ps * h * w):
        return None
    return n * h * w, c, int(ps)


def spade_modulate_supported(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor) -> bool:
    if not (x.is_cuda and x.dtype == gamma.dtype == beta.dtype and x.dtype in (torch.float32, torch.float16, torch.bfloat16)
            and tuple(x.shape) == tuple(gamma.shape) == tuple(beta.shape)):
        return False
    vec = 4 if x.dtype == torch.float32 else 8
    for t in (x, gamma, beta):
        r = _pixel_rows(t)
        if r is None or r[1] % vec or r[2] % vec or t.data_ptr() % 16:
            return False
    return True


def spade_modulate(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, negative_slope: float = 1.0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """act(x * (1 + gamma) + beta) on channels-innermost tensors (reference gaugan/models/sige_normalization.py:84-86 + the
    block's leaky_relu); negative_slope = 1 is the identity.  Returns a channels-last tensor shaped like x."""
    _require_cuda(x, gamma, beta, out)
    if not spade_modulate_supported(x, gamma, beta):
        raise ValueError("spade_modulate: operands must be same-shape, same-dtype, channels-innermost 4-D tensors with 16-byte channel vectors")
    if out is None:
        out = torch.empty(tuple(x.shape), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
    ro = _pixel_rows(out)
    if ro is None or tuple(out.shape) != tuple(x.shape) or out.dtype != x.dtype:
        raise ValueError("spade_modulate: out must be a channels-innermost tensor with x's shape and dtype")
    (px, c, xs), (_, _, gs), (_, _, bs) = _pixel_rows(x), _pixel_rows(gamma), _pixel_rows(beta)
    with torch.cuda.device(x.device):
        _cabi.check(_cabi.lib().sige_spade_modulate(x.data_ptr(), xs, gamma.data_ptr(), gs, beta.data_ptr(), bs, out.data_ptr(), ro[2], px, c,
                                                   float(negative_slope), _dt(x), _stream(x)), "sige_spade_modulate")
    _bump()
    return out


def separable_conv_supported(cin: int, cout: int, dtype: torch.dtype) -> bool:
    code = {torch.float16: _cabi.F16, torch.bfloat16: _cabi.BF16}.get(dtype)
    return code is not None and bool(_cabi.lib().sige_separable_conv_supported(int(cin), int(cout), 3, code))


def separable_fold(dw_weight: torch.Tensor, dw_bias: Optional[torch.Tensor], scale: Optional[torch.Tensor], shift: Optional[torch.Tensor]):
    """fp32 (weight [C, 9], bias [C]) of a depthwise 3x3 conv followed by the per-channel affine x*scale + shift:
    weight = scale*w, bias = scale*b + shift (reference gaugan/models/mobile_modules.py:110-111)."""
    c = int(dw_weight.shape[0])
    w = dw_weight.detach().float().reshape(c, 9)
    b = torch.zeros(c, dtype=torch.float32, device=w.device) if dw_bias is None else dw_bias.detach().float().reshape(c)
    if scale is not None:
        sc = scale.detach().float().reshape(c).to(w.device)
        w, b = w * sc.view(c, 1), b * sc
    if shift is not None:
        b = b + shift.detach().float().reshape(c).to(w.device)
    return w.contiguous(), b.contiguous()


def separable_conv(x: torch.Tensor, branches, idx: Optional[torch.Tensor] = None, *, src_stack: bool = False, dst_stack: bool = False,
                   offset: int = 1, batch: int = 1, flags: int = 0) -> None:
    """Separable 3x3 conv of 6x6 halo tiles -> 4x4 outputs, up to two branches on one input, one launch (sige_separable_conv).

    x: channels-innermost 4-D tensor, possibly a channel slice (torch.split) of a wider one: an NHWC buffer [B, Cin, H, W] read
    through ``idx`` (int32 [N, 2] halo-tile origins), or a tile stack [B*N, Cin, 6, 6] (``src_stack``).  ``branches``: one or two
    (dw_weight fp32 [Cin, 9], dw_bias fp32 [Cin], pw_weight [Cout, Cin] in x's dtype, pw_bias fp32 [Cout] or None, out) with the
    affine folded into the depthwise part (``separable_fold``); ``out`` is a channels-innermost NHWC buffer [B, Cout, dH, dW] whose
    tiles at ``idx + offset`` are overwritten in place, or a stack [B*N, Cout, 4, 4] (``dst_stack``).  With
    CONV_PER_IMAGE_OPERANDS in ``flags`` (a batch of independent edits; buffer source and destinations) ``idx`` holds B lists of
    N rows, row b*N + i = tile i of image b."""
    from ._cabi import CONV_PER_IMAGE_OPERANDS, SeparableConv

    _require_cuda(x, idx)
    if not 1 <= len(branches) <= 2:
        raise ValueError("separable_conv: one or two branches")
    rx = _pixel_rows(x)
    if rx is None or x.data_ptr() % 16:
        raise ValueError("separable_conv: x must be a channels-innermost 4-D tensor with uniformly strided pixels, 16-byte aligned")
    cin = int(x.shape[1])
    d = SeparableConv()
    d.dtype = _dt(x)
    d.src, d.src_is_stack, d.src_C, d.src_c0 = x.data_ptr(), int(src_stack), rx[2], 0
    if src_stack:
        if tuple(x.shape[2:]) != (6, 6) or x.shape[0] % batch:
            raise ValueError("separable_conv: a stack source is [B*N, Cin, 6, 6]")
        d.B, d.H, d.W, d.N = int(batch), 6, 6, int(x.shape[0]) // batch
    else:
        if idx is None:
            raise ValueError("separable_conv: a buffer source needs the tile list")
        d.B, d.H, d.W, d.N = int(x.shape[0]), int(x.shape[2]), int(x.shape[3]), int(idx.shape[0])
        if flags & CONV_PER_IMAGE_OPERANDS:
            if d.N % d.B:
                raise ValueError("separable_conv: per-image lists hold B * N rows")
            d.N //= d.B
    if idx is not None:
        idx = _idx(idx)
        if idx.dim() != 2 or idx.shape[1] != 2 or (src_stack and int(idx.shape[0]) != d.N):
            raise ValueError("separable_conv: idx must be int32 [N, 2] with one row per tile")
    elif not dst_stack:
        raise ValueError("separable_conv: a buffer destination needs the tile list")
    d.idx = None if idx is None else idx.data_ptr()
    d.Cin, d.offH, d.offW, d.nbranch, d.flags = cin, int(offset), int(offset), len(branches), int(flags)
    for i, (dw_w, dw_b, pw_w, pw_b, out) in enumerate(branches):
        pw_w = pw_w.reshape(pw_w.shape[0], -1)
        cout = int(pw_w.shape[0])
        if i == 0:
            d.Cout = cout
        if (cout != d.Cout or tuple(pw_w.shape) != (cout, cin) or pw_w.dtype != x.dtype or not pw_w.is_contiguous() or dw_w.dtype != torch.float32
                or tuple(dw_w.shape) != (cin, 9) or not dw_w.is_contiguous() or (dw_b is not None and (dw_b.dtype != torch.float32 or dw_b.numel() != cin))
                or (pw_b is not None and (pw_b.dtype != torch.float32 or pw_b.numel() != cout))):
            raise ValueError("separable_conv: branch %d: weights do not match (dw fp32 [Cin, 9], pw [Cout, Cin] in x's dtype, fp32 biases)" % i)
        ro = _pixel_rows(out)
        if ro is None or out.dtype != x.dtype or int(out.shape[1]) != cout or (dst_stack and tuple(out.shape) != (d.B * d.N, cout, 4, 4)) \
                or (not dst_stack and int(out.shape[0]) != d.B):
            raise ValueError("separable_conv: branch %d: out must be a channels-innermost %s with Cout channels in x's dtype" % (i, "stack [B*N, Cout, 4, 4]" if dst_stack else "buffer [B, Cout, dH, dW]"))
        _require_cuda(dw_w, dw_b, pw_w, pw_b, out)
        br = d.branch[i]
        br.dw_weight, br.dw_bias = dw_w.data_ptr(), None if dw_b is None else dw_b.data_ptr()
        br.pw_weight, br.pw_bias = pw_w.data_ptr(), None if pw_b is None else pw_b.data_ptr()
        br.dst, br.dst_is_stack, br.dH, br.dW, br.dst_C, br.dst_c0 = out.data_ptr(), int(dst_stack), int(out.shape[2]), int(out.shape[3]), ro[2], 0
    with torch.cuda.device(x.device):
        _cabi.check(_cabi.lib().sige_separable_conv(byref(d), _stream(x)), "sige_separable_conv")
    _bump()


# --------------------------------------------------------------------------------------
# a8: sparse_update write-back       (reference sige/nn/scatter.py:59-60,114-129, scatter_gather.py:65-77)
# --------------------------------------------------------------------------------------
def tile_writeback_launcher(entries):
    """Prepare `sige_tile_writeback` over ``entries`` and return ``run(stream)``, which enqueues it (one launch per
    SIGE_WRITEBACK_MAX_ENTRIES entries).  Entry = (src, dst, idx, off, stride, tile): ``src`` a channels-last f16 / bf16 buffer
    [B, C, H, W]; ``dst`` its cache, the same shape, NCHW- or NHWC-dense, f32 or src's dtype; ``idx`` int32 [N, 2] tile origins
    (SIGE_TILE_NONE entries write nothing); ``off`` / ``stride`` / ``tile`` = (h, w) pairs or ints: tile i writes rows
    [(idx_h + off_h) / stride_h, + tile_h) and the matching columns, clipped to the image.  The tensors are not copied: the
    launch reads them (and the tile lists) as they are when it runs."""
    from ._cabi import WRITEBACK_MAX_ENTRIES, WritebackEntry

    def pair(v):
        return (int(v[0]), int(v[1])) if isinstance(v, (tuple, list)) else (int(v), int(v))

    rows, keep, dev = [], [], None
    for k, (src, dst, idx, off, stride, tile) in enumerate(entries):
        _require_cuda(src, dst, idx)
        idx = _idx(idx)
        if src.dim() != 4 or tuple(dst.shape) != tuple(src.shape) or not src.is_contiguous(memory_format=torch.channels_last):
            raise ValueError("tile_writeback: entry %d: src must be a channels-last [B, C, H, W] buffer and dst the same shape" % k)
        lo = layout_of(dst)
        if lo < 0:
            raise ValueError("tile_writeback: entry %d: dst must be NCHW- or NHWC-dense" % k)
        if idx.dim() != 2 or idx.shape[1] != 2:
            raise ValueError("tile_writeback: entry %d: idx must be int32 [N, 2]" % k)
        dev = dev or src.device
        e = WritebackEntry()
        e.src, e.dst, e.idx = src.data_ptr(), dst.data_ptr(), idx.data_ptr()
        e.N, e.B, e.C, e.H, e.W = int(idx.shape[0]), int(src.shape[0]), int(src.shape[1]), int(src.shape[2]), int(src.shape[3])
        e.src_dtype, e.dst_dtype, e.dst_layout = _dt(src), _dt(dst), lo
        (e.offH, e.offW), (e.strideH, e.strideW), (e.Ro, e.So) = pair(off), pair(stride), pair(tile)
        rows.append(e)
        keep.append((src, dst, idx))
    tables = []
    for s in range(0, len(rows), WRITEBACK_MAX_ENTRIES):
        part = rows[s:s + WRITEBACK_MAX_ENTRIES]
        tables.append(((WritebackEntry * len(part))(*part), len(part)))

    def run(stream: int) -> None:
        _ = keep
        for table, n in tables:
            with torch.cuda.device(dev):
                _cabi.check(_cabi.lib().sige_tile_writeback(table, n, stream), "sige_tile_writeback")
            _bump()

    return run


def cache_load_launcher(entries, dtype: torch.dtype):
    """Prepare `sige_cache_load` over ``entries`` and return ``run(stream)``, which enqueues it (one launch per
    SIGE_CACHE_LOAD_MAX_ENTRIES entries).  Entry = (src, raw, views): ``src`` a module cache [1 or E, C, H, W], NCHW- or
    NHWC-dense, f32 / f16 / bf16; ``raw`` None or a channels-last [E, C, H, W] buffer in ``dtype`` that receives the cache;
    ``views`` up to two (dst, scale, shift, act): dst like raw, receiving act(src * scale + shift) with fp32 [C] scale / shift
    (or None) and act "identity" or "swish".  The tensors are not copied: the launch reads them as they are when it runs."""
    from ._cabi import CACHE_LOAD_MAX_ENTRIES, CacheLoadEntry

    if dtype not in (torch.float16, torch.bfloat16):
        raise ValueError("cache_load: the destinations are f16 or bf16, not %s" % dtype)
    rows, keep, dev = [], [], None
    for k, (src, raw, views) in enumerate(entries):
        views = list(views)
        _require_cuda(src, raw, *[t for v in views for t in v[:3]])
        lo = layout_of(src) if src.dim() == 4 else -1
        if lo < 0 or src.dtype not in _DTYPES:
            raise ValueError("cache_load: entry %d: src must be an NCHW- or NHWC-dense 4-D f32 / f16 / bf16 tensor" % k)
        dsts = ([raw] if raw is not None else []) + [v[0] for v in views]
        if not dsts or len(views) > 2:
            raise ValueError("cache_load: entry %d: a raw destination and / or one or two views" % k)
        E, C, H, W = (int(d) for d in dsts[0].shape)
        if int(src.shape[0]) not in (1, E) or tuple(src.shape[1:]) != (C, H, W) or C % 8:
            raise ValueError("cache_load: entry %d: src %s does not match destinations %s (C a multiple of 8)" % (k, tuple(src.shape), tuple(dsts[0].shape)))
        for d in dsts:
            if tuple(d.shape) != (E, C, H, W) or d.dtype != dtype or not d.is_contiguous(memory_format=torch.channels_last) or d.data_ptr() % 16:
                raise ValueError("cache_load: entry %d: destinations must be channels-last %s [E, C, H, W] buffers, 16-byte aligned" % (k, dtype))
        e = CacheLoadEntry()
        e.src, e.src_dtype, e.src_layout, e.src_batch = src.data_ptr(), _dt(src), lo, int(src.shape[0])
        e.C, e.H, e.W, e.E = C, H, W, E
        e.raw = None if raw is None else raw.data_ptr()
        e.n_views = len(views)
        for i, (dst, sc, sh, act) in enumerate(views):
            for v in (sc, sh):
                if v is not None and (v.dtype != torch.float32 or v.numel() != C or not v.is_contiguous()):
                    raise ValueError("cache_load: entry %d: view %d: scale / shift must be contiguous fp32 [C]" % (k, i))
            ev = e.view[i]
            ev.dst, ev.act = dst.data_ptr(), _act(act)
            ev.scale = None if sc is None else sc.data_ptr()
            ev.shift = None if sh is None else sh.data_ptr()
        dev = dev or src.device
        rows.append(e)
        keep.append((src, raw, views))
    tables = []
    for s in range(0, len(rows), CACHE_LOAD_MAX_ENTRIES):
        part = rows[s:s + CACHE_LOAD_MAX_ENTRIES]
        tables.append(((CacheLoadEntry * len(part))(*part), len(part)))
    dt = _DTYPES[dtype]

    def run(stream: int) -> None:
        _ = keep
        for table, n in tables:
            with torch.cuda.device(dev):
                _cabi.check(_cabi.lib().sige_cache_load(table, n, dt, stream), "sige_cache_load")
            _bump()

    return run


def cache_load(entries, dtype: torch.dtype) -> None:
    """`cache_load_launcher(entries, dtype)` enqueued once on the current stream."""
    entries = list(entries)
    if entries:
        cache_load_launcher(entries, dtype)(_stream(entries[0][0]))


def tile_writeback(entries) -> None:
    """`tile_writeback_launcher(entries)` enqueued once on the current stream."""
    entries = list(entries)
    if entries:
        tile_writeback_launcher(entries)(_stream(entries[0][0]))
