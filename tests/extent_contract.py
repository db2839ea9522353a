"""Launches at the edges of the extents the C ABI accepts, checked against the existing float64 restatements.

sige_tile_conv accepts images of up to 65535 x 65535 pixels.  The cases here are narrow images at that limit — 65535 rows by
16 columns, or 16 rows by 65535 columns — with tiles placed where kernels go wrong: across row 32768 (the first row whose
index no longer fits 15 bits) and against the last row or column.  Each case is an mma_tile_conv_contract Spec whose tile list
is replaced by `edge_origins`; mma_tile_conv_contract.reference is the float64 restatement of the launch (it gathers only the
tiles, so a tall image costs no more than its buffers).

Imported by tests/test_gpu_extent_contracts.py and tests/test_gpu_extent_contracts_ops.py (and, for the host descriptor, by
tests/test_extent_limits.py).
"""
from __future__ import annotations

from dataclasses import dataclass, replace
from typing import List, Sequence, Tuple

import numpy as np
import torch

import kernel_contracts as kc
import mma_tile_conv_contract as mc
from tile_conv_contract import SWISH_LIP

LIMIT = 65535                   # largest H or W sige_tile_conv accepts
MID = 32768                     # first row / column whose index needs the 16th bit
NARROW = 16
GiB = 1 << 30
HOST_PTR = 0x10000              # a 16-byte aligned address that no host-side test dereferences


def need(nbytes: int, device) -> None:
    """Skip the calling test, with the amount it is short, when the device has less than `nbytes` free."""
    import pytest

    free, _ = torch.cuda.mem_get_info(device)
    if free < nbytes:
        pytest.skip("needs %.1f GiB of free device memory, %.1f GiB free (%.1f GiB short)"
                    % (nbytes / GiB, free / GiB, (nbytes - free) / GiB))


def host_tile_conv(cin=128, cout=256, k=3, N=16):
    """A wgmma-eligible sige_tile_conv_t (SIGE_CONV_TC5, 3x3 on 6x6 tiles or 1x1 on 4x4) on a 64 x 64 image whose pointers are
    not device memory: only the plan and the host checks may look at it."""
    from sige_b200 import _cabi

    d = _cabi.TileConv()
    d.dtype = _cabi.F16
    d.n_src, d.src[0].ptr, d.src[0].C = 1, HOST_PTR, cin
    d.B, d.H, d.W, d.idx, d.N = 1, 64, 64, HOST_PTR, N
    d.R = d.S = 6 if k == 3 else 4
    d.w_packed, d.bias = HOST_PTR, HOST_PTR
    d.Cin, d.Cout, d.kH, d.kW, d.stride = cin, cout, k, k, 1
    d.dst, d.dH, d.dW, d.dC = HOST_PTR, 64, 64, cout
    d.offH = d.offW = 1 if k == 3 else 0
    d.flags = _cabi.CONV_TC5
    return d


def _c_div(a: int, b: int) -> int:
    q = abs(a) // b
    return q if a >= 0 else -q


def spread(targets: Sequence[int], R_long: int, R_short: int, off_long: int, off_short: int, stride: int, short_out: int, tall: bool,
           name: str = "") -> List[Tuple[int, int]]:
    """Tile origins (h, w) at the given origins along the long axis, spread over the bands of the regular grid along the short
    axis so that no two R_long x R_short footprints, at (off + origin) / stride (C division), share an output pixel.  Every
    target is placed (asserted)."""
    bands = [stride * R_short * j - off_short for j in range(-(-short_out // R_short))]
    used = {b: [] for b in bands}
    out = []
    for t in targets:
        o = _c_div(off_long + t, stride)
        for b in bands:
            if all(o + R_long <= lo or lo + R_long <= o for lo in used[b]):
                used[b].append(o)
                out.append((t, b) if tall else (b, t))
                break
        else:
            raise AssertionError("%s: no band left for origin %d" % (name, t))
    return out


def edge_origins(spec: mc.Spec, tall: bool, targets: Sequence[int]) -> List[Tuple[int, int]]:
    """`spread` for the output tiles of a tile-conv spec."""
    return spread(targets, spec.Ro if tall else spec.So, spec.So if tall else spec.Ro, spec.offs[0] if tall else spec.offs[1],
                  spec.offs[1] if tall else spec.offs[0], spec.stride, spec.dW if tall else spec.dH, tall, spec.name)


def targets(spec: mc.Spec, tall: bool) -> List[int]:
    """Origins along the long axis: the first grid tile, every origin whose halo crosses row (column) 32768 or ends on it, and
    every origin whose halo reaches the last row (column) or hangs past it."""
    n = spec.H if tall else spec.W
    R = spec.R if tall else spec.Sx
    first = -(spec.offs[0] if tall else spec.offs[1])
    return [first] + list(range(MID - R, MID + 3)) + list(range(n - R - 1, n))


def spec_at_edge(base: mc.Spec, tall: bool) -> mc.Spec:
    """`base` (written for a tall image) turned wide if asked; extents even where a source is read up-sampled."""
    up = any(u for _, u in base.srcs)
    long = LIMIT - 1 if up else LIMIT
    H, W = (long, NARROW) if tall else (NARROW, long)
    return replace(base, name="%s_%s" % (base.name, "tall" if tall else "wide"), H=H, W=W)


def make_edge_case(spec: mc.Spec, tall: bool, dtype: torch.dtype, device) -> mc.Case:
    """The seeded tensors of `spec` with the tile list replaced by the edge origins (one list shared by every image)."""
    org = edge_origins(spec, tall, targets(spec, tall))
    spec = replace(spec, counts=(len(org),))
    case = mc.make_case(spec, dtype, device)
    case.idx = torch.tensor(org, dtype=torch.int32, device=device)
    return case


def peak_bytes(spec: mc.Spec, dtype: torch.dtype) -> int:
    """A generous estimate of a case's peak device memory: its tensors, and the float64 expectation (want, bound, rounding), the
    snapshots and the comparison temporaries of every buffer it writes."""
    es = torch.empty((), dtype=dtype).element_size()
    px = spec.B * spec.H * spec.W
    src = px * spec.Cin * es * (2 if spec.mod else 1) + px * spec.Cin * 4
    dpx = spec.B * spec.dH * spec.dW
    writes = [spec.Cout + spec.dst[0]] if spec.dst is not None else []
    writes += [spec.Cout + a[0] for a in spec.aux]
    res = dpx * (spec.Cout + spec.residual[0]) * es if spec.residual else 0
    return src + res + sum(dpx * c * (4 * 8 + 6 * es + 2) for c in writes)


# ----------------------------------------------------------------------------------------------------------------------
# sige_tile_conv on one NHWC buffer of 2^31 elements or more (byte offsets past 2^32)
# ----------------------------------------------------------------------------------------------------------------------
BIG_C = 2048                    # channels per pixel of the big buffer: every operand is a channel window of it
CHUNK = 1 << 26                 # elements filled (and re-made for the comparison) at a time


@dataclass(frozen=True)
class BigSpec:
    """A 3x3 tile conv whose source window, destination, residual and aux destination are channel windows of one
    [1, H, W, BIG_C] buffer.  `path` is the kernel sige_tile_conv_plan must pick (1 wgmma, 0 mma.sync) with SIGE_CONV_TC5."""
    name: str
    H: int
    W: int
    src_c0: int
    dst_c0: int
    res_c0: int
    aux_c0: int
    path: int
    Cin: int = 1024
    Cout: int = 64
    tiles: int = 12
    seed: int = 0

    @property
    def elements(self):
        return self.H * self.W * BIG_C


BIG_CASES = [
    # 2^31 elements: past the wgmma kernel's 32-bit offsets, so the launch goes to mma.sync; the destination starts at channel
    # 1024, the aux destination holds the last 64 channels
    BigSpec("window_2_31", H=1024, W=1024, src_c0=0, dst_c0=1024, res_c0=1088, aux_c0=BIG_C - 64, path=0, seed=401),
    # 2^31 - 2048 elements: the wgmma kernel.  The source is the top 1024 channels, so the bottom-right tile reads the buffer's
    # last element, the highest offset the 32-bit path may reach
    BigSpec("window_below_2_31", H=1025, W=1023, src_c0=1024, dst_c0=0, res_c0=64, aux_c0=128, path=1, seed=402),
]


def _chunk(flat: torch.Tensor, k: int, seed: int) -> torch.Tensor:
    i0 = k * CHUNK
    g = torch.Generator(device=flat.device)
    g.manual_seed(seed * 100003 + k)
    return torch.randn(min(CHUNK, flat.numel() - i0), generator=g, device=flat.device, dtype=flat.dtype)


def fill(flat: torch.Tensor, seed: int) -> None:
    """Seeded contents, made chunk by chunk so that `changed` can re-make them instead of keeping a copy."""
    for k in range(-(-flat.numel() // CHUNK)):
        flat[k * CHUNK:(k + 1) * CHUNK].copy_(_chunk(flat, k, seed))


def changed(flat: torch.Tensor, seed: int) -> torch.Tensor:
    """Indices of the elements of `flat` that differ bitwise from what `fill` put there."""
    out = []
    for k in range(-(-flat.numel() // CHUNK)):
        part = flat[k * CHUNK:(k + 1) * CHUNK]
        out.append((kc.bits(part) != kc.bits(_chunk(flat, k, seed))).nonzero()[:, 0] + k * CHUNK)
    return torch.cat(out)


@dataclass
class BigCase:
    spec: BigSpec
    flat: torch.Tensor
    case: mc.Case               # the source window, tile list, weights, bias and residual as the float64 restatement reads them
    aux_scale: torch.Tensor
    aux_shift: torch.Tensor


def make_big_case(bs: BigSpec, dtype: torch.dtype, device) -> BigCase:
    gen = torch.Generator(device=device)
    gen.manual_seed(bs.seed)
    flat = torch.empty(bs.elements, dtype=dtype, device=device)
    fill(flat, bs.seed)
    buf = flat.view(1, bs.H, bs.W, BIG_C)
    spec = mc.Spec(bs.name, B=1, H=bs.H, W=bs.W, srcs=((bs.Cin, 0),), Cout=bs.Cout, counts=(bs.tiles,), R=6,
                   window=(BIG_C - bs.Cin, bs.src_c0), residual=(BIG_C - bs.Cout, bs.res_c0), seed=bs.seed)
    idx = torch.tensor(mc.tile_lists(spec, np.random.default_rng(bs.seed))[0], dtype=torch.int32, device=device)
    w = (torch.randn(bs.Cout, bs.Cin, 3, 3, generator=gen, device=device) * (9 * bs.Cin) ** -0.5).to(dtype)
    bias = torch.randn(bs.Cout, generator=gen, device=device)
    case = mc.Case(spec, dtype, [buf[..., bs.src_c0:bs.src_c0 + bs.Cin]], [buf], idx, None, None, w, bias, None, buf, [])
    if torch.device(device).type == "cuda":
        from sige_b200 import ops

        case.wp = ops.pack_conv_weight(w, dtype)
    scale = (1 + 0.3 * torch.randn(bs.Cout, generator=gen, device=device)).float()
    shift = (0.3 * torch.randn(bs.Cout, generator=gen, device=device)).float()
    return BigCase(bs, flat, case, scale, shift)


def big_descriptor(bc: BigCase):
    """SIGE_CONV_TC5 descriptor: the size of the source decides the kernel."""
    from sige_b200 import _cabi

    bs = bc.spec
    d = mc.descriptor(bc.case, 0, _cabi.CONV_TC5)
    assert d.src_pixel_stride == BIG_C and d.rC == BIG_C and d.res_c0 == bs.res_c0
    d.dst, d.dC, d.dst_c0 = bc.flat.data_ptr(), BIG_C, bs.dst_c0
    d.n_aux = 1
    d.aux[0].ptr, d.aux[0].C, d.aux[0].c0, d.aux[0].act = bc.flat.data_ptr(), BIG_C, bs.aux_c0, 1
    d.aux[0].scale, d.aux[0].shift = bc.aux_scale.data_ptr(), bc.aux_shift.data_ptr()
    d._keep = bc
    return d


def big_reference(bc: BigCase):
    """(element indices, want, bound) of every element the launch writes (destination, then aux), in float64."""
    bs = bc.spec
    u = kc.ROUNDOFF[bc.case.dtype]
    v, bound, OB, OH, OW, ok = mc.tile_values(bc.case)
    px = ((OB[ok] * bs.H + OH[ok]) * bs.W + OW[ok]) * BIG_C                  # [K] first element of each written pixel
    assert px.unique().numel() == px.numel(), "%s: two tiles write the same output pixel" % bs.name
    ch = torch.arange(bs.Cout, device=px.device)
    sc, sh = bc.aux_scale.double(), bc.aux_shift.double()
    av = mc._act(v * sc + sh, 1)
    idx = torch.cat([(px[:, None] + bs.dst_c0 + ch).reshape(-1), (px[:, None] + bs.aux_c0 + ch).reshape(-1)])
    want = torch.cat([v[ok].reshape(-1), av[ok].reshape(-1)])
    bnd = torch.cat([bound[ok].reshape(-1), (SWISH_LIP * sc.abs() * bound + u * av.abs())[ok].reshape(-1)])
    return idx, want, bnd


def big_check(label: str, bc: BigCase, idx: torch.Tensor, want: torch.Tensor, bound: torch.Tensor) -> float:
    """The written elements within their bound, every other element of the buffer (the source and residual windows
    included) bitwise as `fill` left it.  Returns the worst error / bound ratio."""
    stray = changed(bc.flat, bc.spec.seed)
    stray = stray[~torch.isin(stray, idx)]
    if stray.numel():
        i = int(stray[0])
        raise AssertionError("%s: %d elements changed outside the written set, the first at pixel %d channel %d"
                             % (label, stray.numel(), i // BIG_C, i % BIG_C))
    err = (bc.flat[idx].double() - want).abs()
    ratio = torch.nan_to_num(torch.where(err == 0, torch.zeros_like(err), err / bound), nan=float("inf"))
    r = float(ratio.max())
    if r > 1.0:
        k = int(ratio.argmax())
        i = int(idx[k])
        raise AssertionError("%s: pixel %d channel %d: got %r, want %r, |err| %.3g > bound %.3g; %d elements over"
                             % (label, i // BIG_C, i % BIG_C, float(bc.flat[i]), float(want[k]), float(err[k]), float(bound[k]),
                                int((ratio > 1).sum())))
    return r


# ----------------------------------------------------------------------------------------------------------------------
# the tile ops, the stem, the GroupNorm fold and conv_out on 65535 x 16 and 16 x 65535 images
# ----------------------------------------------------------------------------------------------------------------------
def paste_targets(n: int, R: int, off: int, stride: int) -> List[int]:
    """Origins along an axis of n output pixels whose R-pixel footprints at (off + origin) / stride (C division) hang out
    before the first pixel, cross pixel 32768 or end on it, and reach the last pixel or hang out past it."""
    first = -off - stride
    mid = range(MID * stride - off - R * stride, MID * stride - off + 3)
    end = range((n - R) * stride - off - 1, n * stride - off)
    return [first] + list(mid) + list(end)


def edge_extent(tall: bool, even: bool = False) -> Tuple[int, int]:
    long = LIMIT - 1 if even else LIMIT
    return (long, NARROW) if tall else (NARROW, long)


def tile_op_origins(spec, tall: bool) -> dict:
    """Tile lists for a step_kernel_contracts.TileSpec on an edge image: gather tiles at every target, cycling over the
    columns (rows) of the short axis, one of them hanging out; pasted and calibration tiles `spread` so none overlap."""
    n, short = (spec.H, spec.W) if tall else (spec.W, spec.H)
    if spec.op == "gather":
        ts = paste_targets(n, 6, 0, 1)
        cols = [-5, 0, short - 6, short - 1, 5]
        return {"idx": [(t, cols[i % len(cols)]) if tall else (cols[i % len(cols)], t) for i, t in enumerate(ts)]}
    if spec.op == "scatter_gather":
        Ro, off, stride = 4, 1, 1
    else:
        (Ro, off), stride = spec.geometry, spec.stride
    out = {"idx": spread(paste_targets(n, Ro, off, stride), Ro, Ro, off, off, stride, short, tall, spec.name)}
    if spec.op == "swbr":
        out["idx1"] = spread(paste_targets(n, 4, 0, 1), 4, 4, 0, 0, 1, short, tall, spec.name)
    return out


def stem_tile_origins(H: int, W: int, R: int, tall: bool) -> List[Tuple[int, int]]:
    """R x R stem tiles at every target along the long axis, cycling over the short axis (the stem allows overlaps)."""
    n, short = (H, W) if tall else (W, H)
    cols = [-(R - 1), 0, short - R, short - 1]
    return [(t, cols[i % len(cols)]) if tall else (cols[i % len(cols)], t) for i, t in enumerate(paste_targets(n, R, 0, 1))]


# ----------------------------------------------------------------------------------------------------------------------
# pure moves (gather, scatter, write-back) on buffers of 2^31 elements or more, checked bitwise
# ----------------------------------------------------------------------------------------------------------------------
def tile_pixels(origins: Sequence[Tuple[int, int]], R: int, off: int, stride: int, H: int, W: int):
    """Per tile n, the in-image pixels of its R x R footprint at (off + origin) / stride (C division): lists of
    (n, row in tile, column in tile, image row, image column) as long tensors (on the CPU)."""
    out = []
    for n, (h, w) in enumerate(origins):
        h0, w0 = _c_div(off + h, stride), _c_div(off + w, stride)
        for r in range(R):
            for s in range(R):
                if 0 <= h0 + r < H and 0 <= w0 + s < W:
                    out.append((n, r, s, h0 + r, w0 + s))
    return torch.tensor(out, dtype=torch.long).unbind(1)


def nchw_offsets(C: int, H: int, W: int, b, h, w) -> torch.Tensor:
    """[K, C] element offsets of the pixels (b, h, w) [K] of an NCHW [B, C, H, W] tensor."""
    c = torch.arange(C, device=h.device)
    return ((b[:, None] * C + c) * H + h[:, None]) * W + w[:, None]


def nhwc_offsets(C: int, H: int, W: int, b, h, w) -> torch.Tensor:
    c = torch.arange(C, device=h.device)
    return ((b[:, None] * H + h[:, None]) * W + w[:, None]) * C + c


def moved_check(label: str, flat: torch.Tensor, seed: int, idx: torch.Tensor, want: torch.Tensor) -> None:
    """Every element of `flat` outside `idx` bitwise as `fill` left it; the elements at `idx` bitwise equal to `want`."""
    idx, want = idx.reshape(-1), want.reshape(-1).to(flat.dtype)
    stray = changed(flat, seed)
    stray = stray[~torch.isin(stray, idx)]
    if stray.numel():
        raise AssertionError("%s: %d elements changed outside the written set, the first at element %d"
                             % (label, stray.numel(), int(stray[0])))
    got = flat[idx]
    bad = kc.bits(got) != kc.bits(want)
    if bool(bad.any()):
        k = int(bad.nonzero()[0])
        raise AssertionError("%s: element %d: got %r, want %r; %d elements differ"
                             % (label, int(idx[k]), float(got[k]), float(want[k]), int(bad.sum())))


def unchanged_outside(label: str, flat: torch.Tensor, seed: int, allowed) -> None:
    """Every element of `flat` for which `allowed(indices)` is False bitwise as `fill` left it, checked chunk by chunk (the
    written set may be too large to list)."""
    for k in range(-(-flat.numel() // CHUNK)):
        part = flat[k * CHUNK:(k + 1) * CHUNK]
        i = torch.arange(k * CHUNK, k * CHUNK + part.numel(), device=flat.device)
        stray = (kc.bits(part) != kc.bits(_chunk(flat, k, seed))) & ~allowed(i)
        if bool(stray.any()):
            raise AssertionError("%s: %d elements changed outside the written set, the first at element %d"
                                 % (label, int(stray.sum()), int(i[stray][0])))
