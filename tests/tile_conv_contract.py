"""The sige_tile_conv descriptor contract (include/sige_b200.h, sige_tile_conv_t), restated in float64.

Imported by tests/test_tile_conv_contract.py (CPU: the restatement against the C oracle, and the case table against the launch
plan) and tests/test_gpu_tile_conv_contract.py (GPU: every wgmma configuration against the restatement).

  * `Spec` describes one launch in numbers; `make_case(spec, dtype, device)` turns it into a `Case` of tensors (seeded).
  * `descriptor(case, ksplit, flags)` is the C descriptor of that launch (it keeps the tensors alive).
  * `reference(case)` computes, in float64, what the launch must leave in every buffer it may write, the mask of the elements
    it writes and the per-element error bound; `check(...)` applies the bound to the written elements and demands that
    every other element is bitwise unchanged.
  * `instantiation(...)` says which `tile_conv_tc5_kernel<T, BN, TAPS, DEEP, ASYNC, S2, DB>` a plan runs.

Buffers are plain contiguous NHWC tensors [B, H, W, C] (the kernels' layout), so indices are (b, h, w, c); failures report them
as (b, c, h, w) like the rest of the suite.
"""
from __future__ import annotations

from ctypes import byref
from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

TILE_NONE = -30000
TC5, PDL, PADDED = 2, 1, 4

# ---- error bound of one written element (see check()) -----------------------------------------------------------------
# |got - want| <= u*|want| + ACC*mag + [pre-op] PRE_ULPS*u*max|w[co]|*max|a| + ABS
#   u        unit roundoff of the launch dtype: the output is rounded once from fp32.
#   ACC      fp32 accumulation (wgmma / mma.sync, any split-K order) relative to mag = the same conv on |operands|.  An
#            estimate (about 2^-24 per add, with the error of K ~ 10^3 products growing like a random walk); the worst
#            error / bound ratio per launch is printed, so the headroom measured on the H100 is on record.  Measured on an
#            H100 80GB HBM3 at a 400 W power limit: over the 232 launches the GPU sweep checks, the error beyond each element's
#            own rounding used at most 0.071 of the rest of the bound.
#   PRE_ULPS the kernel stages its pre-op result act(x*scale + shift) in 16 bits from fp32 arithmetic (swish with __expf and
#            __fdividef); up to four staged operands per output may round to the neighbouring 16-bit value of the float64
#            result, one ulp = 2u relative each.
#   ABS      absolute floor for outputs that cancel to ~0.
# Aux outputs act(v*scale + shift): the same bound scaled by |scale| (swish is at most 1.1-Lipschitz), plus u*|aux| for their
# own rounding.
UNIT_ROUNDOFF = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8, torch.float32: 2.0 ** -24}
ACC = 2.0 ** -18
PRE_ULPS = 8
ABS = 1e-6
SWISH_LIP = 1.1

DTYPE_NAME = {torch.float16: "f16", torch.bfloat16: "bf16"}


# ----------------------------------------------------------------------------------------------------------------------
# case table
# ----------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Spec:
    """One launch in numbers.  Geometry: k = 3 (6x6 halo tiles, offset 1), k = 1 (4x4 tiles, offset 0) or k = 3 with stride 2
    (5x5 tiles, offset 0, output origin (off + idx) / 2 in C division)."""
    name: str
    B: int
    H: int
    W: int
    srcs: Tuple[Tuple[int, int], ...]          # (channels, up) per source segment
    Cout: int
    counts: Tuple[int, ...]                    # real tiles per image; one entry = one list shared by every image
    k: int = 3
    stride: int = 1
    per_image: bool = False
    pad_to: int = 0                            # list length per image with SIGE_TILE_NONE padding (0: the longest count)
    preop: Optional[str] = None                # None, "shared" or "per_sample" affine
    act: int = 0                               # pre-op activation (sige_act_t)
    bias: bool = True
    dst: Optional[Tuple[int, int]] = (0, 0)    # (extra channels, dst_c0); None = aux-only launch
    residual: Optional[Tuple[int, int]] = None # (extra channels, res_c0)
    aux: Tuple[Tuple[int, int, bool, int], ...] = ()   # (extra channels, c0, affine, act) per aux destination
    shortcut: Tuple[int, ...] = ()             # channels of the fused 1x1 shortcut's source segments
    sc_flags: bool = False                     # per-tile shortcut flags (else NULL: every tile)
    padded: bool = False                       # SIGE_CONV_PADDED
    c_div_tile: bool = False                   # replace the (0, 0) corner tile of image 0 by (-1, -1) (stride 2 only)
    ksplits: Tuple[int, ...] = (0,)
    # intended plan per entry of ksplits: (BN, effective ksplit, double-buffered halo); None = the mma.sync kernel
    expect: Tuple[Optional[Tuple[int, int, int]], ...] = ()
    seed: int = 0

    @property
    def R(self):
        return 5 if self.stride == 2 else (6 if self.k == 3 else 4)

    @property
    def off(self):
        return 1 if (self.k == 3 and self.stride == 1) else 0

    @property
    def Ro(self):
        return (self.R - self.k) // self.stride + 1

    @property
    def dH(self):
        return self.H if self.stride == 1 else (self.H + 1 - 3) // 2 + 1

    @property
    def dW(self):
        return self.W if self.stride == 1 else (self.W + 1 - 3) // 2 + 1

    @property
    def Cin(self):
        return sum(c for c, _ in self.srcs)

    @property
    def Cin2(self):
        return sum(self.shortcut)

    @property
    def N(self):
        return max(max(self.counts), self.pad_to)

    @property
    def copy_gather(self):
        return self.preop is None and self.act == 0


W = (128, 1, 0)          # wide tiles, never split
CASES = [
    # ---- BN = 128 (m_blocks * Cout/128 >= 132: wide on any H100) ----
    Spec("W1", B=2, H=90, W=90, srcs=((128, 0), (64, 0)), Cout=256, counts=(300,), preop="per_sample", act=1, residual=(0, 0),
         aux=((0, 0, True, 1), (0, 0, False, 0)), ksplits=(0, 1, 8), expect=(W, W, W), seed=1),
    Spec("W2", B=1, H=100, W=100, srcs=((128, 1), (128, 0)), Cout=256, counts=(560,), residual=(0, 0), shortcut=(64, 128),
         sc_flags=True, ksplits=(0, 2), expect=(W, W), seed=2),
    Spec("W3", B=3, H=78, W=78, srcs=((256, 0),), Cout=128, counts=(360, 290, 201), per_image=True, preop="shared", act=1,
         shortcut=(128,), ksplits=(0, 4), expect=(W, W), seed=3),
    Spec("W4", B=1, H=74, W=74, k=1, srcs=((256, 0),), Cout=512, counts=(300,), preop="shared", act=0, dst=(64, 64),
         residual=(128, 128), aux=((8, 8, True, 1),), ksplits=(0, 2), expect=(W, W), seed=4),
    Spec("W5", B=1, H=82, W=82, k=1, srcs=((128, 0),), Cout=256, counts=(380,), pad_to=560, padded=True, dst=None,
         aux=((0, 0, True, 1),), ksplits=(0,), expect=(W,), seed=5),
    # ---- BN = 64 (m_blocks * Cout/64 <= 100: narrow on any H100) ----
    Spec("N1", B=2, H=46, W=46, srcs=((64, 1),), Cout=128, counts=(100, 70), per_image=True, preop="per_sample", act=1,
         residual=(0, 0), ksplits=(0, 1, 2), expect=((64, 2, 0), (64, 1, 0), (64, 2, 0)), seed=6),
    Spec("N2", B=1, H=62, W=62, srcs=((256, 0),), Cout=64, counts=(203,), pad_to=232, padded=True, ksplits=(1, 2, 8),
         expect=((64, 1, 0), (64, 2, 1), (64, 8, 0)), seed=7),
    Spec("N3", B=1, H=54, W=54, srcs=((256, 0),), Cout=256, counts=(150,), preop="shared", act=1, shortcut=(128, 128),
         aux=((0, 0, True, 1), (0, 0, False, 0)), ksplits=(2, 4, 8), expect=((64, 2, 1), (64, 4, 1), (64, 8, 1)), seed=8),
    Spec("N3s", B=3, H=42, W=42, srcs=((64, 0),), Cout=128, counts=(90, 60, 41), per_image=True, preop="per_sample", act=1,
         residual=(0, 0), shortcut=(64,), sc_flags=True, ksplits=(4,), expect=((64, 4, 0),), seed=9),
    Spec("N3p", B=1, H=42, W=42, srcs=((128, 0),), Cout=128, counts=(100,), preop="shared", act=1, ksplits=(4,),
         expect=((64, 4, 0),), seed=10),
    Spec("N4", B=1, H=46, W=46, srcs=((128, 0), (256, 0)), Cout=192, counts=(120,), dst=(72, 72), residual=(8, 8),
         ksplits=(4, 8), expect=((64, 4, 1), (64, 8, 1)), seed=11),
    Spec("N5r", B=2, H=50, W=50, k=1, srcs=((384, 0),), Cout=128, counts=(150, 110), per_image=True, preop="per_sample", act=1,
         residual=(0, 0), ksplits=(1, 2, 4), expect=((64, 1, 0), (64, 2, 0), (64, 4, 0)), seed=12),
    Spec("N5c", B=2, H=50, W=50, k=1, srcs=((384, 0),), Cout=128, counts=(150, 110), per_image=True, dst=None,
         aux=((16, 8, True, 1),), ksplits=(1, 2, 4), expect=((64, 1, 0), (64, 2, 0), (64, 4, 0)), seed=13),
    Spec("S1", B=2, H=34, W=30, stride=2, srcs=((64, 0), (64, 0)), Cout=128, counts=(60, 45), per_image=True, residual=(0, 0),
         c_div_tile=True, ksplits=(1, 2, 4), expect=((64, 1, 0), (64, 2, 0), (64, 4, 0)), seed=14),
    # stride 2 with a pre-op: not a wgmma geometry, the mma.sync kernel runs it
    Spec("S1p", B=2, H=34, W=30, stride=2, srcs=((64, 0), (64, 0)), Cout=128, counts=(60, 45), per_image=True, preop="shared",
         act=1, residual=(0, 0), c_div_tile=True, ksplits=(0, 2), expect=(None, None), seed=15),
]

# every kernel instantiation tc5_launch can reach: (dtype, BN, taps, S2, DEEP, DB, ASYNC)
ALL_INSTANTIATIONS = sorted(
    [(dt, 128, taps, 0, 0, 0, a) for dt in ("f16", "bf16") for taps in (9, 1) for a in (0, 1)]
    + [(dt, 64, 9, 0, deep, db, a) for dt in ("f16", "bf16") for (deep, db) in ((0, 0), (1, 0), (1, 1)) for a in (0, 1)]
    + [(dt, 64, 1, 0, 0, 0, a) for dt in ("f16", "bf16") for a in (0, 1)]
    + [(dt, 64, 9, 1, 0, 0, 1) for dt in ("f16", "bf16")]
)


def features(spec: Spec) -> set:
    """What a case exercises besides its kernel instantiation."""
    f = set()
    if spec.preop == "per_sample":
        f.add("per_sample_affine")
    if spec.preop == "shared":
        f.add("shared_affine")
    if spec.residual is not None:
        f.add("residual")
    if len(spec.aux) == 2:
        f.add("two_aux")
    if spec.dst is None:
        f.add("aux_only")
    if spec.shortcut:
        f.add("shortcut_flags" if spec.sc_flags else "shortcut_all_tiles")
    if len(spec.shortcut) == 2:
        f.add("shortcut_two_sources")
    if any(up for _, up in spec.srcs):
        f.add("upsampled_source")
    if len(spec.srcs) == 2:
        f.add("two_sources")
    if (spec.dst is not None and spec.dst[1]) or (spec.residual is not None and spec.residual[1]) or any(a[1] for a in spec.aux):
        f.add("channel_windows")
    if spec.per_image:
        f.add("per_image_lists")
    if spec.padded:
        f.add("padded")
    if spec.stride == 2:
        f.add("stride2")
    return f


# ----------------------------------------------------------------------------------------------------------------------
# tensors
# ----------------------------------------------------------------------------------------------------------------------
@dataclass
class Aux:
    buf: torch.Tensor
    c0: int
    scale: Optional[torch.Tensor]
    shift: Optional[torch.Tensor]
    act: int


@dataclass
class Case:
    spec: Spec
    dtype: torch.dtype
    srcs: List[torch.Tensor]                   # NHWC [B, H >> up, W >> up, C]
    idx: torch.Tensor                          # int32 [N, 2] (shared) or [B*N, 2] (per image)
    scale: Optional[torch.Tensor]              # fp32 [B or 1, Cin]
    shift: Optional[torch.Tensor]
    w: torch.Tensor                            # OIHW, launch dtype
    bias: Optional[torch.Tensor]               # fp32 [Cout]
    dst: Optional[torch.Tensor]                # NHWC [B, dH, dW, dC]
    residual: Optional[torch.Tensor]
    aux: List[Aux]
    src2: List[torch.Tensor] = field(default_factory=list)
    w2: Optional[torch.Tensor] = None          # [Cout, Cin2, 1, 1]
    bias2: Optional[torch.Tensor] = None
    sc_flags: Optional[torch.Tensor] = None    # uint8, one per idx row
    wp: Optional[torch.Tensor] = None          # packed weights (device cases)
    wp2: Optional[torch.Tensor] = None

    def buffers(self):
        """name -> every buffer the launch may write."""
        out = {}
        if self.dst is not None:
            out["dst"] = self.dst
        for i, a in enumerate(self.aux):
            out["aux%d" % i] = a.buf
        return out


def candidate_origins(spec: Spec):
    """Tile origins of the regular grid that covers the output (the origins reduce_mask yields), per axis."""
    if spec.stride == 2:
        return [4 * i for i in range(-(-spec.dH // 2))], [4 * i for i in range(-(-spec.dW // 2))]
    return [4 * i - spec.off for i in range(-(-spec.H // 4))], [4 * i - spec.off for i in range(-(-spec.W // 4))]


def tile_lists(spec: Spec, rng: np.random.Generator):
    """Per image: `count` distinct grid origins, row-major, always with the four corner tiles (they overhang every border
    of the input, and the bottom / right ones of the output unless the extent is a multiple of 4)."""
    hs, ws = candidate_origins(spec)
    grid = [(h, w) for h in hs for w in ws]
    corners = {(hs[0], ws[0]), (hs[0], ws[-1]), (hs[-1], ws[0]), (hs[-1], ws[-1])}
    lists = []
    for b, n in enumerate(spec.counts):
        assert 4 <= n <= len(grid), (spec.name, n, len(grid))
        rest = [g for g in grid if g not in corners]
        pick = set(corners) | {rest[i] for i in rng.choice(len(rest), n - len(corners), replace=False)}
        tiles = sorted(pick)
        if spec.c_div_tile and b == 0:
            # origin (-1, -1): output origin (0 + -1) / 2 = 0 in C division (floor division would say -1), so the tile writes
            # outputs (0..1, 0..1) from input rows / columns -1..3
            tiles[tiles.index((0, 0))] = (-1, -1)
        lists.append(tiles)
    return lists


def make_case(spec: Spec, dtype: torch.dtype, device) -> Case:
    rng = np.random.default_rng(spec.seed)
    gen = torch.Generator(device=device)
    gen.manual_seed(spec.seed)

    def randn(*shape, scale=1.0, dt=dtype):
        return (torch.randn(*shape, generator=gen, device=device) * scale).to(dt)

    B, N = spec.B, spec.N
    lists = tile_lists(spec, rng)
    rows = []
    for tiles in lists:
        rows += tiles + [(TILE_NONE, TILE_NONE)] * (N - len(tiles))
    assert spec.per_image or len(lists) == 1
    idx = torch.tensor(rows, dtype=torch.int32).reshape(-1, 2).to(device)

    srcs = [randn(B, spec.H >> up, spec.W >> up, c) for c, up in spec.srcs]
    scale = shift = None
    if spec.preop:
        nb = B if spec.preop == "per_sample" else 1
        scale = (1 + 0.2 * torch.randn(nb, spec.Cin, generator=gen, device=device)).float()
        shift = (0.2 * torch.randn(nb, spec.Cin, generator=gen, device=device)).float()
    K = spec.Cin * spec.k * spec.k
    w = randn(spec.Cout, spec.Cin, spec.k, spec.k, scale=K ** -0.5)
    bias = randn(spec.Cout, dt=torch.float32) if spec.bias else None
    dst = None if spec.dst is None else randn(B, spec.dH, spec.dW, spec.Cout + spec.dst[0])
    residual = None if spec.residual is None else randn(B, spec.dH, spec.dW, spec.Cout + spec.residual[0])
    aux = []
    for extra, c0, affine, act in spec.aux:
        sc = (1 + 0.3 * torch.randn(spec.Cout, generator=gen, device=device)).float() if affine else None
        sh = (0.3 * torch.randn(spec.Cout, generator=gen, device=device)).float() if affine else None
        aux.append(Aux(randn(B, spec.dH, spec.dW, spec.Cout + extra), c0, sc, sh, act))
    case = Case(spec, dtype, srcs, idx, scale, shift, w, bias, dst, residual, aux)
    if spec.shortcut:
        case.src2 = [randn(B, spec.H, spec.W, c) for c in spec.shortcut]
        case.w2 = randn(spec.Cout, spec.Cin2, 1, 1, scale=spec.Cin2 ** -0.5)
        case.bias2 = randn(spec.Cout, dt=torch.float32)
        if spec.sc_flags:
            f = (rng.random(idx.shape[0]) < 0.5).astype(np.uint8)
            f[np.asarray(rows)[:, 0] == TILE_NONE] = 0
            f[0], f[1] = 1, 0
            case.sc_flags = torch.from_numpy(f).to(device)
    if torch.device(device).type == "cuda" and dtype in (torch.float16, torch.bfloat16):
        from sige_b200 import ops

        case.wp = ops.pack_conv_weight(w, dtype)
        if spec.shortcut:
            case.wp2 = ops.pack_conv_weight(case.w2, dtype)
    return case


# ----------------------------------------------------------------------------------------------------------------------
# the C descriptor and its plan
# ----------------------------------------------------------------------------------------------------------------------
def _ptr(t):
    return None if t is None else t.data_ptr()


def descriptor(case: Case, ksplit: int = 0, flags: int = TC5):
    """The sige_tile_conv_t of this case (generalises _fused_desc of test_gpu_conv.py); d._keep holds the tensors."""
    from sige_b200 import _cabi

    s = case.spec
    d = _cabi.TileConv()
    d.dtype = {torch.float16: _cabi.F16, torch.bfloat16: _cabi.BF16, torch.float32: _cabi.F32}[case.dtype]
    d.n_src = len(case.srcs)
    for i, (t, (c, up)) in enumerate(zip(case.srcs, s.srcs)):
        d.src[i].ptr, d.src[i].C, d.src[i].up = t.data_ptr(), c, up
    d.B, d.H, d.W = s.B, s.H, s.W
    d.src_is_stack = 0
    d.idx, d.N = case.idx.data_ptr(), s.N
    d.R = d.S = s.R
    d.scale, d.shift = _ptr(case.scale), _ptr(case.shift)
    d.affine_bstride = s.Cin if s.preop == "per_sample" else 0
    d.act = s.act
    d.w_packed, d.bias = _ptr(case.wp), _ptr(case.bias)
    d.Cin, d.Cout, d.kH, d.kW, d.stride = s.Cin, s.Cout, s.k, s.k, s.stride
    d.dst, d.dst_is_stack = _ptr(case.dst), 0
    d.dH, d.dW = s.dH, s.dW
    d.dC, d.dst_c0 = (0, 0) if case.dst is None else (case.dst.shape[3], s.dst[1])
    d.offH = d.offW = s.off
    d.residual = _ptr(case.residual)
    d.rC, d.res_c0 = (0, 0) if case.residual is None else (case.residual.shape[3], s.residual[1])
    d.ksplit, d.flags = ksplit, flags
    d.n_aux = len(case.aux)
    for i, a in enumerate(case.aux):
        d.aux[i].ptr, d.aux[i].C, d.aux[i].c0 = a.buf.data_ptr(), a.buf.shape[3], a.c0
        d.aux[i].scale, d.aux[i].shift, d.aux[i].act = _ptr(a.scale), _ptr(a.shift), a.act
    d.n_src2 = len(case.src2)
    for i, t in enumerate(case.src2):
        d.src2[i].ptr, d.src2[i].C, d.src2[i].up = t.data_ptr(), t.shape[3], 0
    d.Cin2 = s.Cin2
    d.w2_packed, d.bias2, d.sc_flags = _ptr(case.wp2), _ptr(case.bias2), _ptr(case.sc_flags)
    d.idx_per_image = 1 if s.per_image else 0
    d._keep = case
    return d


def plan_of(d):
    from sige_b200 import _cabi

    p = _cabi.TileConvPlan()
    _cabi.check(_cabi.lib().sige_tile_conv_plan(byref(d), byref(p)), "sige_tile_conv_plan")
    return p


def k_slice(J, kr, ks):
    return (J * kr) // ks


def split_halo_fills(Cin, Cin2, ks):
    """Halo fills of the longest K slice of a split narrow 3x3 launch: the kernel's k_slice / chunk_of partition (ring steps
    of three taps per main 64-channel chunk, then one step per shortcut chunk), restated."""
    NC = Cin // 64
    J_main = 3 * NC
    J = J_main + Cin2 // 64

    def chunk_of(j):
        return j // 3 if j < J_main else NC + (j - J_main)

    most = 0
    for kr in range(ks):
        b, e = k_slice(J, kr, ks), k_slice(J, kr + 1, ks)
        if e > b:
            most = max(most, chunk_of(e - 1) - chunk_of(b) + 1)
    return most


def instantiation(spec: Spec, dtype: torch.dtype, plan):
    """(dtype, BN, taps, S2, DEEP, DB, ASYNC) of the wgmma kernel this plan launches (default halo layout), or None when the
    mma.sync kernel runs."""
    if plan.path != 1:
        return None
    s2 = 1 if spec.stride == 2 else 0
    db = 1 if (plan.deep_ring and split_halo_fills(spec.Cin, spec.Cin2, plan.ksplit) > 1) else 0
    return (DTYPE_NAME[dtype], plan.bn, spec.k * spec.k, s2, plan.deep_ring, db, 1 if spec.copy_gather else 0)


def intended(spec: Spec, dtype: torch.dtype, i: int):
    """The instantiation entry i of spec.expect stands for."""
    e = spec.expect[i]
    if e is None:
        return None
    bn, ks, db = e
    deep = 1 if (bn == 64 and spec.k == 3 and spec.stride == 1 and ks > 1) else 0
    return (DTYPE_NAME[dtype], bn, spec.k * spec.k, 1 if spec.stride == 2 else 0, deep, db, 1 if spec.copy_gather else 0)


def plan_str(plan):
    if plan.path != 1:
        return "mma.sync"
    return "wgmma bn=%d ksplit=%d deep=%d grid=%dx%dx%d" % (plan.bn, plan.ksplit, plan.deep_ring, plan.grid_x, plan.grid_y, plan.grid_z)


# ----------------------------------------------------------------------------------------------------------------------
# float64 reference
# ----------------------------------------------------------------------------------------------------------------------
@dataclass
class Expect:
    name: str
    want: torch.Tensor          # float64, the buffer's shape: the initial contents where nothing is written
    written: torch.Tensor       # bool
    mag: torch.Tensor           # float64: the same computation on |operands| (0 where not written)
    bound: torch.Tensor         # float64 per-element error bound (0 where not written)
    rounding: torch.Tensor      # the part of `bound` that is the element's own rounding to the launch dtype, u*|want|


def _gather(segs, org, img, R, H, W):
    """Halo tiles [NT, R, R, C] (float64) of the virtually concatenated / up-sampled NHWC segments at tile origins `org`
    ([NT, 2]) of images `img`, and the in-image mask [NT, R, R]."""
    d = torch.arange(R, device=org.device)
    hh, ww = org[:, :1] + d, org[:, 1:] + d                                  # [NT, R]
    valid = ((hh >= 0) & (hh < H))[:, :, None] & ((ww >= 0) & (ww < W))[:, None, :]
    parts = []
    for x, up in segs:
        hs, ws = hh.clamp(0, H - 1) >> up, ww.clamp(0, W - 1) >> up
        parts.append(x[img[:, None, None], hs[:, :, None], ws[:, None, :]].double())
    return torch.cat(parts, -1), valid


def _act(x, act):
    return x * torch.sigmoid(x) if act == 1 else x


def reference(case: Case) -> List[Expect]:
    s = case.spec
    dev = case.idx.device
    u = UNIT_ROUNDOFF[case.dtype]
    NT = s.B * s.N
    t = torch.arange(NT, device=dev)
    img = t // s.N
    row = t if s.per_image else t % s.N
    org = case.idx.long()[row]                                                # [NT, 2]

    # 1-3. gather halo tiles, pre-op in float64, rounded to the launch dtype (the kernel stages it in 16 bits), zero outside
    a, valid = _gather(list(zip(case.srcs, [up for _, up in s.srcs])), org, img, s.R, s.H, s.W)
    if s.preop:
        sel = img if s.preop == "per_sample" else torch.zeros_like(img)
        a = _act(a * case.scale.double()[sel][:, None, None, :] + case.shift.double()[sel][:, None, None, :], s.act)
        a = a.to(case.dtype).double()
    a = torch.where(valid[..., None], a, torch.zeros((), dtype=a.dtype, device=dev))
    # 4. conv + bias
    w = case.w.double()
    nchw = a.permute(0, 3, 1, 2)
    v = F.conv2d(nchw, w, stride=s.stride).permute(0, 2, 3, 1)               # [NT, Ro, Ro, Cout]
    mag = F.conv2d(nchw.abs(), w.abs(), stride=s.stride).permute(0, 2, 3, 1)
    pre = torch.zeros(s.Cout, dtype=torch.float64, device=dev)
    if s.preop:
        pre = PRE_ULPS * u * w.abs().amax(dim=(1, 2, 3)) * a.abs().max()
    if case.bias is not None:
        v = v + case.bias.double()
        mag = mag + case.bias.double().abs()
    # 6. output pixels: origin (off + idx) / stride in C division
    Ro = s.Ro
    base = torch.div(s.off + org, s.stride, rounding_mode="trunc") if s.stride == 2 else s.off + org
    d = torch.arange(Ro, device=dev)
    oh, ow = base[:, :1] + d, base[:, 1:] + d                                # [NT, Ro]
    out_ok = ((oh >= 0) & (oh < s.dH))[:, :, None] & ((ow >= 0) & (ow < s.dW))[:, None, :]
    OB = img[:, None, None].expand(NT, Ro, Ro)
    OH, OW = oh[:, :, None].expand(NT, Ro, Ro), ow[:, None, :].expand(NT, Ro, Ro)
    # 5. fresh 1x1 shortcut on flagged tiles, the residual (cached shortcut) elsewhere
    fresh = torch.zeros(NT, dtype=torch.bool, device=dev)
    if s.shortcut:
        fresh = torch.ones(NT, dtype=torch.bool, device=dev) if case.sc_flags is None else case.sc_flags[row] != 0
        x2, ok2 = _gather([(x, 0) for x in case.src2], org + 1, img, 4, s.H, s.W)
        x2 = torch.where(ok2[..., None], x2, torch.zeros((), dtype=x2.dtype, device=dev))
        w2 = case.w2.double()[:, :, 0, 0]
        f = fresh[:, None, None, None]
        v = v + torch.where(f, x2 @ w2.t() + case.bias2.double(), torch.zeros((), dtype=v.dtype, device=dev))
        mag = mag + torch.where(f, x2.abs() @ w2.abs().t() + case.bias2.double().abs(), torch.zeros((), dtype=v.dtype, device=dev))
    if case.residual is not None:
        c0 = s.residual[1]
        r = case.residual[OB, OH.clamp(0, s.dH - 1), OW.clamp(0, s.dW - 1)][..., c0:c0 + s.Cout].double()
        use = (~fresh)[:, None, None, None]
        v = v + torch.where(use, r, torch.zeros((), dtype=v.dtype, device=dev))
        mag = mag + torch.where(use, r.abs(), torch.zeros((), dtype=v.dtype, device=dev))

    bound = u * v.abs() + ACC * mag + pre + ABS
    ob, oh_, ow_ = OB[out_ok], OH[out_ok], OW[out_ok]
    lin = (ob * s.dH + oh_) * s.dW + ow_
    assert lin.unique().numel() == lin.numel(), "case %s: two tiles write the same output pixel" % s.name

    def scatter(buf, c0, val, mg, bd, name):
        want = buf.double().clone()
        written = torch.zeros(buf.shape, dtype=torch.bool, device=dev)
        m, b, rnd = (torch.zeros(buf.shape, dtype=torch.float64, device=dev) for _ in range(3))
        sl = slice(c0, c0 + s.Cout)
        want[ob, oh_, ow_, sl] = val[out_ok]
        written[ob, oh_, ow_, sl] = True
        m[ob, oh_, ow_, sl] = mg[out_ok]
        b[ob, oh_, ow_, sl] = bd[out_ok]
        rnd[ob, oh_, ow_, sl] = u * val[out_ok].abs()
        return Expect(name, want, written, m, b, rnd)

    out = []
    if case.dst is not None:
        out.append(scatter(case.dst, s.dst[1], v, mag, bound, "dst"))
    # 7. aux = act(v * scale + shift)
    for i, ax in enumerate(case.aux):
        sc = torch.ones(s.Cout, dtype=torch.float64, device=dev) if ax.scale is None else ax.scale.double()
        sh = torch.zeros(s.Cout, dtype=torch.float64, device=dev) if ax.shift is None else ax.shift.double()
        av = _act(v * sc + sh, ax.act)
        out.append(scatter(ax.buf, ax.c0, av, mag * sc.abs(), SWISH_LIP * sc.abs() * bound + u * av.abs(), "aux%d" % i))
    return out


def check(label: str, expects: List[Expect], got: dict, init: dict) -> Tuple[float, float]:
    """Every written element within its bound; every other element bitwise equal to the buffer's initial contents.

    Returns the worst error / bound ratio, and the worst ratio of what the error exceeds the element's own rounding by to
    the rest of the bound.  (A result rounded once from the exact value already reaches a ratio close to 1 wherever the
    value sits just above a power of two; the second ratio is the headroom of the accumulation and pre-op terms.)"""
    worst = excess = 0.0
    for e in expects:
        g, g0 = got[e.name], init[e.name]
        changed = g.view(torch.int16) != g0.view(torch.int16)
        stray = changed & ~e.written
        if bool(stray.any()):
            b, h, w, c = (int(z) for z in stray.nonzero()[0])
            raise AssertionError("%s: %s changed outside the written set at (b, c, h, w) = (%d, %d, %d, %d): %r -> %r (%d stray elements)"
                                 % (label, e.name, b, c, h, w, float(g0[b, h, w, c]), float(g[b, h, w, c]), int(stray.sum())))
        err = (g.double() - e.want).abs()
        ratio = torch.where(e.written, torch.nan_to_num(err / torch.where(e.written, e.bound, torch.ones_like(e.bound)), nan=float("inf")),
                            torch.zeros_like(err))
        r = float(ratio.max())
        if r > 1.0:
            b, h, w, c = (int(z) for z in (ratio == ratio.max()).nonzero()[0])
            raise AssertionError("%s: %s at (b, c, h, w) = (%d, %d, %d, %d): got %r, want %r, |err| %.3g > bound %.3g (mag %.3g); %d elements over"
                                 % (label, e.name, b, c, h, w, float(g[b, h, w, c]), float(e.want[b, h, w, c]), float(err[b, h, w, c]),
                                    float(e.bound[b, h, w, c]), float(e.mag[b, h, w, c]), int((ratio > 1).sum())))
        worst = max(worst, r)
        over = torch.where(e.written, (err - e.rounding).clamp(min=0) / (e.bound - e.rounding), torch.zeros_like(err))
        excess = max(excess, float(over.max()))
    return worst, excess
