"""The whole sige_tile_conv descriptor as the mma.sync kernel (sige_b200/csrc/tile_conv_mma.cu) runs it, restated in float64.

tests/tile_conv_contract.py describes the three wgmma geometries on full NHWC tensors; this module describes everything else the
descriptor allows: any R x S tile, any kH x kW, any stride and output offset, a stack or a full tensor on either side, Cout any
multiple of 8, a strided source window, SPADE modulation.  It shares tile_conv_contract's bound (UNIT_ROUNDOFF, ACC, PRE_ULPS, ABS,
SWISH_LIP) and kernel_contracts' guarded buffers and `check`: every buffer a launch may write is a window of a larger flat buffer
of random bytes, so a write one pixel or one channel vector past either end shows.

Imported by tests/test_mma_tile_conv_contract.py (CPU: the restatement against the C oracle and F.conv2d, the launch-plan
restatement against sige_tile_conv_plan, the case table's coverage) and tests/test_gpu_mma_tile_conv_contract.py (GPU).

  * `Spec` is one launch in numbers, `make_case` its seeded tensors, `descriptor` / `modulation` the C structs, `launch` the call.
  * `plan(...)` restates the host heuristic that picks the CTA configuration (L 128x128 / M 64x64 / S 32x64), the tiles per CTA,
    the K split and the grid; `plan_of(d)` is what the library reports for a descriptor.
  * `reference(case)` is what the launch must leave in every buffer it may write, with the written mask and per-element bound.
"""
from __future__ import annotations

from ctypes import byref, pointer
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

import kernel_contracts as kc
from tile_conv_contract import ABS, ACC, DTYPE_NAME, PADDED, PDL, PRE_ULPS, SWISH_LIP, TILE_NONE  # noqa: F401

H100_SMS = 132                  # what the library assumes when no device can be queried
KC = 64                         # channels per K chunk

# CTA configurations of tile_conv_mma_kernel: (GEMM rows BM, output channels BN, halo pixels one buffer holds)
CONFIGS = {"L": (128, 128, 288), "M": (64, 64, 144), "S": (32, 64, 72)}
ALL_INSTANTIATIONS = sorted((dt, cfg, mod) for dt in ("f16", "bf16") for cfg in CONFIGS for mod in (0, 1))


# ----------------------------------------------------------------------------------------------------------------------
# the launch plan, restated
# ----------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Plan:
    config: str
    tpc: int
    ksplit: int
    grid: Tuple[int, int, int]

    @property
    def bn(self):
        return CONFIGS[self.config][1]


def tiles_per_cta(config: str, P: int, RS: int) -> int:
    bm, _, halo = CONFIGS[config]
    return min(bm // P, halo // RS)


def plan(NT, R, S, kH, kW, stride, Cin, Cout, ksplit, sms=H100_SMS, force: Optional[str] = None) -> Optional[Plan]:
    """The plan of a launch the mma.sync kernel accepts; None when the tile fits no configuration.  ValueError: ksplit is not a
    cluster size.  `force` plans a given configuration instead of the heuristic's (to ask whether a case tells two apart)."""
    P, RS = ((R - kH) // stride + 1) * ((S - kW) // stride + 1), R * S

    def ctas(cfg):
        t = tiles_per_cta(cfg, P, RS)
        return -1 if t < 1 else -(-NT // t) * -(-Cout // CONFIGS[cfg][1])

    if ctas("L") < 0:
        return None
    J = -(-Cin // KC) * kH * kW
    if ksplit > J:
        ksplit = 1
    if ksplit not in (0, 1, 2, 4, 8):
        raise ValueError("ksplit must be 1, 2, 4 or 8")
    cL, cM, cS = ctas("L"), ctas("M"), ctas("S")
    if cL >= 2 * sms:
        cfg = "L"
    elif cM >= sms or cS < 0:
        cfg = "M" if cM > 0 else "L"
    else:
        cfg = "S"
    if force is not None:
        cfg = force
        if tiles_per_cta(cfg, P, RS) < 1:
            return None
    tpc = tiles_per_cta(cfg, P, RS)
    gx, gy = -(-NT // tpc), -(-Cout // CONFIGS[cfg][1])
    ks = ksplit
    if ks <= 0:
        ks = 1
        while ks < 8 and gx * gy * ks * 2 <= 2 * sms and J // (ks * 2) >= 4:
            ks *= 2
    return Plan(cfg, tpc, ks, (gx, gy, ks))


def ambiguous(p: Plan, NT, R, S, kH, kW, stride, Cin, Cout, ksplit, sms) -> List[str]:
    """The other configurations whose plan would report the same (bn, grid) — the library's plan could not tell them from p."""
    out = []
    for cfg in CONFIGS:
        if cfg == p.config:
            continue
        q = plan(NT, R, S, kH, kW, stride, Cin, Cout, ksplit, sms, force=cfg)
        if q is not None and (q.bn, q.grid) == (p.bn, p.grid):
            out.append(cfg)
    return out


# ----------------------------------------------------------------------------------------------------------------------
# case table
# ----------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Spec:
    """One launch in numbers.  Full tensors are NHWC [B, H, W, C] (source, logical extent; an up-sampled segment is stored at half
    of it) and [B, dH, dW, C] (destination side); stacks are [B*N, R, S, Cin] and [B*N, Ro, So, C].  Tile lists hold origins
    idx = stride * (Ro * i, So * j) - (offH, offW) of the regular grid that covers the output, so no two tiles write one pixel."""
    name: str
    B: int
    srcs: Tuple[Tuple[int, int], ...]          # (channels, up) per source segment
    Cout: int
    counts: Tuple[int, ...]                    # real tiles per image; one entry = one list shared by every image
    R: int
    k: Tuple[int, int] = (3, 3)                # kH, kW
    S: int = 0                                 # 0: R
    stride: int = 1
    off: Optional[Tuple[int, int]] = None      # offH, offW; None: ((kH - 1) // 2, (kW - 1) // 2) at stride 1, (0, 0) otherwise
    H: int = 0
    W: int = 0
    dHW: Optional[Tuple[int, int]] = None      # None: ceil(H / stride), ceil(W / stride)
    src_stack: bool = False
    dst_stack: bool = False
    per_image: bool = False
    pad_to: int = 0                            # list length per image with SIGE_TILE_NONE padding (0: the longest count)
    padded: bool = False                       # SIGE_CONV_PADDED
    preop: Optional[str] = None                # None, "shared" or "per_sample" affine
    act: int = 0                               # pre-op activation
    bias: bool = True
    dst: Optional[Tuple[int, int]] = (0, 0)    # (extra channels, dst_c0); None = aux-only launch
    residual: Optional[Tuple[int, int]] = None # (extra channels, res_c0)
    aux: Tuple[Tuple[int, int, bool, int], ...] = ()   # (extra channels, c0, affine, act) per aux destination
    mod: Optional[Tuple[int, int, int, int, float]] = None   # SPADE modulation: gamma (extra, c0), beta (extra, c0), slope
    window: Optional[Tuple[int, int]] = None   # src_pixel_stride: the source is channels [c0, c0 + Cin) of (extra + Cin)
    c_div_tile: bool = False                   # move the first grid tile of image 0 up / left by one pixel (stride 2)
    ksplits: Tuple[int, ...] = (0,)
    expect: str = "S"                          # the configuration the case is meant for
    single_cta: bool = False                   # fewer tiles than any configuration packs: one CTA per Cout block whichever runs
    seed: int = 0

    @property
    def kH(self):
        return self.k[0]

    @property
    def kW(self):
        return self.k[1]

    @property
    def Sx(self):
        return self.S or self.R

    @property
    def offs(self):
        if self.off is not None:
            return self.off
        return ((self.kH - 1) // 2, (self.kW - 1) // 2) if self.stride == 1 else (0, 0)

    @property
    def Ro(self):
        return (self.R - self.kH) // self.stride + 1

    @property
    def So(self):
        return (self.Sx - self.kW) // self.stride + 1

    @property
    def dH(self):
        return self.dHW[0] if self.dHW else -(-self.H // self.stride)

    @property
    def dW(self):
        return self.dHW[1] if self.dHW else -(-self.W // self.stride)

    @property
    def Cin(self):
        return sum(c for c, _ in self.srcs)

    @property
    def N(self):
        return max(max(self.counts), self.pad_to)

    @property
    def NT(self):
        return self.B * self.N

    def plan(self, ksplit, sms=H100_SMS, force=None):
        return plan(self.NT, self.R, self.Sx, self.kH, self.kW, self.stride, self.Cin, self.Cout, ksplit, sms, force)

    def ambiguous(self, p, ksplit, sms=H100_SMS):
        return ambiguous(p, self.NT, self.R, self.Sx, self.kH, self.kW, self.stride, self.Cin, self.Cout, ksplit, sms)


ALL_KS = (0, 1, 2, 4, 8)
CASES = [
    # ---- one case per branch of the selection (132 SMs; cL / cM / cS are the CTA counts of L / M / S) ----
    # cL >= 2 SMs: 6x6 / 3x3, P 16: L packs 8 tiles; 1200 tiles x Cout 136 = 150 x 2 CTAs.  A partial second Cout block of 8.
    Spec("L_fills", B=1, H=140, W=140, srcs=((64, 0),), Cout=136, counts=(1200,), R=6, residual=(0, 0), ksplits=(0, 2), expect="L", seed=101),
    # cM >= SMs, cL < 2 SMs: M packs 4 tiles, L 8: 600 tiles -> cM 150, cL 75
    Spec("M_fills", B=1, H=100, W=100, srcs=((64, 0),), Cout=64, counts=(600,), R=6, preop="shared", act=1, ksplits=(0, 1), expect="M", seed=102),
    # cS < 0 -> M: 10x10 / 3x3, P 64 > 32
    Spec("M_no_S", B=2, H=40, W=40, srcs=((40, 0),), Cout=72, counts=(9,), R=10, preop="per_sample", act=1, ksplits=ALL_KS, expect="M", seed=103),
    # cM <= 0 -> L: 12x12 / 3x3, P 100 > 64
    Spec("L_no_M", B=1, H=40, W=40, srcs=((96, 0),), Cout=200, counts=(7,), R=12, residual=(8, 8), dst=(8, 0), ksplits=ALL_KS, expect="L", seed=104),
    # ---- idle GEMM rows: BM % P != 0 ----
    Spec("S_5x5", B=1, H=30, W=28, srcs=((64, 0), (64, 1)), Cout=72, counts=(23,), R=5, ksplits=(0, 1, 2, 4), seed=105,
         aux=((8, 8, True, 1), (0, 0, False, 2)), residual=(0, 0)),                        # P 9: tpc min(3, 2) = 2 by the halo, NT odd
    Spec("S_7x7", B=2, H=32, W=32, srcs=((64, 0),), Cout=64, counts=(11,), R=7, preop="shared", ksplits=(0, 4), seed=106),   # P 25: tpc 1
    Spec("S_5x5_s2", B=1, H=40, W=40, srcs=((64, 0),), Cout=64, counts=(37,), R=5, stride=2, ksplits=(0, 2), seed=107, dHW=(20, 20),
         preop="shared", act=1, c_div_tile=True),                                          # P 4: tpc min(8, 2) = 2; the SD downsample
    Spec("S_7x7_s2", B=2, H=36, W=30, srcs=((64, 0),), Cout=64, counts=(14, 9), R=7, stride=2, per_image=True, ksplits=(0, 8), seed=108,
         c_div_tile=True, residual=(0, 0)),                                                # P 9: tpc 1
    Spec("M_7x7_idle", B=1, H=100, W=100, srcs=((64, 0),), Cout=64, counts=(300,), R=7, ksplits=(0,), expect="M", seed=109),   # P 25: tpc 2, 14 idle rows
    Spec("L_5x5_idle", B=1, H=150, W=150, srcs=((64, 0),), Cout=136, counts=(1700,), R=5, ksplits=(1,), expect="L", seed=110),  # P 9: tpc 11 by the halo, 29 idle rows
    # ---- few tiles ----
    # (a grid of one CTA looks the same under M and S: single_cta, see test_no_case_is_ambiguous)
    Spec("S_one_tile", B=1, H=8, W=8, srcs=((128, 0),), Cout=64, counts=(1,), R=6, ksplits=ALL_KS, single_cta=True, seed=111),
    Spec("S_rows4", B=1, H=4, W=4, srcs=((192, 0),), Cout=64, counts=(1,), R=4, ksplits=ALL_KS, single_cta=True, seed=112,
         dHW=(2, 2)),                                                                     # one 4x4 / 3x3 tile: 4 rows over 8 ranks
    Spec("S_fewer_than_tpc", B=1, H=12, W=12, srcs=((64, 0),), Cout=8, counts=(2,), R=3, k=(1, 1), ksplits=ALL_KS, single_cta=True,
         seed=113),                                                                       # 2 tiles, tpc 3; J = 1: every split falls back to 1
    # ---- non-square ----
    Spec("S_6x10", B=1, H=24, W=40, srcs=((64, 0),), Cout=72, counts=(13,), R=6, S=10, ksplits=(0, 2), seed=114, preop="shared", act=1),
    Spec("S_4x8_1x3", B=2, H=16, W=24, srcs=((48, 0),), Cout=64, counts=(9,), R=4, S=8, k=(1, 3), ksplits=(0, 1), seed=115),
    Spec("S_8x4_3x1", B=1, H=24, W=16, srcs=((64, 0),), Cout=64, counts=(10,), R=8, S=4, k=(3, 1), ksplits=(0, 2), seed=116),
    Spec("S_off_h_w", B=1, H=20, W=20, srcs=((64, 0),), Cout=64, counts=(12,), R=6, S=5, k=(3, 2), off=(1, 0), ksplits=(0,), seed=117),
    # ---- stacks ----
    Spec("stack_stack", B=1, srcs=((64, 0),), Cout=136, counts=(21,), R=6, src_stack=True, dst_stack=True, ksplits=(0, 2), seed=118),
    Spec("stack_stack_7", B=1, srcs=((24, 0),), Cout=8, counts=(5,), R=7, src_stack=True, dst_stack=True, preop="shared", act=1,
         residual=(0, 0), ksplits=(0,), seed=119),
    Spec("full_stack", B=2, H=24, W=24, srcs=((64, 0),), Cout=72, counts=(17,), R=6, dst_stack=True, dst=(8, 8), preop="per_sample",
         ksplits=(0, 4), seed=120),
    Spec("stack_full", B=2, H=24, W=24, srcs=((64, 0),), Cout=64, counts=(17,), R=6, src_stack=True, residual=(0, 0), preop="per_sample",
         act=1, ksplits=(0, 4), seed=121),
    Spec("full_stack_s2", B=1, H=30, W=30, srcs=((64, 0),), Cout=64, counts=(19,), R=5, stride=2, dst_stack=True, dHW=(15, 15),
         ksplits=(0,), seed=122),
    # ---- K splits: mid-chunk slice starts, narrow last chunks ----
    Spec("K_27_over_4", B=1, H=20, W=20, srcs=((192, 0),), Cout=64, counts=(14,), R=6, ksplits=ALL_KS, seed=123),             # 3 chunks x 9 taps
    Spec("K_cin40", B=1, H=20, W=20, srcs=((40, 0),), Cout=64, counts=(14,), R=6, ksplits=ALL_KS, seed=124),
    Spec("K_cin96", B=1, H=20, W=20, srcs=((96, 0),), Cout=64, counts=(14,), R=6, preop="shared", act=1, ksplits=ALL_KS, seed=125),
    Spec("K_cin200", B=1, H=20, W=20, srcs=((200, 0),), Cout=72, counts=(14,), R=6, ksplits=ALL_KS, seed=126),
    Spec("K_1x1_cin64", B=1, H=20, W=20, srcs=((64, 0),), Cout=64, counts=(20,), R=4, k=(1, 1), ksplits=ALL_KS, seed=127),    # J = 1: every split falls back to 1
    # ---- sources ----
    Spec("two_src_mixed_up", B=1, H=28, W=28, srcs=((64, 1), (128, 0)), Cout=64, counts=(30,), R=5, ksplits=(0, 4), seed=128,
         preop="shared", act=1),
    Spec("two_src_up_second", B=2, H=28, W=28, srcs=((128, 0), (64, 1)), Cout=64, counts=(20, 13), R=6, per_image=True,
         bias=False, ksplits=(0, 2), seed=129),
    Spec("window_5x5", B=1, H=25, W=25, srcs=((40, 0),), Cout=64, counts=(20,), R=5, window=(24, 16), ksplits=(0, 2), seed=130),
    Spec("window_up", B=2, H=24, W=24, srcs=((64, 1),), Cout=64, counts=(15,), R=7, window=(8, 8), preop="shared", ksplits=(0,), seed=131),
    # ---- stride 2 ----
    Spec("s2_preop_neg_origin", B=2, H=34, W=30, srcs=((64, 0), (64, 0)), Cout=72, counts=(30, 22), R=5, stride=2, per_image=True,
         dHW=(17, 15), preop="shared", act=1, residual=(0, 0), c_div_tile=True, ksplits=(0, 2), seed=132),
    Spec("sd_downsample", B=1, H=32, W=32, srcs=((128, 0),), Cout=128, counts=(40,), R=5, stride=2, dHW=(16, 16), ksplits=(0, 1), seed=133),
    # ---- padded lists ----
    Spec("padded_runs", B=1, H=40, W=40, srcs=((64, 0),), Cout=64, counts=(37,), pad_to=64, padded=True, R=6, ksplits=(0, 4), seed=134,
         residual=(0, 0)),                                                                 # 37 of 64 slots, S tpc 2: 13 CTAs of padding
    Spec("per_image_padding", B=3, H=24, W=24, srcs=((64, 0),), Cout=64, counts=(20, 9, 4), pad_to=24, per_image=True, R=5,
         ksplits=(0, 2), seed=135),
    # ---- epilogue ----
    Spec("aux_only", B=1, H=20, W=20, srcs=((64, 0),), Cout=72, counts=(16,), R=6, dst=None, aux=((16, 8, True, 2),), ksplits=(0, 2), seed=136),
    Spec("epilogue_windows", B=2, H=20, W=20, srcs=((64, 0),), Cout=200, counts=(16,), R=7, dst=(16, 8), residual=(24, 16),
         aux=((8, 0, True, 1), (16, 16, False, 2)), preop="per_sample", act=1, ksplits=(0, 4), seed=137),
    # ---- SPADE modulation (MOD instantiations) ----
    Spec("mod_S_5x5", B=1, H=25, W=25, srcs=((40, 0),), Cout=72, counts=(18,), R=5, mod=(16, 8, 8, 0, 0.2), preop="shared", ksplits=(0, 2), seed=138),
    Spec("mod_S_up_slope1", B=2, H=28, W=28, srcs=((64, 1),), Cout=64, counts=(12,), R=7, mod=(0, 0, 24, 16, 1.0), preop="per_sample",
         ksplits=(0, 4), seed=139),
    Spec("mod_M", B=1, H=40, W=40, srcs=((24, 0),), Cout=64, counts=(9,), R=10, mod=(8, 8, 0, 0, 0.2), ksplits=(0,), expect="M", seed=140,
         residual=(0, 0)),
    Spec("mod_M_fills", B=1, H=100, W=100, srcs=((64, 0),), Cout=64, counts=(600,), R=6, mod=(0, 0, 0, 0, 0.2), preop="shared", ksplits=(1,),
         expect="M", seed=141),
    Spec("mod_L", B=1, H=40, W=40, srcs=((64, 0),), Cout=136, counts=(7,), R=12, mod=(8, 0, 8, 8, 0.2), aux=((0, 0, False, 2),),
         ksplits=(0, 8), expect="L", seed=142),
    Spec("mod_s2", B=1, H=30, W=30, srcs=((64, 0),), Cout=64, counts=(25,), R=5, stride=2, dHW=(15, 15), mod=(0, 0, 0, 0, 0.2),
         ksplits=(0,), seed=143),
]


def features(spec: Spec) -> set:
    """What a case exercises besides its kernel instantiation."""
    f = set()
    P, RS = spec.Ro * spec.So, spec.R * spec.Sx
    bm, _, halo = CONFIGS[spec.expect]
    tpc = tiles_per_cta(spec.expect, P, RS)
    if bm > tpc * P:
        f.add("idle_rows")
    if P & (P - 1):
        f.add("non_pow2_pixels")
    if halo // RS < bm // P:
        f.add("tpc_by_halo")
    if spec.NT % tpc:
        f.add("partial_last_cta")
    if tpc > spec.NT:
        f.add("fewer_tiles_than_tpc")
    if spec.NT == 1:
        f.add("one_tile")
    if spec.R != spec.Sx:
        f.add("non_square_tile")
    if spec.kH != spec.kW:
        f.add("non_square_kernel")
    if spec.offs[0] != spec.offs[1]:
        f.add("off_h_ne_off_w")
    if spec.Cout % 64:
        f.add("partial_cout_block")
    f.add("src_%s_dst_%s" % ("stack" if spec.src_stack else "full", "stack" if spec.dst_stack else "full"))
    if (spec.src_stack or spec.dst_stack) and spec.B > 1:
        f.add("stack_batch")
    J = -(-spec.Cin // KC) * spec.kH * spec.kW
    for ks in spec.ksplits:
        if ks > 1:
            f.add("split_k")
            if ks > J:
                f.add("ksplit_gt_steps")
            elif spec.NT == 1 and ks > P:
                f.add("rows_lt_ksplit")
            if ks <= J and any((J * r // ks) % (spec.kH * spec.kW) for r in range(1, ks)) and J > spec.kH * spec.kW:
                f.add("mid_chunk_slice")
            if ks <= J and spec.Cin % KC and spec.Cin > KC:
                f.add("narrow_last_chunk_split")
    if spec.Cin % KC:
        f.add("narrow_cin")
    if len(spec.srcs) == 2:
        f.add("two_sources")
        if spec.srcs[0][1] != spec.srcs[1][1]:
            f.add("mixed_up")
    if any(up for _, up in spec.srcs):
        f.add("upsampled_source")
    if spec.window:
        f.add("strided_window")
    if spec.stride == 2:
        f.add("stride2")
        if spec.preop:
            f.add("stride2_preop")
        if spec.dst_stack:
            f.add("stride2_into_stack")
    if spec.c_div_tile:
        f.add("negative_origin")
    if spec.per_image:
        f.add("per_image_lists")
    if spec.N > min(spec.counts):
        f.add("tile_none_padding")
    if spec.padded:
        f.add("padded")
    if spec.preop == "shared":
        f.add("shared_affine")
    if spec.preop == "per_sample":
        f.add("per_sample_affine")
    if spec.act == 1:
        f.add("swish")
    if spec.mod:
        f.add("modulated")
        if spec.mod[0] or spec.mod[1] or spec.mod[2] or spec.mod[3]:
            f.add("gamma_beta_windows")
        f.add("slope1" if spec.mod[4] == 1.0 else "leaky")
        if spec.R % 2:
            f.add("modulated_odd_tile")
        if spec.Cin % KC:
            f.add("modulated_narrow_cin")
        if any(up for _, up in spec.srcs):
            f.add("modulated_upsampled")
    if spec.residual is not None:
        f.add("residual")
    if len(spec.aux) == 2:
        f.add("two_aux")
    if any(a[3] == 2 for a in spec.aux):
        f.add("aux_relu")
    if any(a[2] and a[3] == 1 for a in spec.aux):
        f.add("aux_affine_swish")
    if spec.dst is None:
        f.add("aux_only")
    if not spec.bias:
        f.add("no_bias")
    if (spec.dst is not None and (spec.dst[0] or spec.dst[1])) or (spec.residual is not None and spec.residual[1]) or any(a[0] or a[1] for a in spec.aux):
        f.add("channel_windows")
    return f


REQUIRED_FEATURES = {
    "idle_rows", "non_pow2_pixels", "tpc_by_halo", "partial_last_cta", "fewer_tiles_than_tpc", "one_tile", "non_square_tile",
    "non_square_kernel", "off_h_ne_off_w", "partial_cout_block", "src_stack_dst_stack", "src_full_dst_stack", "src_stack_dst_full",
    "src_full_dst_full", "stack_batch", "split_k", "ksplit_gt_steps", "rows_lt_ksplit", "mid_chunk_slice", "narrow_last_chunk_split",
    "narrow_cin", "two_sources", "mixed_up", "upsampled_source", "strided_window", "stride2", "stride2_preop", "stride2_into_stack",
    "negative_origin", "per_image_lists", "tile_none_padding", "padded", "shared_affine", "per_sample_affine", "swish", "modulated",
    "gamma_beta_windows", "slope1", "leaky", "modulated_odd_tile", "modulated_narrow_cin", "modulated_upsampled", "residual", "two_aux",
    "aux_relu", "aux_affine_swish", "aux_only", "no_bias", "channel_windows",
}


# ----------------------------------------------------------------------------------------------------------------------
# tensors
# ----------------------------------------------------------------------------------------------------------------------
@dataclass
class Aux:
    g: kc.Guarded
    c0: int
    scale: Optional[torch.Tensor]
    shift: Optional[torch.Tensor]
    act: int


@dataclass
class Case:
    spec: Spec
    dtype: torch.dtype
    srcs: List[torch.Tensor]                   # per segment: NHWC [B, H >> up, W >> up, C] or the stack; a view for a strided window
    src_bufs: List[torch.Tensor]               # the buffers the sources live in
    idx: Optional[torch.Tensor]                # int32 [N, 2] (shared) or [B*N, 2] (per image); None for stack -> stack
    scale: Optional[torch.Tensor]
    shift: Optional[torch.Tensor]
    w: torch.Tensor                            # OIHW, launch dtype
    bias: Optional[torch.Tensor]
    dst: Optional[kc.Guarded]
    residual: Optional[torch.Tensor]
    aux: List[Aux]
    gamma: Optional[torch.Tensor] = None       # NHWC [B, H, W, Cin + extra]
    beta: Optional[torch.Tensor] = None
    wp: Optional[torch.Tensor] = None          # packed weights (device cases)

    def buffers(self) -> Dict[str, kc.Guarded]:
        out = {}
        if self.dst is not None:
            out["dst"] = self.dst
        for i, a in enumerate(self.aux):
            out["aux%d" % i] = a.g
        return out

    def inputs(self) -> Dict[str, torch.Tensor]:
        out = {"src%d" % i: t for i, t in enumerate(self.src_bufs)}
        named = {"idx": self.idx, "scale": self.scale, "shift": self.shift, "bias": self.bias, "residual": self.residual,
                 "gamma": self.gamma, "beta": self.beta, "w_packed": self.wp}
        out.update({k: v for k, v in named.items() if v is not None})
        for i, a in enumerate(self.aux):
            if a.scale is not None:
                out["aux%d_scale" % i], out["aux%d_shift" % i] = a.scale, a.shift
        return out


def tile_lists(spec: Spec, rng: np.random.Generator):
    """Per image: `count` distinct origins of the output grid, row-major, always with the four corner tiles (they overhang the
    borders of the input, and the bottom / right ones those of the output unless the extent is a multiple of the tile)."""
    oh, ow = spec.offs
    hs = [spec.stride * spec.Ro * i - oh for i in range(-(-spec.dH // spec.Ro))]
    ws = [spec.stride * spec.So * i - ow for i in range(-(-spec.dW // spec.So))]
    grid = [(h, w) for h in hs for w in ws]
    corners = {(hs[0], ws[0]), (hs[0], ws[-1]), (hs[-1], ws[0]), (hs[-1], ws[-1])}
    lists = []
    for b, n in enumerate(spec.counts):
        assert n <= len(grid), (spec.name, n, len(grid))
        if n < len(corners):
            tiles = sorted(corners)[:n]
        else:
            rest = [g for g in grid if g not in corners]
            tiles = sorted(set(corners) | {rest[i] for i in rng.choice(len(rest), n - len(corners), replace=False)})
        if spec.c_div_tile and b == 0:
            # (off + idx) = -1 on both axes: output origin -1 / 2 = 0 in C division (floor division would say -1)
            assert spec.stride == 2 and spec.offs == (0, 0)
            tiles[tiles.index((0, 0))] = (-1, -1)
        lists.append(tiles)
    return lists


def make_case(spec: Spec, dtype: torch.dtype, device) -> Case:
    rng = np.random.default_rng(spec.seed)
    gen = torch.Generator(device=device)
    gen.manual_seed(spec.seed)

    def randn(*shape, scale=1.0, dt=dtype):
        return (torch.randn(*shape, generator=gen, device=device) * scale).to(dt)

    def writable(C):
        shape = (spec.NT, spec.Ro, spec.So, C) if spec.dst_stack else (spec.B, spec.dH, spec.dW, C)
        g = kc.guarded(shape, dtype, device, gen, "nhwc", lead_bytes=256, tail_bytes=272)
        g.view.copy_(randn(*shape))
        return g

    B, N = spec.B, spec.N
    idx = None
    if not (spec.src_stack and spec.dst_stack):
        rows = []
        for tiles in tile_lists(spec, rng):
            rows += tiles + [(TILE_NONE, TILE_NONE)] * (N - len(tiles))
        idx = torch.tensor(rows, dtype=torch.int32).reshape(-1, 2).to(device)
        assert idx.shape[0] == (B * N if spec.per_image else N)
    if spec.src_stack:
        assert len(spec.srcs) == 1 and spec.srcs[0][1] == 0 and not spec.window and not spec.mod
        srcs = [randn(spec.NT, spec.R, spec.Sx, spec.Cin)]
        bufs = list(srcs)
    elif spec.window:
        extra, c0 = spec.window
        (c, up), = spec.srcs
        buf = randn(B, spec.H >> up, spec.W >> up, c + extra)
        srcs, bufs = [buf[..., c0:c0 + c]], [buf]
    else:
        srcs = [randn(B, spec.H >> up, spec.W >> up, c) for c, up in spec.srcs]
        bufs = list(srcs)
    scale = shift = None
    if spec.preop:
        nb = B if spec.preop == "per_sample" else 1
        scale = (1 + 0.2 * torch.randn(nb, spec.Cin, generator=gen, device=device)).float()
        shift = (0.2 * torch.randn(nb, spec.Cin, generator=gen, device=device)).float()
    K = spec.Cin * spec.kH * spec.kW
    w = randn(spec.Cout, spec.Cin, spec.kH, spec.kW, scale=K ** -0.5)
    bias = randn(spec.Cout, dt=torch.float32) if spec.bias else None
    dst = None if spec.dst is None else writable(spec.Cout + spec.dst[0])
    residual = None
    if spec.residual is not None:
        shape = (spec.NT, spec.Ro, spec.So) if spec.dst_stack else (B, spec.dH, spec.dW)
        residual = randn(*shape, spec.Cout + spec.residual[0])
    aux = []
    for extra, c0, affine, act in spec.aux:
        sc = (1 + 0.3 * torch.randn(spec.Cout, generator=gen, device=device)).float() if affine else None
        sh = (0.3 * torch.randn(spec.Cout, generator=gen, device=device)).float() if affine else None
        aux.append(Aux(writable(spec.Cout + extra), c0, sc, sh, act))
    case = Case(spec, dtype, srcs, bufs, idx, scale, shift, w, bias, dst, residual, aux)
    if spec.mod:
        case.gamma = randn(B, spec.H, spec.W, spec.Cin + spec.mod[0], scale=0.5)
        case.beta = randn(B, spec.H, spec.W, spec.Cin + spec.mod[2], scale=0.5)
    if torch.device(device).type == "cuda":
        from sige_b200 import ops

        # a narrow source's weights are packed zero-padded to a whole number of 64-channel chunks
        case.wp = ops.pack_conv_weight(F.pad(w, (0, 0, 0, 0, 0, -spec.Cin % KC)), dtype)
    return case


# ----------------------------------------------------------------------------------------------------------------------
# the C descriptor, its plan and the launch
# ----------------------------------------------------------------------------------------------------------------------
def _ptr(t):
    return None if t is None else t.data_ptr()


def descriptor(case: Case, ksplit: int = 0, flags: int = 0):
    """The sige_tile_conv_t of this case; d._keep holds the tensors.  (No SIGE_CONV_TC5: the mma.sync kernel takes the launch.)"""
    from sige_b200 import _cabi

    s = case.spec
    d = _cabi.TileConv()
    d.dtype = {torch.float16: _cabi.F16, torch.bfloat16: _cabi.BF16, torch.float32: _cabi.F32}[case.dtype]
    d.n_src = len(case.srcs)
    for i, (t, (c, up)) in enumerate(zip(case.srcs, s.srcs)):
        d.src[i].ptr, d.src[i].C, d.src[i].up = t.data_ptr(), c, up
    d.B = s.B
    d.H, d.W = (s.R, s.Sx) if s.src_stack else (s.H, s.W)
    d.src_is_stack = 1 if s.src_stack else 0
    d.idx, d.N = _ptr(case.idx), s.N
    d.R, d.S = s.R, s.Sx
    d.scale, d.shift = _ptr(case.scale), _ptr(case.shift)
    d.affine_bstride = s.Cin if s.preop == "per_sample" else 0
    d.act = s.act
    d.w_packed, d.bias = _ptr(case.wp), _ptr(case.bias)
    d.Cin, d.Cout, d.kH, d.kW, d.stride = s.Cin, s.Cout, s.kH, s.kW, s.stride
    d.dst = None if case.dst is None else case.dst.view.data_ptr()
    d.dst_is_stack = 1 if s.dst_stack else 0
    d.dH, d.dW = (s.Ro, s.So) if s.dst_stack else (s.dH, s.dW)
    d.dC, d.dst_c0 = (0, 0) if case.dst is None else (case.dst.view.shape[3], s.dst[1])
    d.offH, d.offW = s.offs
    d.residual = _ptr(case.residual)
    d.rC, d.res_c0 = (0, 0) if case.residual is None else (case.residual.shape[3], s.residual[1])
    d.ksplit, d.flags = ksplit, flags
    d.n_aux = len(case.aux)
    for i, a in enumerate(case.aux):
        d.aux[i].ptr, d.aux[i].C, d.aux[i].c0 = a.g.view.data_ptr(), a.g.view.shape[3], a.c0
        d.aux[i].scale, d.aux[i].shift, d.aux[i].act = _ptr(a.scale), _ptr(a.shift), a.act
    d.idx_per_image = 1 if s.per_image else 0
    if s.window:
        d.src_pixel_stride = case.src_bufs[0].shape[3]
    if s.mod:
        d.modulation = pointer(modulation(case))
    d._keep = case
    return d


def modulation(case: Case):
    from sige_b200 import _cabi

    m = _cabi.ConvModulation()
    m.gamma, m.gamma_C, m.gamma_c0 = case.gamma.data_ptr(), case.gamma.shape[3], case.spec.mod[1]
    m.beta, m.beta_C, m.beta_c0 = case.beta.data_ptr(), case.beta.shape[3], case.spec.mod[3]
    m.negative_slope = case.spec.mod[4]
    m._keep = case
    return m


def plan_of(d):
    """sige_tile_conv_plan of a descriptor."""
    from sige_b200 import _cabi

    p = _cabi.TileConvPlan()
    _cabi.check(_cabi.lib().sige_tile_conv_plan(byref(d), byref(p)), "sige_tile_conv_plan")
    return p


def plan_tuple(p):
    return (p.path, p.bn, p.ksplit, p.deep_ring, p.grid_x, p.grid_y, p.grid_z)


def expected_plan_tuple(p: Optional[Plan]):
    return (0, 0, 0, 0, 0, 0, 0) if p is None else (0, p.bn, p.ksplit, 0) + p.grid


# ----------------------------------------------------------------------------------------------------------------------
# float64 reference
# ----------------------------------------------------------------------------------------------------------------------
def _act(x, act):
    return x * torch.sigmoid(x) if act == 1 else (x.clamp(min=0) if act == 2 else x)


def c_div(a: torch.Tensor, b: int) -> torch.Tensor:
    """Integer division as C does it: towards zero."""
    return torch.div(a, b, rounding_mode="trunc")


def operand(case: Case):
    """(a, t, img, org): the conv's A operand [NT, R, S, Cin] in float64 — gathered (or the stack), pre-op and modulation applied,
    rounded to the launch dtype where the kernel stages it so, zero outside the image — with each row's tile number, image and
    origin (None for a stack source)."""
    s = case.spec
    dev = case.w.device
    t = torch.arange(s.NT, device=dev)
    img = t // s.N
    org = None
    if case.idx is not None:
        org = case.idx.long()[t if s.per_image else t % s.N]
    if s.src_stack:
        a = case.srcs[0].double()
        valid = torch.ones(s.NT, s.R, s.Sx, dtype=torch.bool, device=dev)
        hh = ww = None
    else:
        hh = org[:, :1] + torch.arange(s.R, device=dev)                       # [NT, R]
        ww = org[:, 1:] + torch.arange(s.Sx, device=dev)                      # [NT, S]
        valid = ((hh >= 0) & (hh < s.H))[:, :, None] & ((ww >= 0) & (ww < s.W))[:, None, :]
        hc, wc = hh.clamp(0, s.H - 1), ww.clamp(0, s.W - 1)
        a = torch.cat([x[img[:, None, None], (hc >> up)[:, :, None], (wc >> up)[:, None, :]].double()
                       for x, (_, up) in zip(case.srcs, s.srcs)], -1)
    staged = bool(s.preop) or s.act != 0 or s.mod is not None
    if s.preop:
        sel = img if s.preop == "per_sample" else torch.zeros_like(img)
        a = a * case.scale.double()[sel][:, None, None, :] + case.shift.double()[sel][:, None, None, :]
    a = _act(a, s.act)
    if s.mod:
        g = case.gamma.double()[img[:, None, None], hc[:, :, None], wc[:, None, :]][..., s.mod[1]:s.mod[1] + s.Cin]
        b = case.beta.double()[img[:, None, None], hc[:, :, None], wc[:, None, :]][..., s.mod[3]:s.mod[3] + s.Cin]
        a = a * (1 + g) + b
        a = torch.where(a < 0, a * s.mod[4], a)
    if staged:
        a = a.to(case.dtype).double()
    a = torch.where(valid[..., None], a, torch.zeros((), dtype=a.dtype, device=dev))
    return a, t, img, org, staged


def output_pixels(case: Case, t, img, org, floor_division: bool = False):
    """(OB, OH, OW, ok), each [NT, Ro, So]: where every output pixel of every tile goes, and whether it is inside the buffer."""
    s = case.spec
    dev = t.device
    dy, dx = torch.arange(s.Ro, device=dev), torch.arange(s.So, device=dev)
    if s.dst_stack:
        ob, oh, ow = t, dy[None, :].expand(s.NT, -1), dx[None, :].expand(s.NT, -1)
        H, W = s.Ro, s.So
    else:
        div = (lambda a, b: torch.div(a, b, rounding_mode="floor")) if floor_division else c_div
        oh = div(s.offs[0] + org[:, :1], s.stride) + dy
        ow = div(s.offs[1] + org[:, 1:], s.stride) + dx
        ob, H, W = img, s.dH, s.dW
    ok = ((oh >= 0) & (oh < H))[:, :, None] & ((ow >= 0) & (ow < W))[:, None, :]
    shape = (s.NT, s.Ro, s.So)
    return ob[:, None, None].expand(shape), oh[:, :, None].expand(shape), ow[:, None, :].expand(shape), ok


def tile_values(case: Case, floor_division: bool = False):
    """(v, bound, OB, OH, OW, ok): the launch's result before rounding, [NT, Ro, So, Cout] in float64, its per-element bound,
    and where every output pixel goes (see output_pixels).  Only the tiles are gathered, so the buffers may be any size."""
    s = case.spec
    dev = case.w.device
    u = kc.ROUNDOFF[case.dtype]
    a, t, img, org, staged = operand(case)
    w = case.w.double()
    nchw = a.permute(0, 3, 1, 2)
    v = F.conv2d(nchw, w, stride=s.stride).permute(0, 2, 3, 1)                # [NT, Ro, So, Cout]
    mag = F.conv2d(nchw.abs(), w.abs(), stride=s.stride).permute(0, 2, 3, 1)
    assert tuple(v.shape[1:3]) == (s.Ro, s.So)
    pre = torch.zeros(s.Cout, dtype=torch.float64, device=dev)
    if staged:
        pre = PRE_ULPS * u * w.abs().amax(dim=(1, 2, 3)) * a.abs().max()
    if case.bias is not None:
        v = v + case.bias.double()
        mag = mag + case.bias.double().abs()
    OB, OH, OW, ok = output_pixels(case, t, img, org, floor_division)
    if case.residual is not None:
        c0 = s.residual[1]
        r = case.residual[OB, OH.clamp(0, case.residual.shape[1] - 1), OW.clamp(0, case.residual.shape[2] - 1)][..., c0:c0 + s.Cout].double()
        v, mag = v + r, mag + r.abs()
    return v, u * v.abs() + ACC * mag + pre + ABS, OB, OH, OW, ok


def reference(case: Case, floor_division: bool = False) -> List[kc.Expect]:
    """`floor_division` computes the output origin with floor instead of C division: a deliberately wrong contract, for the
    tests that show `check` tells the two apart."""
    s = case.spec
    dev = case.w.device
    u = kc.ROUNDOFF[case.dtype]
    v, bound, OB, OH, OW, ok = tile_values(case, floor_division)
    ob, oh, ow = OB[ok], OH[ok], OW[ok]
    shape = (s.NT, s.Ro, s.So) if s.dst_stack else (s.B, s.dH, s.dW)
    lin = (ob * shape[1] + oh) * shape[2] + ow
    assert lin.unique().numel() == lin.numel(), "case %s: two tiles write the same output pixel" % s.name

    def scatter(name, g, c0, val, bd):
        e, (want, written, b, rnd) = kc.expect_for(name, g, u)
        sl = slice(c0, c0 + s.Cout)
        want[ob, oh, ow, sl] = val[ok]
        written[ob, oh, ow, sl] = True
        b[ob, oh, ow, sl] = bd[ok]
        rnd[ob, oh, ow, sl] = u * val[ok].abs()
        return e

    out = []
    if case.dst is not None:
        out.append(scatter("dst", case.dst, s.dst[1], v, bound))
    for i, ax in enumerate(case.aux):
        sc = torch.ones(s.Cout, dtype=torch.float64, device=dev) if ax.scale is None else ax.scale.double()
        sh = torch.zeros(s.Cout, dtype=torch.float64, device=dev) if ax.shift is None else ax.shift.double()
        av = _act(v * sc + sh, ax.act)
        out.append(scatter("aux%d" % i, ax.g, ax.c0, av, SWISH_LIP * sc.abs() * bound + u * av.abs()))
    return out


def rounded_result(case: Case, expects: List[kc.Expect]) -> Dict[str, torch.Tensor]:
    """What an exact kernel would leave: the expectation rounded once to the launch dtype where written, the initial bytes elsewhere."""
    out = {}
    for e in expects:
        got = e.g.flat.clone()
        got[e.written] = e.want[e.written].to(case.dtype)
        out[e.name] = got
    return out
