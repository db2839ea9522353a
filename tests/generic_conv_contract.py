"""The C-ABI contract of sige_tile_conv_generic (the CUDA-core tile conv, sige_b200/csrc/tile_conv_simt.cu), restated in float64.

Every sparse SIGEConv2d of an fp32 model runs here, and so does every grouped, dilated or anisotropic-stride conv in any dtype
(GauGAN's depthwise convs among them).  Imported by tests/test_generic_conv_contract.py (CPU: the restatement against F.conv2d,
the C oracle and a float32 conv of another summation order; mutants of the kernel that the bound must reject; the case table
against the launcher's predicate; the refusals) and tests/test_gpu_generic_conv_contract.py (GPU: every case against the
restatement, and the bitwise invariants the kernels' fixed summation order implies).  Same vocabulary as tests/kernel_contracts.py:
a frozen `GenSpec`, `make_gen(spec, dtype, device)`, `gen_call(case, lib)` and `gen_reference(case) -> List[Expect]`.

Operands: the stack x (M, Cin, R, S) in NCHW or NHWC, the OIHW weight [Cout][Cin/groups][kH][kW] and a bias in the launch dtype
(or NULL), each a window of a flat buffer of random bytes so that a read past its end shows; the output stack (M, Cout, Ro, So)
in the same layout is a guarded window (16-byte aligned, or one element off with `misalign`).

Unlike the tensor-core contracts (tile_conv_contract.ACC is an estimate), this kernel's error has a rigorous bound: it
accumulates K = (Cin/groups) kH kW products by sequential fp32 fmaf from 0 and adds the bias once; see gen_reference.
"""
from __future__ import annotations

from dataclasses import dataclass, replace
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from kernel_contracts import H100_SMS, ROUNDOFF, Expect, Guarded, expect_for, guarded
from step_kernel_contracts import HALF_SUBNORMAL, _code, _esize, _stream

U32 = 2.0 ** -24
SIMT_CO, SIMT_CI, SIMT_PG, SIMT_MAXPP = 64, 16, 4, 8   # tile_conv_simt.cu: Cout per CTA, Cin per chunk, pixel groups, pixels per thread
DW_THREADS, DW_BLOCKS_PER_SM = 256, 16
SMEM_DEFAULT = 48 * 1024
VEC = {torch.float32: 4, torch.float16: 8, torch.bfloat16: 8}
PATHS = ("simt", "simt_big_smem", "dw_vec", "dw_nhwc_scalar", "dw_nchw")
MUTANTS = ("drop_last", "group_shift", "transpose", "swap_stride", "swap_dilation", "no_bias", "other16")
OTHER16 = {torch.float16: torch.bfloat16, torch.bfloat16: torch.float16}


@dataclass(frozen=True)
class GenSpec:
    """One sige_tile_conv_generic launch.  misalign: the output window one element off 16-byte alignment.  spread: input channel
    c scaled by 2^(-10 + 20 c / (Cin - 1)), so that products of very different magnitudes cancel."""
    name: str
    M: int
    Cin: int
    Cout: int
    R: int
    S: int
    kH: int = 3
    kW: int = 3
    strideH: int = 1
    strideW: int = 1
    dilH: int = 1
    dilW: int = 1
    groups: int = 1
    layout: str = "nchw"
    bias: bool = True
    misalign: bool = False
    spread: bool = False
    seed: int = 0

    @property
    def Ro(self) -> int:
        return (self.R - self.dilH * (self.kH - 1) - 1) // self.strideH + 1

    @property
    def So(self) -> int:
        return (self.S - self.dilW * (self.kW - 1) - 1) // self.strideW + 1

    @property
    def P(self) -> int:
        return self.Ro * self.So

    @property
    def cig(self) -> int:
        return self.Cin // self.groups

    @property
    def cog(self) -> int:
        return self.Cout // self.groups

    @property
    def K(self) -> int:
        """Products accumulated per output element."""
        return self.cig * self.kH * self.kW

    @property
    def depthwise(self) -> bool:
        return self.groups == self.Cin == self.Cout

    @property
    def stride(self):
        return (self.strideH, self.strideW)

    @property
    def dilation(self):
        return (self.dilH, self.dilW)


def simt_smem(spec: GenSpec) -> int:
    """Dynamic shared memory of tile_conv_simt_kernel: a 16-channel halo chunk and a 64-channel weight slab (odd row pitch)."""
    return 4 * (SIMT_CI * spec.R * spec.S + SIMT_CO * (SIMT_CI * spec.kH * spec.kW + 1))


def generic_path(spec: GenSpec, dtype, misalign: bool) -> str:
    """The kernel form the launcher picks: depthwise (groups == Cin == Cout) in NCHW, NHWC with 16-byte channel vectors (C a
    multiple of the vector and both stacks 16-byte aligned; x always is here) or NHWC scalar; else the generic kernel, with its
    dynamic shared-memory limit raised above 48 KB."""
    if spec.depthwise:
        if spec.layout == "nchw":
            return "dw_nchw"
        return "dw_vec" if spec.Cin % VEC[dtype] == 0 and not misalign else "dw_nhwc_scalar"
    return "simt_big_smem" if simt_smem(spec) > SMEM_DEFAULT else "simt"


def pixel_passes(spec: GenSpec) -> int:
    """Passes of the generic kernel over the output pixels of a tile (32 per pass)."""
    return -(-spec.P // (SIMT_PG * SIMT_MAXPP))


def cout_blocks(spec: GenSpec) -> int:
    """CTAs per (tile, group) along the output channels of a group."""
    return -(-spec.cog // SIMT_CO)


def k_chunks(spec: GenSpec) -> int:
    """16-input-channel chunks of a group."""
    return -(-spec.cig // SIMT_CI)


def dw_items(spec: GenSpec, dtype, misalign: bool) -> int:
    vec = generic_path(spec, dtype, misalign) == "dw_vec"
    return spec.M * spec.P * (spec.Cin // VEC[dtype] if vec else spec.Cin)


def dw_trips(spec: GenSpec, dtype, misalign: bool, sms: int = H100_SMS) -> int:
    """Trips of the depthwise grid-stride loop for its busiest thread: one thread per item, at most 16 CTAs of 256 per SM."""
    items = dw_items(spec, dtype, misalign)
    blocks = min(-(-items // DW_THREADS), DW_BLOCKS_PER_SM * sms)
    return -(-items // (blocks * DW_THREADS))


G = GenSpec
GEN_CASES = [
    # chunk and block edges
    G("cin8_cout12", 5, 8, 12, 6, 6, seed=1),
    G("cin36_cout70", 7, 36, 70, 6, 6, seed=2),
    G("cin36_cout48_nhwc_nobias", 6, 36, 48, 6, 6, layout="nhwc", bias=False, seed=3),
    G("cin36_cout20_1x1_r4", 2, 36, 20, 4, 4, kH=1, kW=1, layout="nhwc", seed=4),
    G("cin64_cout64_m64", 64, 64, 64, 6, 6, layout="nhwc", seed=5),
    G("cin8_cout12_nhwc_misaligned", 5, 8, 12, 6, 6, layout="nhwc", misalign=True, seed=6),
    # pixel passes and shared memory
    G("rgb_cin3_cout5_r10_p64", 2, 3, 5, 10, 10, seed=7),
    G("cin24_cout40_1x1_r8_p64", 4, 24, 40, 8, 8, kH=1, kW=1, layout="nhwc", seed=8),
    G("k5_r9_big_smem", 6, 20, 24, 9, 9, kH=5, kW=5, seed=9),
    G("k3_r14_big_smem", 3, 16, 32, 14, 14, layout="nhwc", seed=10),
    # large kernel and grid
    G("k7_r12", 3, 18, 16, 12, 12, kH=7, kW=7, seed=11),
    G("m1600", 1600, 16, 24, 6, 6, layout="nhwc", seed=12),
    # anisotropic geometry
    G("r6_s9", 5, 12, 20, 6, 9, seed=13),
    G("k1x3", 4, 20, 24, 4, 6, kH=1, kW=3, seed=14),
    G("k3x1_nhwc", 4, 20, 24, 6, 4, kH=3, kW=1, layout="nhwc", seed=15),
    G("stride2x1", 5, 16, 24, 7, 6, strideH=2, strideW=1, seed=16),
    G("dil1x2_nhwc", 4, 16, 16, 6, 8, dilH=1, dilW=2, layout="nhwc", seed=17),
    G("k3x5_stride1x2_dil2x1", 3, 8, 8, 9, 11, kH=3, kW=5, strideH=1, strideW=2, dilH=2, dilW=1, seed=18),
    G("stride2_r5", 3, 16, 16, 5, 5, strideH=2, strideW=2, seed=19),
    # groups
    G("g2_cig20_cog70", 4, 40, 140, 6, 6, groups=2, seed=20),
    G("g2_cin8_dil2_r7", 3, 8, 8, 7, 7, dilH=2, dilW=2, groups=2, seed=21),
    G("g4_dil2_nhwc", 3, 32, 16, 7, 7, dilH=2, dilW=2, groups=4, layout="nhwc", seed=22),
    G("multiplier_g16_cout32", 6, 16, 32, 6, 6, groups=16, seed=23),
    # depthwise forms
    G("dw_c128_nchw_m300", 300, 128, 128, 6, 6, groups=128, seed=30),
    G("dw_c128_nhwc", 40, 128, 128, 6, 6, groups=128, layout="nhwc", seed=31),
    G("dw_c96_nhwc", 40, 96, 96, 6, 6, groups=96, layout="nhwc", seed=32),
    G("dw_c96_nchw", 40, 96, 96, 6, 6, groups=96, seed=33),
    G("dw_c6_nhwc_stride2_r5", 9, 6, 6, 5, 5, strideH=2, strideW=2, groups=6, layout="nhwc", seed=34),
    G("dw_c12_nhwc", 4, 12, 12, 6, 6, groups=12, layout="nhwc", seed=35),
    G("dw_c12_nchw", 4, 12, 12, 6, 6, groups=12, seed=36),
    G("dw_c64_nhwc_dil2_r8_misaligned", 5, 64, 64, 8, 8, dilH=2, dilW=2, groups=64, layout="nhwc", misalign=True, seed=37),
    G("dw_c64_nchw_dil2_r8", 5, 64, 64, 8, 8, dilH=2, dilW=2, groups=64, seed=38),
    G("dw_c16_nhwc_nobias_k3x1_stride1x2", 7, 16, 16, 6, 7, kH=3, kW=1, strideH=1, strideW=2, groups=16, layout="nhwc", bias=False,
      seed=39),
    G("dw_c128_nhwc_m2200_grid_stride", 2200, 128, 128, 6, 6, groups=128, layout="nhwc", seed=40),
    G("dw_c128_nhwc_m2200_grid_stride_misaligned", 2200, 128, 128, 6, 6, groups=128, layout="nhwc", misalign=True, seed=41),
    # values
    G("spread_cin32_cout24", 8, 32, 24, 6, 6, spread=True, seed=50),
    G("spread_g2_nhwc_nobias", 4, 36, 20, 6, 6, groups=2, layout="nhwc", bias=False, spread=True, seed=51),
]
del G


@dataclass
class GenCase:
    spec: GenSpec
    dtype: torch.dtype
    x: Guarded                  # physical layout: NCHW (M, Cin, R, S) or NHWC (M, R, S, Cin)
    w: Guarded                  # (Cout, Cin/groups, kH, kW)
    b: Optional[Guarded]        # (Cout,)
    out: Guarded                # (M, Cout, Ro, So) or (M, Ro, So, Cout)

    def buffers(self) -> Dict[str, Guarded]:
        return {"out": self.out}

    def inputs(self) -> Dict[str, torch.Tensor]:
        d = {"x": self.x.flat, "w": self.w.flat}
        if self.b is not None:
            d["bias"] = self.b.flat
        return d

    def logical(self, t: torch.Tensor) -> torch.Tensor:
        """NCHW view of a stack in the case's layout."""
        return t.permute(0, 3, 1, 2) if self.spec.layout == "nhwc" else t

    @property
    def x_nchw(self) -> torch.Tensor:
        return self.logical(self.x.view)

    @property
    def bias(self) -> Optional[torch.Tensor]:
        return None if self.b is None else self.b.view


def _phys(shape, layout):
    n, c, h, w = shape
    return (n, h, w, c) if layout == "nhwc" else (n, c, h, w)


def make_gen(spec: GenSpec, dtype: torch.dtype, device, layout: Optional[str] = None, misalign: Optional[bool] = None) -> GenCase:
    """The values depend on the spec's seed only: `layout` / `misalign` override the spec's and give the same operands."""
    if layout is not None or misalign is not None:
        spec = replace(spec, layout=spec.layout if layout is None else layout, misalign=spec.misalign if misalign is None else misalign)
    gen = torch.Generator(device=device)
    gen.manual_seed(spec.seed)

    def randn(*shape, scale=1.0):
        return torch.randn(*shape, generator=gen, device=device, dtype=torch.float64) * scale

    x = randn(spec.M, spec.Cin, spec.R, spec.S)
    if spec.spread:
        x = x * torch.exp2(-10 + 20 * torch.arange(spec.Cin, device=device, dtype=torch.float64) / (spec.Cin - 1)).view(1, -1, 1, 1)
    w = randn(spec.Cout, spec.cig, spec.kH, spec.kW, scale=spec.K ** -0.5)
    b = randn(spec.Cout, scale=0.3) if spec.bias else None

    def holding(t, shape, layout_name):
        g = guarded(shape, dtype, device, gen, layout_name)
        g.view.copy_(t.to(dtype))
        return g

    xg = holding(x.permute(0, 2, 3, 1) if spec.layout == "nhwc" else x, _phys(x.shape, spec.layout), spec.layout)
    wg = holding(w, tuple(w.shape), "nchw")
    bg = None if b is None else holding(b, (spec.Cout,), "bc")
    lead = 64 + (_esize(dtype) if spec.misalign else 0)
    out = guarded(_phys((spec.M, spec.Cout, spec.Ro, spec.So), spec.layout), dtype, device, gen, spec.layout, lead_bytes=lead)
    return GenCase(spec, dtype, xg, wg, bg, out)


def gen_call(case: GenCase, lib, stream=None):
    """Calls sige_tile_conv_generic for the case on the current stream; returns the status."""
    s = case.spec
    lay = 1 if s.layout == "nhwc" else 0
    return lib.sige_tile_conv_generic(case.x.view.data_ptr(), case.w.view.data_ptr(), None if case.b is None else case.b.view.data_ptr(),
                                      case.out.view.data_ptr(), _code(case.dtype), lay, s.M, s.Cin, s.R, s.S, s.Cout, s.kH, s.kW,
                                      s.strideH, s.strideW, s.dilH, s.dilW, s.groups, _stream() if stream is None else stream)


def gamma(n: int, u: float = U32) -> float:
    """Higham's gamma_n = n u / (1 - n u): the relative error of n successive roundings."""
    return n * u / (1 - n * u)


def conv64(x, w, b, stride, dilation, groups, Ro, So):
    """F.conv2d(x, w, b, stride, 0, dilation, groups) cropped to (Ro, So), written out as a sum over the taps of grouped channel
    contractions (float64 grouped convs are slow in torch's CPU conv; this is also independent of it).  The input is
    zero-extended at the bottom / right where the geometry needs more of it than the tile holds (a mutant's geometry may)."""
    M, Cin = x.shape[:2]
    Cout, cig, kH, kW = w.shape
    (sH, sW), (dH, dW) = stride, dilation
    needH, needW = (Ro - 1) * sH + dH * (kH - 1) + 1, (So - 1) * sW + dW * (kW - 1) + 1
    x = F.pad(x, (0, max(0, needW - x.shape[3]), 0, max(0, needH - x.shape[2])))
    wg = w.reshape(groups, Cout // groups, cig, kH, kW)
    out = torch.zeros(M, groups, Cout // groups, Ro, So, dtype=x.dtype, device=x.device)
    for ky in range(kH):
        for kx in range(kW):
            xs = x[:, :, ky * dH:ky * dH + (Ro - 1) * sH + 1:sH, kx * dW:kx * dW + (So - 1) * sW + 1:sW]
            out += torch.einsum("mgchw,gdc->mgdhw", xs.reshape(M, groups, cig, Ro, So), wg[..., ky, kx])
    out = out.reshape(M, Cout, Ro, So)
    return out if b is None else out + b.view(1, -1, 1, 1)


def gen_values(case: GenCase):
    """float64 value and magnitude (the same conv of |x|, |w|, |b|) of every output element, logical NCHW."""
    s = case.spec
    x, w = case.x_nchw.double(), case.w.view.double()
    b = None if case.b is None else case.bias.double()
    v = conv64(x, w, b, s.stride, s.dilation, s.groups, s.Ro, s.So)
    mag = conv64(x.abs(), w.abs(), None if b is None else b.abs(), s.stride, s.dilation, s.groups, s.Ro, s.So)
    return v, mag


def gen_reference(case: GenCase) -> List[Expect]:
    """out = F.conv2d(x, w, b, stride, 0, dilation, groups) in float64 on the stored operands, with a rigorous bound.

    Both kernel forms compute each output as acc = fmaf(x_K, w_K, ... fmaf(x_1, w_1, 0)) over its K = (Cin/groups) kH kW
    products (each exact inside its fmaf: the operands are fp32 or exactly widened 16-bit values), then fl32(acc + b) (b = 0
    without a bias: exact), then the store in the launch dtype.  With U = 2^-24 and every fp32 rounding
    fl(t) = t (1 + d) + e, |d| <= U, |e| <= 2^-150 (e only below the normal range), the k-th product reaches the fp32 result
    through at most K + 1 factors (1 + d), and the bias through one, so
        |fp32 result - value| <= gamma_{K+1} mag + (K + 1) 2^-150 (1 + gamma_{K+1}) =: E,
    mag = |b| + sum |x||w| (a float64 conv of absolute values), whatever the order of the products.  f32 stores the fp32 result
    as it is.  A 16-bit store rounds it once more: |fl16(r) - r| <= u |r| + HALF_SUBNORMAL <= u (|want| + E) + HALF_SUBNORMAL, so
        bound = (1 + u) E + u |want| + HALF_SUBNORMAL,
    of which u |want| + HALF_SUBNORMAL is the element's own rounding (`rounding`; 0 for f32).  Nothing here is an estimate, so
    one dropped or misplaced product of a typical magnitude exceeds it (tests/test_generic_conv_contract.py's mutants)."""
    s = case.spec
    u = ROUNDOFF[case.dtype]
    v, mag = gen_values(case)
    g = gamma(s.K + 1)
    E = g * mag + (s.K + 1) * 2.0 ** -150 * (1 + g)
    if case.dtype in (torch.float32, torch.float64):
        rounding = torch.zeros_like(v)
        bound = E
    else:
        rounding = u * v.abs() + HALF_SUBNORMAL[case.dtype]
        bound = (1 + u) * E + rounding
    e, (want, written, bd, rnd) = expect_for("out", case.out, u)
    for t, val in ((want, v), (written, True), (bd, bound), (rnd, rounding)):
        case.logical(t)[:] = val
    return [e]


# ----------------------------------------------------------------------------------------------------------------------
# mutants: what a subtly wrong kernel would compute (the CPU suite demands that `check` rejects each)
# ----------------------------------------------------------------------------------------------------------------------
def mutant_applies(spec: GenSpec, dtype, name: str) -> bool:
    """Does the mutation change the math of this case?  (other16: rounding bf16 weights through f16 is exact above f16's
    normal range; it moves only weights below 2^-14, by less than any bound, so it applies to f16 weights only.)"""
    return {"drop_last": True, "group_shift": spec.groups > 1, "transpose": (spec.kH, spec.kW) != (1, 1),
            "swap_stride": spec.strideH != spec.strideW, "swap_dilation": spec.dilH != spec.dilW, "no_bias": spec.bias,
            "other16": dtype == torch.float16}[name]


def gen_mutant(case: GenCase, name: str) -> torch.Tensor:
    """float64 outputs (logical NCHW) of a kernel with one mistake:
      drop_last      the last product of the last K chunk (ci = Cin/groups - 1, the last tap) is never added
      group_shift    group g >= 1 reads its input channels at group g - 1's offset
      transpose      the kernel's taps are read transposed: a kW x kH kernel of w^T
      swap_stride    strideH and strideW exchanged
      swap_dilation  dilH and dilW exchanged
      no_bias        the bias is not added
      other16        the weights rounded through the other 16-bit type"""
    s = case.spec
    x, w = case.x_nchw.double(), case.w.view.double()
    b = None if case.b is None else case.bias.double()
    stride, dil = s.stride, s.dilation
    if name == "drop_last":
        w = w.clone()
        w[:, -1, -1, -1] = 0
    elif name == "group_shift":
        x = x.clone()
        for g in range(1, s.groups):
            x[:, g * s.cig:(g + 1) * s.cig] = case.x_nchw[:, (g - 1) * s.cig:g * s.cig].double()
    elif name == "transpose":
        w = w.transpose(2, 3)
    elif name == "swap_stride":
        stride = stride[::-1]
    elif name == "swap_dilation":
        dil = dil[::-1]
    elif name == "no_bias":
        b = None
    elif name == "other16":
        w = case.w.view.to(OTHER16[case.dtype]).double()
    else:
        raise ValueError(name)
    return conv64(x, w, b, stride, dil, s.groups, s.Ro, s.So)


def gen_written(case: GenCase, val: torch.Tensor) -> torch.Tensor:
    """The flat output buffer a launch leaves when it writes `val` (logical NCHW, rounded to the dtype): the guard bands as
    they were."""
    flat = case.out.flat.clone()
    win = flat[case.out.off:case.out.off + case.out.view.numel()].view(*case.out.view.shape)
    case.logical(win)[:] = val.to(case.dtype)
    return flat


def gen_cost(spec: GenSpec) -> int:
    """Multiply-adds of the launch (to keep the float64 CPU checks to the cases they finish quickly on)."""
    return spec.M * spec.Cout * spec.P * spec.K
