"""The C-ABI contracts of the sparse-query attention, SPADE modulation and the tile ops, restated in float64.

These are the kernels a compiled step launches besides the tile convs and the dense glue: sige_sparse_attention (the SD step's
attention, and attention cores outside the cluster kernel's range), sige_spade_modulate (the GauGAN steps' SPADE layers that
stay off the modulated tile conv) and sige_gather / sige_scatter / sige_scatter_gather / sige_scatter_with_block_residual (the
fused step's gathers and the eager modules).  Imported by tests/test_step_kernel_contracts.py (CPU: each restatement against an
independent computation, the case tables against the launchers' predicates, the C-ABI refusals) and
tests/test_gpu_step_kernel_contracts.py (GPU: every case against its restatement).  Same vocabulary as tests/kernel_contracts.py:
a frozen `...Spec`, `make_...(spec, dtype, device)`, `..._call(case, lib)` and `..._reference(case) -> List[Expect]`; every
buffer a launch may write is a window of a guarded flat buffer, and `check` demands the per-element bound on what is written and
bitwise equality everywhere else, inputs included.

Bounds (u = unit roundoff of the launch dtype, U32 = 2^-24):

  sparse attention  derived at sattn_reference.
  SPADE             out = act(fmaf(x, fl32(1 + g), b)): the fmaf and the leaky slope's multiply round in fp32, the store rounds
                    once: (u + 2 U32) |want| + HALF_SUBNORMAL (an f16 result below the normal range rounds to a
                    fixed step).  With g = b = 0 and slope 1 the output is x, bitwise (bound 0).
  tile ops          identity moves: 0 (every path is bitwise exact).  Affine / swish: the fp32 chain's error (U32 per
                    multiply and add, SWISH_LIP through swish, and swish's own error: for 16-bit storage the fast swish's
                    swish_rel (__expf and __fdividef, common.cuh swish<true>), for f32 the accurate one's SWISH_ACCURATE_REL
                    (expf and an IEEE division, swish<false>)), plus one rounding u |want| + HALF_SUBNORMAL.  Residual add: U32 + u.
                    scatter_with_block_residual: scatter's rounding restated literally (fp32 add, then the launch dtype),
                    then calibrate's out + (x1 - y1) bounded like a residual add.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from kernel_contracts import (Expect, Guarded, ROUNDOFF, U32, bits, check, expect_for, guarded, restore,  # noqa: F401
                              snapshot)
from tile_conv_contract import ABS, ACC, SWISH_LIP

F16_BF16 = (torch.float16, torch.bfloat16)
# half the spacing of the dtype's subnormals: the absolute error of a rounding below the normal range, where u |want| does not hold
HALF_SUBNORMAL = {torch.float16: 2.0 ** -25, torch.bfloat16: 2.0 ** -134, torch.float32: 2.0 ** -150, torch.float64: 0.0}


def _code(dtype):
    from sige_b200 import _cabi

    return {torch.float32: _cabi.F32, torch.float16: _cabi.F16, torch.bfloat16: _cabi.BF16}[dtype]


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _esize(dtype) -> int:
    return torch.empty((), dtype=dtype).element_size()


def _random_bits(shape, dtype, device, gen) -> torch.Tensor:
    """Random bytes (NaN and Inf patterns included) in `dtype`: what the padding of an input buffer holds, so a read of it shows."""
    it = {2: torch.int16, 4: torch.int32, 8: torch.int64}[_esize(dtype)]
    info = torch.iinfo(it)
    t = torch.randint(info.min, info.max, shape, dtype=it, generator=gen, device=device).view(dtype)
    return torch.randn(shape, generator=gen, device=device, dtype=dtype) if dtype == torch.float64 else t


# ----------------------------------------------------------------------------------------------------------------------
# sige_sparse_attention
# ----------------------------------------------------------------------------------------------------------------------
HEAD_DIMS = (32, 40, 64, 80, 128, 160)
BNK = 64                        # keys per ring stage (one online-softmax block)
BM = 64                         # queries per CTA
LOG2E = 1.4426950408889634
EX2_REL = 2.0 ** -22            # ex2.approx.ftz.f32, relative
ETA_P = {torch.float16: 2.0 ** -25, torch.bfloat16: 0.0, torch.float32: 0.0, torch.float64: 0.0}   # half an f16 subnormal step
MODES = ("random", "flat", "dominant", "rising", "falling", "large", "constant_v")
LAYOUTS = ("bhnd", "bnhd", "kv_pair")
GUARD_COLS = 8                  # columns of guard band after each head in the bnhd / kv_pair layouts


@dataclass(frozen=True)
class SAttnSpec:
    """One sige_sparse_attention launch on [B, heads, N, D] operands.

    layout: "bhnd" (contiguous), "bnhd" (q, k, v and out addressed in place in "b n (h d)" buffers with a head pitch of D + 8:
    the 8 columns after each head are guard band) or "kv_pair" (q and out as in bnhd; k and v the two halves of one
    [B, Nk, 2 heads D] buffer, as cached text keys are).  Size-1 dims get stride 0, as ops.sparse_attention passes them.
    mode (scaled logits): "random" ~ N(0, 4); "flat" q = 0; "dominant" one key ~12 above the rest, key 17 of the first block
    (dom="first") or the last key (dom="last"); "rising" each key block ~8 above the previous one; "falling" each block ~3 below
    the previous one; "large" a_i t_j with |a|, |t| <= sqrt(80); "constant_v" random logits, every v_j equal.
    scale: None for D^-0.5."""
    name: str
    B: int
    heads: int
    Nq: int
    Nk: int
    D: int
    mode: str = "random"
    layout: str = "bhnd"
    scale: Optional[float] = None
    dom: str = "first"
    seed: int = 0

    @property
    def s32(self) -> float:
        """The scale as the descriptor's float holds it."""
        return float(np.float32(self.D ** -0.5 if self.scale is None else self.scale))

    @property
    def blocks(self) -> int:
        return -(-self.Nk // BNK)

    @property
    def dom_key(self) -> int:
        return min(17, self.Nk - 1) if self.dom == "first" else self.Nk - 1


def sattn_padded(D: int) -> int:
    """The head dim the kernel works on: D padded to the MMA k-step of 16 (sparse_attention.cu Lay<D>::DP)."""
    return (D + 15) // 16 * 16


def _sattn_cases():
    P = SAttnSpec
    cases = []
    for i, D in enumerate(HEAD_DIMS):
        sd = 100 * D
        cases += [
            P("d%d_q63_k63_random_bhnd" % D, 2, 2, 63, 63, D, seed=sd + 1),
            P("d%d_q65_k130_random_bnhd" % D, 1, 3, 65, 130, D, layout="bnhd", seed=sd + 2),
            P("d%d_q200_k77_kvpair_scale" % D, 2, 2, 200, 77, D, layout="kv_pair", scale=0.0917, seed=sd + 3),
            P("d%d_q64_k1024_rising" % D, 1, 2, 64, 1024, D, mode="rising", seed=sd + 4),
            P("d%d_q1_k65_dominant_last_bnhd" % D, 1, 4, 1, 65, D, mode="dominant", dom="last", layout="bnhd", seed=sd + 5),
            P("d%d_q65_k4096_random" % D, 1, 1, 65, 4096, D, seed=sd + 6),
        ]
    cases += [
        P("d40_q63_k1_single_key", 2, 2, 63, 1, 40, seed=1),
        P("d80_q1_k1_bnhd", 1, 1, 1, 1, 80, layout="bnhd", seed=2),
        P("d64_q64_k64_flat", 2, 2, 64, 64, 64, mode="flat", seed=3),
        P("d40_q200_k130_flat_bnhd", 1, 2, 200, 130, 40, mode="flat", layout="bnhd", seed=4),
        P("d40_q65_k4096_dominant_first", 1, 2, 65, 4096, 40, mode="dominant", seed=5),
        P("d80_q63_k4033_dominant_last_kvpair", 1, 1, 63, 4033, 80, mode="dominant", dom="last", layout="kv_pair", seed=6),
        P("d160_q64_k77_dominant_first_kvpair", 2, 2, 64, 77, 160, mode="dominant", layout="kv_pair", seed=7),
        P("d64_q65_k130_dominant_last_scale", 2, 1, 65, 130, 64, mode="dominant", dom="last", scale=0.0917, seed=8),
        P("d40_q200_k1024_rising_bnhd", 1, 2, 200, 1024, 40, mode="rising", layout="bnhd", seed=9),
        P("d128_q65_k130_falling", 2, 2, 65, 130, 128, mode="falling", seed=10),
        P("d40_q64_k4096_falling_kvpair", 1, 1, 64, 4096, 40, mode="falling", layout="kv_pair", seed=11),
        P("d80_q65_k1024_large", 1, 2, 65, 1024, 80, mode="large", seed=12),
        P("d40_q200_k77_large_kvpair", 2, 1, 200, 77, 40, mode="large", layout="kv_pair", seed=13),
        P("d32_q63_k4096_large_scale", 1, 1, 63, 4096, 32, mode="large", scale=0.0917, seed=14),
        P("d40_q65_k130_constant_v", 2, 2, 65, 130, 40, mode="constant_v", seed=15),
        P("d160_q64_k4096_constant_v_bnhd", 1, 1, 64, 4096, 160, mode="constant_v", layout="bnhd", seed=16),
        P("d80_q200_k77_constant_v_kvpair", 1, 2, 200, 77, 80, mode="constant_v", layout="kv_pair", seed=17),
        P("d40_q65_k64_random_b3_h2", 3, 2, 65, 64, 40, seed=18),
    ]
    return cases


SATTN_CASES = _sattn_cases()


def sattn_values(spec: SAttnSpec, device) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """float64 q [B, heads, Nq, D], k, v [B, heads, Nk, D] of the case's mode; independent of the layout."""
    gen = torch.Generator(device=device)
    gen.manual_seed(spec.seed)
    B, H, Nq, Nk, D = spec.B, spec.heads, spec.Nq, spec.Nk, spec.D
    sc = spec.s32

    def randn(*shape):
        return torch.randn(*shape, generator=gen, device=device, dtype=torch.float64)

    q, k, v = randn(B, H, Nq, D), randn(B, H, Nk, D), randn(B, H, Nk, D)
    d = torch.where(randn(D) < 0, -1.0, 1.0) / D ** 0.5                                  # a unit direction
    if spec.mode in ("random", "constant_v"):
        q = q * 2 / (sc * D ** 0.5)                                                      # scaled logits ~ N(0, 4)
        if spec.mode == "constant_v":
            v = v[:, :, :1].expand(B, H, Nk, D).clone()
        return q, k, v
    if spec.mode == "flat":
        return torch.zeros_like(q), k, v
    # q ~ d, k_j ~ (t_j / scale) d: the scaled logits are about t_j (plus a little noise)
    blk = (torch.arange(Nk, device=device) // BNK).double()
    noise = randn(B, H, 1, Nk)
    if spec.mode == "dominant":
        t = 0.5 * noise
        t[..., spec.dom_key] = 12.0
    elif spec.mode == "rising":
        t = 8.0 * blk + noise
    elif spec.mode == "falling":
        t = -3.0 * blk + noise
    elif spec.mode == "large":
        a = (torch.rand(B, H, Nq, 1, generator=gen, device=device, dtype=torch.float64) * 2 - 1) * 80 ** 0.5
        tt = (torch.rand(B, H, Nk, 1, generator=gen, device=device, dtype=torch.float64) * 2 - 1) * 80 ** 0.5
        return a * d + 0.01 * q / D ** 0.5, tt * d / sc + 0.01 * k / (sc * D ** 0.5), v
    else:
        raise ValueError(spec.mode)
    q = d + 0.05 * q / D ** 0.5
    k = t.transpose(2, 3) * d / sc + 0.05 * k / (sc * D ** 0.5)
    return q, k, v


@dataclass
class SAttnCase:
    spec: SAttnSpec
    dtype: torch.dtype
    q: torch.Tensor                 # [B, heads, Nq, D] views of the input buffers
    k: torch.Tensor
    v: torch.Tensor
    bufs: Dict[str, torch.Tensor]   # the input buffers (their padding columns hold random bytes)
    out: Guarded
    o4: torch.Tensor                # [B, heads, Nq, D] view of out's window

    def buffers(self):
        return {"out": self.out}

    def inputs(self):
        return dict(self.bufs)


def _bnhd(vals: torch.Tensor, dtype, gen) -> Tuple[torch.Tensor, torch.Tensor]:
    """A "b n (h d)" buffer with a head pitch of D + 8 holding vals [B, H, N, D], and the [B, H, N, D] view of it."""
    B, H, N, D = vals.shape
    buf = _random_bits((B, N, H, D + GUARD_COLS), dtype, vals.device, gen)
    buf[..., :D] = vals.permute(0, 2, 1, 3).to(dtype)
    return buf, buf[..., :D].permute(0, 2, 1, 3)


def make_sattn(spec: SAttnSpec, dtype: torch.dtype, device, layout: Optional[str] = None) -> SAttnCase:
    """`layout` overrides the spec's (the same values in another layout)."""
    layout = layout or spec.layout
    qv, kv_, vv = sattn_values(spec, device)
    gen = torch.Generator(device=device)
    gen.manual_seed(spec.seed + 7919)
    B, H, Nq, Nk, D = spec.B, spec.heads, spec.Nq, spec.Nk, spec.D
    if layout == "bhnd":
        q, k, v = (t.to(dtype).contiguous() for t in (qv, kv_, vv))
        bufs = {"q": q, "k": k, "v": v}
        out = guarded((B, H, Nq, D), dtype, device, gen, "bhnd")
        o4 = out.view
    else:
        qb, q = _bnhd(qv, dtype, gen)
        if layout == "bnhd":
            kb, k = _bnhd(kv_, dtype, gen)
            vb, v = _bnhd(vv, dtype, gen)
            bufs = {"q": qb, "k": kb, "v": vb}
        else:
            pair = torch.cat([kv_.permute(0, 2, 1, 3).reshape(B, Nk, H * D), vv.permute(0, 2, 1, 3).reshape(B, Nk, H * D)], dim=2)
            pair = pair.to(dtype).contiguous()
            k = pair[..., :H * D].view(B, Nk, H, D).permute(0, 2, 1, 3)
            v = pair[..., H * D:].view(B, Nk, H, D).permute(0, 2, 1, 3)
            bufs = {"q": qb, "kv": pair}
        out = guarded((B, Nq, H, D + GUARD_COLS), dtype, device, gen, "bnhd")
        o4 = out.view[..., :D].permute(0, 2, 1, 3)
    return SAttnCase(spec, dtype, q, k, v, bufs, out, o4)


def sattn_descriptor(case: SAttnCase, scale: Optional[float] = None):
    """The sige_sparse_attention_t of the case (strides 0 on size-1 dims); d._keep holds the case."""
    from sige_b200 import _cabi

    s = case.spec
    d = _cabi.SparseAttention()
    d.q, d.k, d.v, d.out = case.q.data_ptr(), case.k.data_ptr(), case.v.data_ptr(), case.o4.data_ptr()
    d.B, d.heads, d.Nq, d.Nk, d.D = s.B, s.heads, s.Nq, s.Nk, s.D
    for name, t in (("q_stride", case.q), ("k_stride", case.k), ("v_stride", case.v), ("out_stride", case.o4)):
        assert t.stride(3) == 1
        st = getattr(d, name)
        for i in range(3):
            st[i] = int(t.stride(i)) if t.shape[i] > 1 else 0
    d.scale = s.s32 if scale is None else scale
    d.dtype = _code(case.dtype)
    d.flags = 0
    d._keep = case
    return d


def sattn_call(case: SAttnCase, lib, d=None):
    from ctypes import byref

    return lib.sige_sparse_attention(byref(sattn_descriptor(case) if d is None else d), _stream())


def sattn_reference(case: SAttnCase, chunk: int = 16) -> List[Expect]:
    """out_i = sum_j s_ij v_j, s_i = softmax_j(scale q_i . k_j), in float64 on the 16-bit operands and the descriptor's fp32 scale.

    How the kernel computes it (sparse_attention.cu): fp32 mma logits l_j; per key block t of 64 the running maximum m_t;
    numerators p_j = ex2.approx.ftz(fmaf(l_j, c, -fl(m_t c))), c = fl32(scale log2 e); the block's o and l are multiplied by
    corr = ex2(fl(m_{t-1} - m_t) c) before P V is added; P is rounded to 16 bits for P V while l sums the unrounded fp32 p_j; at
    the end out = o * (1 / l), rounded once.  Every factor a key's weight picks up telescopes to 2^(c (l_j - M)), M the final
    maximum, so a relative error e_j on key j's weight that reaches numerator and denominator alike moves the result by
    sum_j s_j e_j (v_j - want) (centred on want).  Per key j of block t:
        e_j <= EX2_REL (T - t)                       ex2.approx of p_j and of the corr of each later block
             + U32 c (|m_t| + |l_j - m_t|)            the rounding of fl(m_t c) and of the fmaf argument
             + 2 U32 c (M - m_t)                      the roundings of the later corr arguments (their differences telescope)
             + 2 U32 scale |l_j - M|                  c against scale * log2 e: two fp32 roundings
             + 2 scale dl                             the fp32 logit's error, dl = ACC * max_j sum_c |q_c k_jc|
    The P rounding is NOT centred: P V uses fl16(p_j) = p_j (1 + r_j), l the p_j, so the result moves by sum_j s_j r_j v_j,
    up to u sum_j s_j |v_j| (pinned by the constant_v mode, where every other term vanishes).  An f16 numerator below the normal
    range has an absolute error up to ETA_P instead, weighted by the later corr factors and 1 / l:
    ETA_P sum_j exp(scale (m_t - M)) |v_j| / L.  ftz flushes numerators below 2^-126 (ABS covers them).  The fp32 rest: the P V
    accumulate (ACC mag, mag = sum_j s_j |v_j|), one rounding of o per block (o *= corr), the fmaf of l per block, the 16-term
    sum of a lane's numerators and the 4-lane sum of l, the reciprocal and the product o * inv: (2T + 24) U32 mag.  The
    output is rounded once: u |want|."""
    s = case.spec
    u = ROUNDOFF[case.dtype]
    sc = s.s32
    c = sc * LOG2E
    T = s.blocks
    B, H, Nq, Nk, D = s.B, s.heads, s.Nq, s.Nk, s.D
    q, k, v = case.q.double(), case.k.double(), case.v.double()
    want = torch.empty(B, H, Nq, D, dtype=torch.float64, device=q.device)
    bound = torch.empty_like(want)
    tj = torch.arange(Nk, device=q.device) // BNK
    for b in range(B):
        for h in range(H):
            kk, vv = k[b, h], v[b, h]
            for i0 in range(0, Nq, chunk):
                qq = q[b, h, i0:i0 + chunk]
                S = qq @ kk.t()                                                           # [n, Nk] unscaled logits
                n = S.shape[0]
                dl = ACC * (qq.abs() @ kk.abs().t()).amax(dim=1, keepdim=True)
                padded = torch.full((n, T * BNK), -math.inf, dtype=torch.float64, device=q.device)
                padded[:, :Nk] = S
                run = padded.view(n, T, BNK).amax(dim=2).cummax(dim=1).values            # m_t, the running maximum
                M = run[:, -1:]
                mt = run[:, tj]                                                           # [n, Nk]
                e = torch.exp(sc * (S - M))
                L = e.sum(dim=1, keepdim=True)
                sm = e / L
                w = sm @ vv
                ce = (EX2_REL * (T - tj) + U32 * c * (mt.abs() + (S - mt).abs()) + 2 * U32 * c * (M - mt)
                      + 2 * U32 * sc * (S - M).abs() + 2 * sc * dl)
                cen = torch.einsum("qk,qkd->qd", ce * sm, (vv[None] - w[:, None]).abs())
                mag = sm @ vv.abs()
                eta = ETA_P[case.dtype] * (torch.exp(sc * (mt - M)) / L) @ vv.abs()
                want[b, h, i0:i0 + n] = w
                bound[b, h, i0:i0 + n] = u * w.abs() + u * mag + cen + (ACC + (2 * T + 24) * U32) * mag + eta + ABS
    ex, (wv, wr, bd, rnd) = expect_for("out", case.out, u)
    if case.out.layout == "bhnd":
        view = lambda t: t                                                               # noqa: E731
    else:
        view = lambda t: t[..., :D].permute(0, 2, 1, 3)                                  # noqa: E731
    view(wv)[:], view(wr)[:], view(bd)[:], view(rnd)[:] = want, True, bound, u * want.abs()
    return [ex]


# ----------------------------------------------------------------------------------------------------------------------
# sige_sparse_attention at D = 512 (sparse_attention.cu, namespace wide)
# ----------------------------------------------------------------------------------------------------------------------
WIDE_D = 512
WIDE_BNK = 32                   # keys per ring stage of the wide kernel
WIDE_MAX_CS = 8                 # portable cluster size


def wide_cluster(Nq: int, Nk: int, BH: int, sms: int) -> int:
    """The launcher's cluster size: the smallest power of two that puts about one CTA on every SM, at most one key block per
    CTA and 8 (wide::launch)."""
    ctas = -(-Nq // BM) * BH
    nblk = -(-Nk // WIDE_BNK)
    cs = 1
    while cs < WIDE_MAX_CS and 2 * cs <= nblk and ctas * cs < sms:
        cs *= 2
    return cs


def wide_ranges(Nk: int, cs: int) -> List[Tuple[int, int]]:
    """Key blocks [t0, t1) of each CTA of the cluster, in rank order."""
    nblk = -(-Nk // WIDE_BNK)
    return [(nblk * r // cs, nblk * (r + 1) // cs) for r in range(cs)]


P = SAttnSpec
WIDE_CASES = [
    # cluster sizes at 132 SMs in the comments
    P("q1_k1", 1, 1, 1, 1, 512, seed=1),                                                  # cs 1, one block
    P("q63_k65_bnhd", 1, 1, 63, 65, 512, layout="bnhd", seed=2),                          # cs 2, a key tail of 1 after 2 blocks
    P("q64_k4096", 1, 1, 64, 4096, 512, seed=3),                                          # cs 8
    P("q65_k9216_bnhd", 1, 1, 65, 9216, 512, layout="bnhd", seed=4),                      # cs 8
    P("q800_k4096", 1, 1, 800, 4096, 512, seed=5),                                        # cs 8, 13 query blocks
    P("q800_k9216_bnhd", 1, 1, 800, 9216, 512, layout="bnhd", seed=6),
    P("q64_k1_bnhd", 1, 1, 64, 1, 512, layout="bnhd", seed=7),
    P("q65_k65", 1, 1, 65, 65, 512, seed=8),                                              # cs 2
    P("q1_k4096_bnhd", 1, 1, 1, 4096, 512, layout="bnhd", seed=9),
    P("q63_k9216_falling", 1, 1, 63, 9216, 512, mode="falling", seed=10),                 # 8 ranges across the falling blocks
    P("q65_k4096_dominant_last_bnhd", 1, 1, 65, 4096, 512, mode="dominant", dom="last", layout="bnhd", seed=11),
    P("q800_k65_dominant_first", 1, 1, 800, 65, 512, mode="dominant", seed=12),
    P("q64_k4096_constant_v", 1, 1, 64, 4096, 512, mode="constant_v", seed=13),
    P("b2_q65_k130_bnhd", 2, 1, 65, 130, 512, layout="bnhd", seed=14),                    # cs 4, B * heads 2
    P("q8449_k96_cs1", 1, 1, 8449, 96, 512, seed=15),                                     # cs 1 over 3 blocks: 133 query blocks
    P("q200_k96_falling_cs2", 1, 1, 200, 96, 512, mode="falling", seed=16),              # cs 2: ranges [0, 32) and [32, 96)
    P("q64_k160_dominant_cs4", 1, 1, 64, 160, 512, mode="dominant", seed=17),             # cs 4: the dominant key in range 0 of 4
    P("b2h2_q64_k1000_cs8", 2, 2, 64, 1000, 512, seed=18),                                # cs 8, B * heads 4, a key tail of 8
    P("q64_k96_constant_v_cs2", 1, 1, 64, 96, 512, mode="constant_v", seed=19),
]
del P


def wide_sattn_reference(case: SAttnCase, sms: int, chunk: int = 16) -> List[Expect]:
    """out_i = softmax_j(scale q_i . k_j) v_j in float64, with the bound of the wide kernel's own algorithm.

    How it computes (sparse_attention.cu, wide::kernel): the key range is split over a cluster of cs CTAs (wide_cluster), CTA r
    taking the 32-key blocks [t0, t1) of wide_ranges; each runs its own online softmax from t0: fp32 logits l_j, the running
    maximum m_t of its blocks t0 .. t, p_j = ex2.approx(fmaf(l_j, c, -fl(m_t c))), corr = ex2(fl(fl(m_{t-1} - m_t) c)) on o
    and on l = fmaf(l, corr, sum); P rounded to 16 bits for P V.  The merge takes M = max_r m_r (m_r: CTA r's last maximum),
    e_r = ex2(fl(fl(m_r - M) c)), L = sum_r fmaf(e_r, l_r), inv = fl(1 / L), w_r = fl(e_r inv) and out = sum_r fmaf(w_r, O_r),
    peers in rank order, rounded once.  Per key j of block t in CTA r, the relative error of its weight that reaches numerator
    and denominator alike (centred, as in sattn_reference):
        e_j <= EX2_REL (t1 - t + 1)                   ex2 of p_j, of the t1 - 1 - t later corrs and of the merge weight
             + U32 c (|m_t| + |l_j - m_t|)            the rounding of fl(m_t c) and of the fmaf argument
             + 2 U32 c (m_r - m_t)                    the later corr arguments of the CTA (their differences telescope)
             + 2 U32 c (M - m_r)                      the merge weight's argument: the difference and the product, rounded
             + 2 U32 scale |l_j - M|                  c against scale * log2 e
             + 2 scale dl                             the fp32 logit's error
    Uncentred: the P rounding u sum_j s_j |v_j|, the f16 subnormal numerators ETA_P sum_j 2^(c (m_t - M)) |v_j| / L, the
    per-CTA fp32 rest (2 T + 24) U32 mag with T the most blocks of a CTA, and the merge's (2 cs + 2) U32 mag: the cs fmaf of
    L, the reciprocal, the product e_r inv and the cs fmaf of the output.  The output is rounded once: u |want|."""
    s = case.spec
    assert s.D == WIDE_D, s.name
    u = ROUNDOFF[case.dtype]
    sc = s.s32
    c = sc * LOG2E
    B, H, Nq, Nk, D = s.B, s.heads, s.Nq, s.Nk, s.D
    cs = wide_cluster(Nq, Nk, B * H, sms)
    ranges = wide_ranges(Nk, cs)
    T = max(t1 - t0 for t0, t1 in ranges)
    nblk = -(-Nk // WIDE_BNK)
    dev = case.q.device
    tj = torch.arange(Nk, device=dev) // WIDE_BNK                                          # block of each key
    rank = torch.zeros(nblk, dtype=torch.long, device=dev)
    t1_of = torch.zeros(nblk, dtype=torch.long, device=dev)
    for r, (t0, t1) in enumerate(ranges):
        rank[t0:t1], t1_of[t0:t1] = r, t1
    rj, t1j = rank[tj], t1_of[tj]
    q, k, v = case.q.double(), case.k.double(), case.v.double()
    want = torch.empty(B, H, Nq, D, dtype=torch.float64, device=dev)
    bound = torch.empty_like(want)
    for b in range(B):
        for h in range(H):
            kk, vv = k[b, h], v[b, h]
            for i0 in range(0, Nq, chunk):
                qq = q[b, h, i0:i0 + chunk]
                S = qq @ kk.t()
                n = S.shape[0]
                dl = ACC * (qq.abs() @ kk.abs().t()).amax(dim=1, keepdim=True)
                padded = torch.full((n, nblk * WIDE_BNK), -math.inf, dtype=torch.float64, device=dev)
                padded[:, :Nk] = S
                bm = padded.view(n, nblk, WIDE_BNK).amax(dim=2)                           # block maxima
                run = torch.empty_like(bm)
                mr = torch.empty(n, cs, dtype=torch.float64, device=dev)
                for r, (t0, t1) in enumerate(ranges):
                    run[:, t0:t1] = bm[:, t0:t1].cummax(dim=1).values                    # each CTA's running maximum from t0
                    mr[:, r] = run[:, t1 - 1]
                M = mr.amax(dim=1, keepdim=True)
                mt, mrj = run[:, tj], mr[:, rj]                                           # [n, Nk]
                e = torch.exp(sc * (S - M))
                L = e.sum(dim=1, keepdim=True)
                sm = e / L
                w = sm @ vv
                ce = (EX2_REL * (t1j - tj + 1) + U32 * c * (mt.abs() + (S - mt).abs()) + 2 * U32 * c * (mrj - mt)
                      + 2 * U32 * c * (M - mrj) + 2 * U32 * sc * (S - M).abs() + 2 * sc * dl)
                cen = torch.einsum("qk,qkd->qd", ce * sm, (vv[None] - w[:, None]).abs())
                mag = sm @ vv.abs()
                eta = ETA_P[case.dtype] * (torch.exp(sc * (mt - M)) / L) @ vv.abs()
                want[b, h, i0:i0 + n] = w
                bound[b, h, i0:i0 + n] = (u * w.abs() + u * mag + cen + (ACC + (2 * T + 24 + 2 * cs + 2) * U32) * mag + eta + ABS)
    ex, (wv, wr, bd, rnd) = expect_for("out", case.out, u)
    view = (lambda t: t) if case.out.layout == "bhnd" else (lambda t: t[..., :D].permute(0, 2, 1, 3))      # noqa: E731
    view(wv)[:], view(wr)[:], view(bd)[:], view(rnd)[:] = want, True, bound, u * want.abs()
    return [ex]


def wide_sattn_emulate(case: SAttnCase, sms: int) -> torch.Tensor:
    """The wide kernel's arithmetic in float32, in its order (blocks of 32 keys, the cluster's key ranges, each range's online
    softmax, the merge in rank order), on the case's 16-bit operands: [B, heads, Nq, D] float64 of the rounded output.  The fp32
    logits are the exact dot products rounded once, ex2.approx is exp2 in float32, each fmaf one rounding of the float64 value."""
    s = case.spec
    f32 = torch.float32
    c = float(np.float32(s.s32 * LOG2E))
    cs = wide_cluster(s.Nq, s.Nk, s.B * s.heads, sms)
    out = torch.empty(s.B, s.heads, s.Nq, s.D, dtype=torch.float64, device=case.q.device)

    def fma(a, b, z):
        return (a.double() * b.double() + z.double()).float()

    for b in range(s.B):
        for h in range(s.heads):
            S = (case.q[b, h].double() @ case.k[b, h].double().t()).float()
            v = case.v[b, h].float()
            parts = []
            for t0, t1 in wide_ranges(s.Nk, cs):
                m = torch.full((s.Nq,), -math.inf, dtype=f32)
                l = torch.zeros(s.Nq, dtype=f32)
                o = torch.zeros(s.Nq, s.D, dtype=f32)
                for t in range(t0, t1):
                    j0, j1 = t * WIDE_BNK, min((t + 1) * WIDE_BNK, s.Nk)
                    sb = S[:, j0:j1]
                    m_new = torch.maximum(m, sb.amax(dim=1))
                    corr = torch.exp2((m - m_new) * c)
                    mb = m_new * c
                    p = torch.exp2(fma(sb, torch.tensor(c, dtype=f32), -mb[:, None]))
                    l = fma(l, corr, p.sum(dim=1))
                    o = o * corr[:, None] + p.to(case.dtype).float() @ v[j0:j1]
                    m = m_new
                parts.append((m, l, o))
            M = torch.stack([pm for pm, _, _ in parts]).amax(dim=0)
            L = torch.zeros(s.Nq, dtype=f32)
            es = []
            for pm, pl, _ in parts:
                e = torch.exp2((pm - M) * c)
                es.append(e)
                L = fma(e, pl, L)
            inv = 1.0 / L
            acc = torch.zeros(s.Nq, s.D, dtype=f32)
            for e, (_, _, po) in zip(es, parts):
                acc = fma((e * inv)[:, None], po, acc)
            out[b, h] = acc.to(case.dtype).double()
    return out


# ----------------------------------------------------------------------------------------------------------------------
# sige_spade_modulate
# ----------------------------------------------------------------------------------------------------------------------
SPADE_VEC = {torch.float32: 4, torch.float16: 8, torch.bfloat16: 8}
SPADE_THREADS = 256
SPADE_BLOCKS_PER_SM = 16


def spade_blocks(items: int, sms: int) -> int:
    """The launcher's grid: one thread per 16-byte channel vector, at most 16 CTAs of 256 per SM (a grid-stride loop beyond)."""
    return (items + 255) // 256 if items + 255 < SPADE_BLOCKS_PER_SM * sms * SPADE_THREADS else SPADE_BLOCKS_PER_SM * sms


def spade_iterations(items: int, sms: int) -> int:
    """Trips of the grid-stride loop of the busiest thread."""
    return -(-items // (spade_blocks(items, sms) * SPADE_THREADS))


@dataclass(frozen=True)
class SpadeSpec:
    """C = 0: the dtype's minimum vector (4 for f32, 8 for 16 bits).  x is a channel window of a (C + 2 vec)-channel pixel,
    gamma and beta the two halves of a [pixels, 2C] buffer, out has a pixel stride of C + vec (the gap is guard band).
    identity: gamma = beta = 0, slope 1."""
    name: str
    C: int
    pixels: int
    slope: float = 0.2
    identity: bool = False
    seed: int = 0

    def channels(self, dtype) -> int:
        return self.C or SPADE_VEC[dtype]


SPADE_CASES = (
    [SpadeSpec("c%s_p%d_slope%g" % (C or "vec", p, sl), C, p, sl, seed=10 * i + j)
     for i, (C, p) in enumerate(((0, 257), (64, 333), (256, 1), (256, 40))) for j, sl in enumerate((1.0, 0.2, 0.0))]
    + [
        SpadeSpec("c64_p70000_grid_stride", 64, 70000, 0.2, seed=101),
        SpadeSpec("identity_c64_p333", 64, 333, 1.0, identity=True, seed=102),
        SpadeSpec("identity_cvec_p1", 0, 1, 1.0, identity=True, seed=103),
    ]
)


@dataclass
class SpadeCase:
    spec: SpadeSpec
    dtype: torch.dtype
    xbuf: torch.Tensor              # [P, C + 2 vec]
    gb: torch.Tensor                # [P, 2C]
    out: Guarded                    # [P, C + vec]

    @property
    def vec(self):
        return SPADE_VEC[self.dtype] if self.dtype in SPADE_VEC else 4

    @property
    def C(self):
        return self.gb.shape[1] // 2

    @property
    def x(self):
        return self.xbuf[:, self.vec:self.vec + self.C]

    @property
    def gamma(self):
        return self.gb[:, :self.C]

    @property
    def beta(self):
        return self.gb[:, self.C:]

    def buffers(self):
        return {"out": self.out}

    def inputs(self):
        return {"x": self.xbuf, "gamma_beta": self.gb}


def make_spade(spec: SpadeSpec, dtype: torch.dtype, device) -> SpadeCase:
    gen = torch.Generator(device=device)
    gen.manual_seed(spec.seed)
    vec = SPADE_VEC.get(dtype, 4)
    C, P = spec.C or vec, spec.pixels

    def randn(*shape, scale=1.0):
        return (torch.randn(*shape, generator=gen, device=device, dtype=torch.float64) * scale).to(dtype)

    xbuf = randn(P, C + 2 * vec)
    gb = torch.zeros(P, 2 * C, dtype=dtype, device=device) if spec.identity else randn(P, 2 * C, scale=0.6)
    return SpadeCase(spec, dtype, xbuf, gb, guarded((P, C + vec), dtype, device, gen, "pc"))


def spade_call(case: SpadeCase, lib):
    C, v = case.C, case.vec
    return lib.sige_spade_modulate(case.x.data_ptr(), C + 2 * v, case.gamma.data_ptr(), 2 * C, case.beta.data_ptr(), 2 * C,
                                   case.out.view.data_ptr(), C + v, case.spec.pixels, C, float(case.spec.slope), _code(case.dtype),
                                   _stream())


def spade_reference(case: SpadeCase) -> List[Expect]:
    u = ROUNDOFF[case.dtype]
    a = (1 + case.gamma.float()).double()                                                 # the kernel's 1.0f + g, in fp32
    f = case.x.double() * a + case.beta.double()
    slope = float(np.float32(case.spec.slope))
    want = torch.where(f > 0, f, f * slope)
    bound = torch.zeros_like(want) if case.spec.identity else (u + 2 * U32) * want.abs() + HALF_SUBNORMAL[case.dtype] + 2.0 ** -149
    e, (w, wr, bd, rnd) = expect_for("out", case.out, u)
    C = case.C
    w[:, :C], wr[:, :C], bd[:, :C] = want, True, bound
    rnd[:, :C] = torch.zeros_like(want) if case.spec.identity else u * want.abs() + HALF_SUBNORMAL[case.dtype]
    return [e]


# ----------------------------------------------------------------------------------------------------------------------
# sige_gather / sige_scatter / sige_scatter_gather / sige_scatter_with_block_residual in f32, f16 and bf16
# ----------------------------------------------------------------------------------------------------------------------
ACT_IDENTITY, ACT_SWISH = 0, 1
TILE_OPS = ("gather", "scatter", "scatter_gather", "swbr")
# a broadcast operand's shape: which of (B, C, H, W) it spans (the others are 1)
BCAST_SHAPES = ((0, 0, 0, 0), (1, 0, 0, 0), (0, 1, 0, 0), (1, 1, 0, 0), (0, 0, 1, 1), (0, 1, 1, 1), (1, 1, 1, 1))


def swish_rel(z):
    """Relative error of the fast swish z / (1 + __expf(-z)) with __fdividef: __expf rounds its argument times log2(e) (U32 |z|
    relative in the result) and ex2.approx adds 2^-22; 1 + e rounds once and __fdividef is within 2 ulp.  Doubled."""
    return (16 + 2 * z.abs()) * U32


# expf's maximum error, in ulps of its result, over its whole range (CUDA C++ Programming Guide, "Mathematical Functions":
# single-precision functions without -use_fast_math)
EXPF_ULPS = 2
# The accurate swish z / (1 + expf(-z)) of f32 storage, relative to z sigmoid(z): t = expf(-z) is within EXPF_ULPS ulps of e^-z,
# a relative error of at most EXPF_ULPS * 2^-23 = 2 EXPF_ULPS U32 (an fp32 ulp is at most 2^-23 of the value); 1 + t rounds once
# (U32) and moves by less than t's relative error, since t / (1 + t) < 1; the IEEE division rounds once more (U32).  First order
# 2 EXPF_ULPS + 2 = 6 U32; one U32 more covers the products of these terms.  Much tighter than swish_rel, so f32 switched to the
# fast intrinsics would not pass unnoticed.
SWISH_ACCURATE_REL = (2 * EXPF_ULPS + 3) * U32


@dataclass(frozen=True)
class TileSpec:
    """One tile-op launch on a [B, C, H, W] tensor (NCHW or NHWC) and its tile stacks.

    gather: 6x6 tiles at `N` random origins (many stick out); up = 1 reads a (H/2, W/2) source through nearest x2 up-sampling.
    scatter: Ro x So tiles pasted at (off + origin) / stride (C division) + r, origins chosen so that no two tiles write the same
    pixel; the copy form writes the whole destination (y's copy), the in-place form only the tiles.  scatter_gather: 6x6 tiles
    whose pixels come from the stack of 4x4 conv outputs (via the map of get_scatter_map) or the cached tensor.  swbr: scatter
    with the cached shortcut output as residual, then 4x4 calibration tiles at raw origins.
    scale / shift / residual: a broadcast shape (BCAST_SHAPES) or None; aff_dt: "f32" or "x" (the launch dtype).
    misalign: the destination one element (4 bytes for f32, 2 for 16 bits) off 16-byte alignment (on NHWC: the scalar path)."""
    name: str
    op: str
    layout: str
    B: int = 2
    C: int = 16
    H: int = 19
    W: int = 22
    N: int = 9
    up: int = 0
    scale: Optional[Tuple[int, int, int, int]] = None
    shift: Optional[Tuple[int, int, int, int]] = None
    aff_dt: str = "f32"
    act: int = ACT_IDENTITY
    act_first: bool = False
    residual: Optional[Tuple[int, int, int, int]] = None
    stride: int = 1
    inplace: bool = False
    misalign: bool = False
    seed: int = 0

    @property
    def identity(self) -> bool:
        """A pure move: no arithmetic at all."""
        return self.scale is None and self.shift is None and self.act == ACT_IDENTITY and self.residual is None and self.op != "swbr"

    @property
    def geometry(self):
        """(Ro, So, off) of the pasted stack: 3x3 stride-1 outputs of 6x6 tiles at offset 1, or stride-2 outputs (2x2 of 5x5 tiles)
        at offset 0, so that origins -1 and -2 land on output rows 0 and -1 (C division truncates)."""
        return (4, 1) if self.stride == 1 else (2, 0)


def tile_path(spec: TileSpec, dtype) -> str:
    """Which kernel variant the launcher picks (tile_ops.cu launch_*): NCHW; NHWC with 16-byte vectors when C is a multiple
    of the vector and every pointer is 16-byte aligned; else NHWC scalar."""
    if spec.layout == "nchw":
        return "nchw"
    return "scalar" if (spec.C % (16 // _esize(dtype)) or spec.misalign) else "vec"


def _cdiv(a: int, b: int) -> int:
    """C integer division (truncates toward zero)."""
    return int(a / b) if a * b >= 0 else -(-a // b)


def _paste_origins(spec: TileSpec, rng, n: int, R: int, off: int, stride: int, forced=()):
    """Up to n origins whose pasted R x R footprints (in-image pixels) do not overlap: the forced ones first, then random ones
    from a grid that reaches past every border."""
    taken = np.zeros((spec.H, spec.W), bool)
    cand = list(forced)
    hs, ws = np.arange(-3 * stride, stride * spec.H + 2), np.arange(-3 * stride, stride * spec.W + 2)
    cand += [(int(h), int(w)) for h, w in zip(rng.choice(hs, 400), rng.choice(ws, 400))]
    out = []
    for (h, w) in cand:
        h0, w0 = _cdiv(off + h, stride), _cdiv(off + w, stride)
        ys = [y for y in range(h0, h0 + R) if 0 <= y < spec.H]
        xs = [x for x in range(w0, w0 + R) if 0 <= x < spec.W]
        if not ys or not xs or taken[np.ix_(ys, xs)].any():
            continue
        taken[np.ix_(ys, xs)] = True
        out.append((h, w))
        if len(out) == n:
            break
    return out


@dataclass
class TileCase:
    spec: TileSpec
    dtype: torch.dtype
    t: Dict[str, torch.Tensor]              # inputs, in the buffers' physical layout
    idx: Dict[str, torch.Tensor]            # int32 [N, 2] lists ("idx", "idx1"), and "map" for scatter_gather
    bc: Dict[str, torch.Tensor]             # broadcast operands (logical [b, c, h, w] shapes)
    out: Guarded

    def buffers(self):
        return {"out": self.out}

    def inputs(self):
        d = dict(self.t)
        d.update(self.idx)
        d.update({"bc_" + k: v for k, v in self.bc.items()})
        return d

    def logical(self, name: str) -> torch.Tensor:
        """NCHW view of an input (or, name "out", of the destination window)."""
        t = self.out.view if name == "out" else self.t[name]
        return t.permute(0, 3, 1, 2) if self.spec.layout == "nhwc" else t


def _phys(shape, layout):
    n, c, h, w = shape
    return (n, h, w, c) if layout == "nhwc" else (n, c, h, w)


def make_tile(spec: TileSpec, dtype: torch.dtype, device, oracle_safe: bool = False, origins: Optional[Dict[str, list]] = None) -> TileCase:
    """Inputs are drawn before the destination, so two specs that differ only in `misalign` hold the same values.

    origins: the tile lists to use ("idx", and "idx1" for swbr) instead of the drawn ones (spec.N is then not used).

    oracle_safe: drop the tiles whose pasted output starts above or left of the image.  The C oracle, like the reference's CPU
    code it restates, has no lower bound check there (only the CUDA kernels skip negative rows and columns), so it can only
    judge the restatement on the other tiles."""
    def safe(origins, off, stride):
        return [o for o in origins if not oracle_safe or min(_cdiv(off + o[0], stride), _cdiv(off + o[1], stride)) >= 0]

    rng = np.random.default_rng(spec.seed)
    gen = torch.Generator(device=device)
    gen.manual_seed(spec.seed)
    B, C, H, W = spec.B, spec.C, spec.H, spec.W

    def randn(shape, dt=dtype, scale=1.0, offset=0.0):
        return (offset + torch.randn(*shape, generator=gen, device=device, dtype=torch.float64) * scale).to(dt)

    def phys(shape, **kw):
        return randn(_phys(shape, spec.layout), **kw).contiguous()

    t, idx, bc = {}, {}, {}
    aff_dt = torch.float32 if spec.aff_dt == "f32" else dtype
    for name, shp, off_, sc_ in (("scale", spec.scale, 1.0, 0.3), ("shift", spec.shift, 0.0, 0.3), ("residual", spec.residual, 0.0, 1.0)):
        if shp is not None:
            bc[name] = randn(tuple(n if f else 1 for f, n in zip(shp, (B, C, H, W))), dt=aff_dt, scale=sc_, offset=off_)
    if spec.op == "gather":
        o = [(int(h), int(w)) for h, w in zip(rng.integers(-5, H, spec.N), rng.integers(-5, W, spec.N))]
        o = [(-5, -5), (H - 1, W - 1)] + o if origins is None else origins["idx"]
        idx["idx"] = torch.tensor(o, dtype=torch.int32, device=device)
        t["x"] = phys((B, C, H >> spec.up, W >> spec.up))
        N, R = idx["idx"].shape[0], 6
        out_shape = (B * N, C, R, R)
    elif spec.op in ("scatter", "swbr"):
        Ro, off = spec.geometry
        forced = [(-1, 3), (3, -2), (-2, -1), (-1, -1)] if spec.stride == 2 else [(-1, -1), (H - 2, W - 3)]
        o = safe(_paste_origins(spec, rng, spec.N, Ro, off, spec.stride, forced), off, spec.stride) if origins is None else origins["idx"]
        idx["idx"] = torch.tensor(o, dtype=torch.int32, device=device)
        t["x"] = phys((B * len(o), C, Ro, Ro))
        t["y"] = phys((B, C, H, W))
        if spec.op == "swbr":
            o1 = safe(_paste_origins(spec, rng, spec.N, 4, 0, 1, [(-2, -1), (H - 2, W - 1)]), 0, 1) if origins is None else origins["idx1"]
            idx["idx1"] = torch.tensor(o1, dtype=torch.int32, device=device)
            t["x1"] = phys((B * len(o1), C, 4, 4))
            t["y1"] = phys((B, C, H, W))
        out_shape = (B, C, H, W)
    elif spec.op == "scatter_gather":
        o = safe(_paste_origins(spec, rng, spec.N, 4, 1, 1, [(-1, -1), (H - 2, W - 3), (H - 4, -2)]), 1, 1) if origins is None else origins["idx"]
        idx["idx"] = torch.tensor(o, dtype=torch.int32, device=device)
        idx["map"] = scatter_map(H, W, idx["idx"], 4, 4, 1, 1, 1, 1)
        t["x"] = phys((B * len(o), C, 4, 4))
        t["y"] = phys((B, C, H, W))
        out_shape = (B * len(o), C, 6, 6)
    else:
        raise ValueError(spec.op)
    lead = 64 + (_esize(dtype) if spec.misalign else 0)
    out = guarded(_phys(out_shape, spec.layout), dtype, device, gen, spec.layout, lead_bytes=lead)
    return TileCase(spec, dtype, t, idx, bc, out)


def scatter_map(H, W, idx, Ro, So, offH, offW, strideH, strideW) -> torch.Tensor:
    """int32 [H, W, 3]: (tile, r, s) of the pasted output that covers each pixel, -1 elsewhere (get_scatter_map restated)."""
    m = torch.full((H, W, 3), -1, dtype=torch.int32)
    for n, (h, w) in enumerate(idx.tolist()):
        h0, w0 = _cdiv(offH + h, strideH), _cdiv(offW + w, strideW)
        for r in range(Ro):
            for s in range(So):
                if 0 <= h0 + r < H and 0 <= w0 + s < W:
                    m[h0 + r, w0 + s] = torch.tensor([n, r, s], dtype=torch.int32)
    return m.to(idx.device)


def _bcast_struct(t: Optional[torch.Tensor]):
    from sige_b200 import _cabi

    if t is None:
        return None
    b = _cabi.Bcast()
    b.ptr = t.data_ptr()
    for d in range(4):
        b.dims[d], b.stride[d] = t.shape[d], t.stride(d)
    b.dtype = _code(t.dtype)
    return b


def tile_call(case: TileCase, lib, keep: list = None):
    """Calls the case's C-ABI entry point on the current stream; returns the status."""
    from ctypes import byref

    s = case.spec
    lay = 1 if s.layout == "nhwc" else 0
    dt = _code(case.dtype)
    B, C, H, W = s.B, s.C, s.H, s.W
    bs = {k: _bcast_struct(v) for k, v in case.bc.items()}
    if keep is not None:
        keep.append(bs)
    ref = lambda k: byref(bs[k]) if k in bs else None                                    # noqa: E731
    idx = case.idx["idx"]
    N = idx.shape[0]
    outp = case.out.view.data_ptr()
    if s.op == "gather":
        return lib.sige_gather_upsampled(case.t["x"].data_ptr(), dt, lay, B, C, H, W, s.up, 6, 6, idx.data_ptr(), N, ref("scale"),
                                         ref("shift"), s.act, int(s.act_first), outp, _stream())
    Ro, off = s.geometry
    if s.op == "scatter":
        y = None if s.inplace else case.t["y"].data_ptr()
        return lib.sige_scatter(case.t["x"].data_ptr(), y, outp, dt, lay, B, C, H, W, Ro, Ro, off, off, s.stride, s.stride, idx.data_ptr(),
                                N, ref("residual"), _stream())
    if s.op == "scatter_gather":
        return lib.sige_scatter_gather(case.t["x"].data_ptr(), case.t["y"].data_ptr(), dt, lay, B, C, H, W, 4, 4, 6, 6, idx.data_ptr(), N,
                                       case.idx["map"].data_ptr(), ref("scale"), ref("shift"), s.act, int(s.act_first), outp, _stream())
    idx1 = case.idx["idx1"]
    return lib.sige_scatter_with_block_residual(case.t["x"].data_ptr(), case.t["y"].data_ptr(), case.t["x1"].data_ptr(),
                                                case.t["y1"].data_ptr(), outp, dt, lay, B, C, H, W, Ro, Ro, 4, 4, off, off, s.stride,
                                                s.stride, idx.data_ptr(), N, idx1.data_ptr(), idx1.shape[0], _stream())


def _bc(case: TileCase, name: str) -> Optional[torch.Tensor]:
    t = case.bc.get(name)
    return None if t is None else t.double()


def affine_act_bound(z: torch.Tensor, scale, shift, act: int, act_first: bool, dtype):
    """The float64 value of the kernels' affine_act (common.cuh) and a bound on the fp32 evaluation's error.  The kernels
    evaluate swish accurately for f32 storage and with the fast intrinsics for 16-bit storage (tile_ops.cu kFast)."""
    err = torch.zeros_like(z)

    def affine(z, err):
        if scale is not None:
            z = scale * z
            err = scale.abs() * err + U32 * z.abs()
        if shift is not None:
            z = shift + z
            err = err + U32 * z.abs()
        return z, err

    if not act_first:
        z, err = affine(z, err)
    if act == ACT_SWISH:
        y = z * torch.sigmoid(z)
        rel = SWISH_ACCURATE_REL if dtype == torch.float32 else swish_rel(z)
        err = SWISH_LIP * err + rel * y.abs()
        z = y
    if act_first:
        z, err = affine(z, err)
    return z, err


def _stack_origins(idx: torch.Tensor, B: int, R: int):
    """Per stack row (b, n) and tile pixel (r, s): image row / column [B*N, R] and the batch index [B*N]."""
    N = idx.shape[0]
    i = idx.long().repeat(B, 1)                                                           # [B*N, 2]
    d = torch.arange(R, device=idx.device)
    return i[:, :1] + d, i[:, 1:] + d, torch.arange(B * N, device=idx.device) // N


def tile_reference(case: TileCase) -> List[Expect]:
    s = case.spec
    u = ROUNDOFF[case.dtype]
    eta = HALF_SUBNORMAL[case.dtype]
    B, C, H, W = s.B, s.C, s.H, s.W
    e, (want_p, wr_p, bd_p, rnd_p) = expect_for("out", case.out, u)
    perm = (lambda t: t.permute(0, 3, 1, 2)) if s.layout == "nhwc" else (lambda t: t)   # noqa: E731
    want, written, bound, rnd = perm(want_p), perm(wr_p), perm(bd_p), perm(rnd_p)
    dev = want.device

    def finish(val, err, where=None, exact=None):
        """val / err [.., C, .., ..] logical; the element's rounding only where arithmetic happened (not on `exact`)."""
        r = torch.zeros_like(val) if s.identity else u * val.abs() + eta
        if exact is not None:
            r = torch.where(exact, torch.zeros_like(r), r)
        if where is None:
            want[:], written[:], bound[:], rnd[:] = val, True, r + err, r
        else:
            want[where], written[where], bound[where], rnd[where] = val[where], True, (r + err)[where], r[where]

    if s.op in ("gather", "scatter_gather"):
        idx = case.idx["idx"]
        hh, ww, bi = _stack_origins(idx, B, 6)                                           # [BN, 6]
        inside = ((hh >= 0) & (hh < H))[:, :, None] & ((ww >= 0) & (ww < W))[:, None, :]  # [BN, 6, 6]
        hc, wc = hh.clamp(0, H - 1), ww.clamp(0, W - 1)
        if s.op == "gather":
            x = case.logical("x").double()
            z = x[bi[:, None, None], :, (hc >> s.up)[:, :, None], (wc >> s.up)[:, None, :]]          # [BN, 6, 6, C]
        else:
            x, y = case.logical("x").double(), case.logical("y").double()
            m = case.idx["map"].long()[hc[:, :, None], wc[:, None, :]]                   # [BN, 6, 6, 3]
            N = idx.shape[0]
            from_x = m[..., 0] >= 0
            row = bi[:, None, None] * N + m[..., 0].clamp(min=0)
            zx = x[row, :, m[..., 1].clamp(min=0), m[..., 2].clamp(min=0)]
            zy = y[bi[:, None, None], :, hc[:, :, None], wc[:, None, :]]
            z = torch.where(from_x[..., None], zx, zy)
        z = z.permute(0, 3, 1, 2)                                                         # [BN, C, 6, 6]

        def at(name):
            t = _bc(case, name)
            if t is None:
                return None
            t = t.expand(B, C, H, W)
            return t[bi[:, None, None], :, hc[:, :, None], wc[:, None, :]].permute(0, 3, 1, 2)

        val, err = affine_act_bound(z, at("scale"), at("shift"), s.act, s.act_first, case.dtype)
        ins = inside[:, None].expand_as(val)
        val, err = torch.where(ins, val, torch.zeros((), dtype=val.dtype, device=dev)), torch.where(ins, err, torch.zeros((), dtype=val.dtype, device=dev))
        finish(val, err, exact=~ins)                                                   # zeros outside the image: exact
        return [e]

    # scatter / swbr: the pasted pixels
    Ro, off = s.geometry
    idx = case.idx["idx"]
    N = idx.shape[0]
    x = case.logical("x").double()
    paste = torch.zeros(B, H, W, dtype=torch.bool, device=dev)
    src = torch.zeros(B, C, H, W, dtype=torch.float64, device=dev)
    for n, (h, w) in enumerate(idx.tolist()):
        h0, w0 = _cdiv(off + h, s.stride), _cdiv(off + w, s.stride)
        ys, xs = slice(max(h0, 0), min(h0 + Ro, H)), slice(max(w0, 0), min(w0 + Ro, W))
        if ys.start >= ys.stop or xs.start >= xs.stop:
            continue
        assert not paste[:, ys, xs].any(), "case %s: two tiles paste the same pixel" % s.name
        paste[:, ys, xs] = True
        rows = torch.arange(B, device=dev) * N + n
        src[:, :, ys, xs] = x[rows][:, :, ys.start - h0:ys.stop - h0, xs.start - w0:xs.stop - w0]
    pm = paste[:, None].expand(B, C, H, W)
    base = want.clone() if (s.op == "scatter" and s.inplace) else case.logical("y").double()
    if s.op == "scatter":
        if s.residual is None:
            val, err = src, torch.zeros_like(src)
        else:
            val = _bc(case, "residual").expand(B, C, H, W) + src
            err = U32 * val.abs()
        val, err = torch.where(pm, val, base), torch.where(pm, err, torch.zeros_like(err))
        if s.inplace:
            finish(val, err, pm)
        else:
            r = torch.where(pm, u * val.abs() + eta, torch.zeros_like(val)) if not s.identity else torch.zeros_like(val)
            want[:], written[:], bound[:], rnd[:] = val, True, r + err, r
        return [e]
    # swbr: scatter's rounding restated literally (fp32 add, then the launch dtype), then the calibration
    y1 = case.logical("y1")
    stage = torch.where(pm, (y1.float() + src.float()).to(case.dtype).double(), base)
    x1 = case.logical("x1").double()
    idx1 = case.idx["idx1"]
    N1 = idx1.shape[0]
    cal = torch.zeros(B, H, W, dtype=torch.bool, device=dev)
    x1p = torch.zeros(B, C, H, W, dtype=torch.float64, device=dev)
    for n, (h, w) in enumerate(idx1.tolist()):
        ys, xs = slice(max(h, 0), min(h + 4, H)), slice(max(w, 0), min(w + 4, W))
        if ys.start >= ys.stop or xs.start >= xs.stop:
            continue
        assert not cal[:, ys, xs].any(), "case %s: two calibration tiles overlap" % s.name
        cal[:, ys, xs] = True
        x1p[:, :, ys, xs] = x1[torch.arange(B, device=dev) * N1 + n][:, :, ys.start - h:ys.stop - h, xs.start - w:xs.stop - w]
    cm = cal[:, None].expand(B, C, H, W)
    diff = x1p - y1.double()
    val = torch.where(cm, stage + diff, stage)
    r = torch.where(cm, u * val.abs() + eta, torch.zeros_like(val))
    err = torch.where(cm, U32 * (diff.abs() + val.abs()), torch.zeros_like(val))
    want[:], written[:], bound[:], rnd[:] = val, True, r + err, r
    return [e]


def _tile_cases():
    T = TileSpec
    cases = [
        # gather: every path, identity moves, up-sampled sources
        T("g_nchw_identity", "gather", "nchw", seed=1),
        T("g_nhwc_vec_identity", "gather", "nhwc", C=32, seed=2),
        T("g_nhwc_scalar_c12_identity", "gather", "nhwc", C=12, seed=3),
        T("g_nhwc_scalar_misaligned_identity", "gather", "nhwc", C=32, misalign=True, seed=4),
        T("g_nhwc_vec_up", "gather", "nhwc", C=16, H=20, W=22, up=1, seed=5),
        T("g_nchw_up_swish", "gather", "nchw", C=8, H=18, W=24, up=1, act=ACT_SWISH, seed=6),
        T("g_nhwc_scalar_c12_up", "gather", "nhwc", C=12, H=20, W=18, up=1, seed=7),
        T("g_nhwc_vec_swish", "gather", "nhwc", C=24, act=ACT_SWISH, seed=8),
        T("g_nhwc_scalar_misaligned_swish", "gather", "nhwc", C=24, act=ACT_SWISH, misalign=True, seed=9),
    ]
    # gather: scale and shift in every broadcast shape, in f32 and in the launch dtype, across the paths and both orders
    paths = (("nhwc", 16, False), ("nhwc", 20, False), ("nhwc", 16, True), ("nchw", 16, False))
    for i, shp in enumerate(BCAST_SHAPES):
        for j, adt in enumerate(("f32", "x")):
            lay, C, mis = paths[(i + j) % 4]
            act, first = ((ACT_SWISH, True), (ACT_SWISH, False), (ACT_IDENTITY, False))[(i + 2 * j) % 3]
            cases.append(T("g_%s_%s_aff%s_%s_%s%s" % (lay, "".join(map(str, shp)), adt, "swish" if act else "id", "first" if first else "last",
                                                      "_mis" if mis else ""), "gather", lay, C=C, scale=shp, shift=BCAST_SHAPES[(i + 3) % 7],
                           aff_dt=adt, act=act, act_first=first, misalign=mis, seed=20 + 2 * i + j))
    cases += [
        T("g_nhwc_vec_scale_only", "gather", "nhwc", C=16, scale=(0, 1, 0, 0), seed=40),
        T("g_nhwc_vec_shift_only_swish_first", "gather", "nhwc", C=16, shift=(1, 1, 0, 0), act=ACT_SWISH, act_first=True, seed=41),
        # C not a multiple of 4: the scalar NHWC path in every dtype, f32 included, with aligned pointers
        T("g_nhwc_scalar_c6_affine_swish", "gather", "nhwc", C=6, scale=(1, 1, 0, 0), shift=(0, 1, 1, 1), act=ACT_SWISH, seed=42),
        T("g_nhwc_scalar_c10_up_identity", "gather", "nhwc", C=10, H=20, W=18, up=1, seed=43),
        # scatter: copy and in-place forms, every path, stride 2 with origins -1 and -2, residual in every broadcast shape
        T("s_nchw_copy", "scatter", "nchw", seed=50),
        T("s_nhwc_vec_copy", "scatter", "nhwc", C=32, seed=51),
        T("s_nhwc_scalar_c12_copy", "scatter", "nhwc", C=12, seed=52),
        T("s_nhwc_scalar_misaligned_copy", "scatter", "nhwc", C=16, misalign=True, seed=53),
        T("s_nchw_inplace", "scatter", "nchw", inplace=True, seed=54),
        T("s_nhwc_vec_inplace", "scatter", "nhwc", C=16, inplace=True, seed=55),
        T("s_nhwc_scalar_c12_inplace_residual", "scatter", "nhwc", C=12, inplace=True, residual=(1, 1, 1, 1), seed=56),
        T("s_nhwc_scalar_misaligned_inplace", "scatter", "nhwc", C=16, inplace=True, misalign=True, seed=57),
        T("s_nchw_stride2", "scatter", "nchw", stride=2, seed=58),
        T("s_nhwc_vec_stride2_inplace", "scatter", "nhwc", C=16, stride=2, inplace=True, seed=59),
        T("s_nhwc_scalar_c12_stride2_residual", "scatter", "nhwc", C=12, stride=2, residual=(0, 1, 0, 0), seed=60),
        T("s_nhwc_scalar_c6_copy", "scatter", "nhwc", C=6, seed=61),
        T("s_nhwc_scalar_c10_inplace_residual", "scatter", "nhwc", C=10, inplace=True, residual=(1, 1, 0, 0), seed=62),
    ]
    for i, shp in enumerate(BCAST_SHAPES):
        lay, C, mis = paths[i % 4]
        cases.append(T("s_%s_res%s_%s%s" % (lay, "".join(map(str, shp)), ("f32", "x")[i % 2], "_mis" if mis else ""), "scatter", lay, C=C,
                       residual=shp, aff_dt=("f32", "x")[i % 2], misalign=mis, inplace=bool(i % 3 == 2), seed=70 + i))
    cases += [
        # scatter_gather, with the map of get_scatter_map
        T("sg_nchw_identity", "scatter_gather", "nchw", seed=80),
        T("sg_nhwc_vec_identity", "scatter_gather", "nhwc", C=32, seed=81),
        T("sg_nhwc_scalar_c12_identity", "scatter_gather", "nhwc", C=12, seed=82),
        T("sg_nhwc_scalar_misaligned_identity", "scatter_gather", "nhwc", C=16, misalign=True, seed=83),
        T("sg_nhwc_vec_affine_swish", "scatter_gather", "nhwc", C=16, scale=(1, 1, 0, 0), shift=(0, 1, 0, 0), act=ACT_SWISH, seed=84),
        T("sg_nchw_affine_x_swish_first", "scatter_gather", "nchw", scale=(0, 1, 1, 1), shift=(1, 1, 1, 1), aff_dt="x", act=ACT_SWISH,
          act_first=True, seed=85),
        T("sg_nhwc_scalar_c12_swish", "scatter_gather", "nhwc", C=12, act=ACT_SWISH, shift=(0, 0, 1, 1), seed=86),
        T("sg_nhwc_scalar_c10_affine_swish_first", "scatter_gather", "nhwc", C=10, scale=(0, 1, 0, 0), shift=(1, 1, 0, 0), act=ACT_SWISH,
          act_first=True, seed=87),
        # scatter_with_block_residual
        T("swbr_nchw", "swbr", "nchw", seed=90),
        T("swbr_nhwc_vec", "swbr", "nhwc", C=32, seed=91),
        T("swbr_nhwc_scalar_c12", "swbr", "nhwc", C=12, seed=92),
        T("swbr_nhwc_scalar_misaligned", "swbr", "nhwc", C=16, misalign=True, seed=93),
        T("swbr_nhwc_vec_stride2", "swbr", "nhwc", C=16, stride=2, seed=94),
        T("swbr_nhwc_scalar_c6", "swbr", "nhwc", C=6, seed=95),
    ]
    return cases


TILE_CASES = _tile_cases()
