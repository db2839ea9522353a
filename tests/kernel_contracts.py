"""The C-ABI contracts of the separable SPADE conv, the dense glue kernels and the attention core, restated in float64.

Imported by tests/test_kernel_contracts.py (CPU: each restatement against an independent computation, the case tables against
the kernels' branch predicates, the C-ABI refusals) and tests/test_gpu_kernel_contracts.py (GPU: every case against its
restatement).  Modelled on tests/tile_conv_contract.py, whose bound vocabulary it shares:

  * a frozen `...Spec` describes one launch in numbers; `make_...(spec, dtype, device)` turns it into a case of seeded tensors.
    Every buffer a launch may write is a 16-byte aligned window of a larger flat buffer filled with random bytes (a `Guarded`),
    so a stray write anywhere shows.
  * `..._descriptor` / `..._args` is the C descriptor or argument list of the launch (it keeps the tensors alive).
  * `..._reference(case)` computes in float64 what the launch must leave in every buffer it may write: the expected values,
    the mask of the elements it writes and a per-element error bound, all over the whole flat buffer.
  * `check(...)` applies the bounds to the written elements and demands that every other element of every buffer, and every
    element of every input, is bitwise unchanged.

Bounds (u = unit roundoff of the launch dtype; ACC, PRE_ULPS, ABS, SWISH_LIP as in tile_conv_contract):

  separable   u*|want| + ACC*mag + PRE_ULPS*u*sum_c |pw_w[co,c]|*|a64[c]| + ABS.  The depthwise result a64 is staged once in the
              launch dtype from fp32 arithmetic, so each staged value may sit one 16-bit ulp (2u relative) from round(a64);
              the third term allows that for every input channel of the 1x1.
  conv_in     u*|want| + ACC*mag + ABS; an aux act(acc*scale + shift) of the unrounded accumulator gets SWISH_LIP*|scale| times
              that bound plus its own rounding u*|aux| (tile_conv_contract's aux bound).
  conv_out    u*|want| + ACC*mag + [pre-op] PRE_ULPS*u*max|w[co]|*max|a| + ABS (tile_conv_contract's pre-op bound).
  GroupNorm   see gn_reference: a first-order worst case of the kernel's fp32 partial sums, carried through the variance,
              rstd, scale and shift.
  attention   u*|want| + C_P*u*sum_j s_j|v_j| + sum_j (c_e[j]*s_j + eta*w_r(j)/L)*|v_j - want| + ACC*mag + ABS; derived at
              attn_reference.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from tile_conv_contract import ABS, ACC, PRE_ULPS, SWISH_LIP, TILE_NONE, UNIT_ROUNDOFF

PDL = 1
U32 = 2.0 ** -24
H100_SMS = 132                  # what the library assumes when no device can be queried
ROUNDOFF = {**UNIT_ROUNDOFF, torch.float64: 2.0 ** -53}


def _act(x, act):
    return x * torch.sigmoid(x) if act == 1 else x


def _ptr(t):
    return None if t is None else t.data_ptr()


# ----------------------------------------------------------------------------------------------------------------------
# guarded buffers, expectations and the shared check
# ----------------------------------------------------------------------------------------------------------------------
@dataclass
class Guarded:
    """`view` (contiguous, `shape`) sits at element `off` of the flat buffer `flat`; everything else in `flat` is guard band."""
    flat: torch.Tensor
    view: torch.Tensor
    off: int
    layout: str                 # how to name an element of view: "nhwc", "nchw", "bnc" or "bc"


def guarded(shape, dtype, device, gen: torch.Generator, layout: str, lead_bytes: int = 64, tail_bytes: int = 80) -> Guarded:
    """A window of a flat buffer of random bytes; the window starts 16-byte aligned, `lead_bytes` into the buffer."""
    es = torch.empty((), dtype=dtype).element_size()
    n = int(np.prod(shape))
    lead, tail = lead_bytes // es, tail_bytes // es
    bits = {2: torch.int16, 4: torch.int32, 8: torch.int64}[es]
    info = torch.iinfo(bits)
    flat = torch.randint(info.min, info.max, (lead + n + tail,), dtype=bits, generator=gen, device=device).view(dtype)
    if dtype == torch.float64:          # CPU cases: plain values (float64 NaN bit patterns are the same either way)
        flat = torch.randn(lead + n + tail, generator=gen, device=device, dtype=torch.float64)
    assert flat.data_ptr() % 16 == 0
    return Guarded(flat, flat[lead:lead + n].view(*shape), lead, layout)


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


@dataclass
class Expect:
    name: str
    want: torch.Tensor          # float64, flat: the initial contents where nothing is written
    written: torch.Tensor       # bool, flat
    bound: torch.Tensor         # float64, flat (0 where not written)
    rounding: torch.Tensor      # the part of `bound` that is the element's own rounding, u*|want|
    g: Guarded
    scratch: Optional[torch.Tensor] = None   # bool, flat: may change to anything (a workspace)

    def where(self, i: int) -> str:
        j = i - self.g.off
        if j < 0 or j >= self.g.view.numel():
            return "guard element %d" % i
        c = np.unravel_index(j, tuple(self.g.view.shape))
        if self.g.layout == "nhwc":
            return "(b, c, h, w) = (%d, %d, %d, %d)" % (c[0], c[3], c[1], c[2])
        if self.g.layout == "nchw":
            return "(b, c, h, w) = (%d, %d, %d, %d)" % tuple(c)
        if self.g.layout == "bnc":
            return "(b, token, c) = (%d, %d, %d)" % tuple(c)
        if self.g.layout == "bhnd":
            return "(b, head, token, d) = (%d, %d, %d, %d)" % tuple(c)
        if self.g.layout == "bnhd":
            return "(b, token, head, d) = (%d, %d, %d, %d)" % tuple(c)
        if self.g.layout == "pc":
            return "(pixel, c) = (%d, %d)" % tuple(c)
        return "(b, c) = (%d, %d)" % tuple(c)


def expect_for(name: str, g: Guarded, u: float) -> Tuple[Expect, tuple]:
    """An Expect of a guarded buffer with nothing written yet, and (want, written, bound, rounding) as views of its window."""
    dev = g.flat.device
    e = Expect(name, g.flat.double().clone(), torch.zeros(g.flat.shape, dtype=torch.bool, device=dev),
               torch.zeros(g.flat.shape, dtype=torch.float64, device=dev), torch.zeros(g.flat.shape, dtype=torch.float64, device=dev), g)
    n, s = g.view.numel(), tuple(g.view.shape)
    return e, tuple(t[g.off:g.off + n].view(*s) for t in (e.want, e.written, e.bound, e.rounding))


def check(label: str, expects: List[Expect], got: Dict[str, torch.Tensor], init: Dict[str, torch.Tensor],
          inputs: Dict[str, torch.Tensor] = None, inputs0: Dict[str, torch.Tensor] = None) -> Tuple[float, float]:
    """Every written element within its bound; every other element bitwise equal to the buffer's initial contents; every
    input bitwise unchanged.  `got` / `init` hold the flat buffers by name.

    Returns the worst error / bound ratio, and the worst ratio of what the error exceeds the element's own rounding by to the
    rest of the bound (the headroom of the accumulation and staging terms)."""
    for name, t in (inputs or {}).items():
        if not torch.equal(bits(t), bits(inputs0[name])):
            raise AssertionError("%s: input %s was modified (%d elements)" % (label, name, int((bits(t) != bits(inputs0[name])).sum())))
    worst = excess = 0.0
    for e in expects:
        g, g0 = got[e.name], init[e.name]
        allowed = e.written if e.scratch is None else (e.written | e.scratch)
        stray = (bits(g) != bits(g0)) & ~allowed
        if bool(stray.any()):
            i = int(stray.nonzero()[0])
            raise AssertionError("%s: %s changed outside the written set at %s: %r -> %r (%d stray elements)"
                                 % (label, e.name, e.where(i), float(g0[i]), float(g[i]), int(stray.sum())))
        w = e.written
        if not bool(w.any()):
            continue
        err = (g.double()[w] - e.want[w]).abs()
        # a bound of 0 demands the exact value (0 / 0 passes); a NaN error fails
        ratio = torch.nan_to_num(torch.where(err == 0, torch.zeros_like(err), err / e.bound[w]), nan=float("inf"))
        r = float(ratio.max())
        if r > 1.0:
            k = int(ratio.argmax())
            i = int(w.nonzero()[k])
            raise AssertionError("%s: %s at %s: got %r, want %r, |err| %.3g > bound %.3g; %d elements over"
                                 % (label, e.name, e.where(i), float(g[i]), float(e.want[i]), float(err[k]), float(e.bound[i]),
                                    int((ratio > 1).sum())))
        worst = max(worst, r)
        rest = (e.bound[w] - e.rounding[w]).clamp(min=1e-300)
        excess = max(excess, float(((err - e.rounding[w]).clamp(min=0) / rest).max()))
    return worst, excess


def snapshot(bufs: Dict[str, Guarded]) -> Dict[str, torch.Tensor]:
    return {k: g.flat.clone() for k, g in bufs.items()}


def restore(bufs: Dict[str, Guarded], init: Dict[str, torch.Tensor]) -> None:
    for k, g in bufs.items():
        g.flat.copy_(init[k])


# ----------------------------------------------------------------------------------------------------------------------
# launching a case on the device (the GPU test files)
# ----------------------------------------------------------------------------------------------------------------------
def _launch(case, init, call):
    """Restore every written buffer, run `call` (a C-ABI call returning a status), wait, and return the flat buffers."""
    from sige_b200 import _cabi

    restore(case.buffers(), init)
    rc = call()
    torch.cuda.synchronize()
    assert rc == 0, _cabi.last_error()
    return {k: g.flat.clone() for k, g in case.buffers().items()}


def _same(a, b):
    return all(torch.equal(bits(a[k]), bits(b[k])) for k in a)


def _report(kernel, label, r):
    print("[kernel contract] %-10s %-52s worst |err| / bound %.3f, beyond rounding %.3f" % (kernel, label, r[0], r[1]))


def _run_and_check(kernel, label, case, expects, call, flag_variants=(0,)):
    """Launch once per flags value and once more with the first: each within the contract, all bitwise equal."""
    init = snapshot(case.buffers())
    inputs0 = {k: t.clone() for k, t in case.inputs().items()}
    first = None
    for flags in flag_variants:
        lab = label + (" pdl" if flags & PDL else "")
        got = _launch(case, init, lambda: call(flags))
        _report(kernel, lab, check(lab, expects, got, init, case.inputs(), inputs0))
        if first is None:
            first = got
        else:
            assert _same(got, first), "%s: programmatic dependent launch changed the result" % lab
    assert _same(_launch(case, init, lambda: call(flag_variants[0])), first), "%s: a second launch differs" % label
    return first


def graph_equals_stream(case, call):
    """`call` (a C-ABI call returning a status) captured in a CUDA graph and replayed leaves bitwise what a stream launch does."""
    init = snapshot(case.buffers())
    want = _launch(case, init, call)
    g = torch.cuda.CUDAGraph()
    restore(case.buffers(), init)
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        rc = call()
    assert rc == 0
    restore(case.buffers(), init)
    g.replay()
    torch.cuda.synchronize()
    got = {k: gb.flat.clone() for k, gb in case.buffers().items()}
    assert _same(got, want), "a graph replay differs from the stream launch"


# ----------------------------------------------------------------------------------------------------------------------
# sige_separable_conv
# ----------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class SepSpec:
    """One sige_separable_conv launch.  The source is the channel window [pre, pre + Cin) of a (pre + Cin + post)-channel pixel,
    of an NHWC buffer [B, H, W, .] read through the tile list or of a stack [B*N, 6, 6, .].  The tile list holds `real` origins
    of the destination's 4x4 output grid (always the four corners) with a run of `pad_run` SIGE_TILE_NONE entries after the
    first `lead` of them and `tail` more at the end.  Each branch writes ("buf" | "stack", extra channels, c0)."""
    name: str
    B: int
    Cin: int
    Cout: int
    H: int = 24
    W: int = 28
    real: int = 12
    lead: int = 5
    pad_run: int = 0
    tail: int = 0
    pre: int = 0
    post: int = 0
    src_stack: bool = False
    no_list: bool = False           # stack -> stack launch without a tile list (every row is a tile)
    offH: int = 1
    offW: int = 1
    dH: int = 0                     # 0: the source's extent
    dW: int = 0
    dsts: Tuple[Tuple[str, int, int], ...] = (("buf", 0, 0), ("buf", 0, 0))
    dw_bias: bool = True
    pw_bias: bool = True
    per_image: bool = False         # B lists of N rows (SIGE_CONV_PER_IMAGE_OPERANDS): row b*N + i is tile i of image b
    seed: int = 0

    @property
    def dh(self):
        return self.dH or self.H

    @property
    def dw(self):
        return self.dW or self.W

    @property
    def N(self):
        return self.real + self.pad_run + self.tail

    @property
    def src_C(self):
        return self.pre + self.Cin + self.post


# (Cin, Cout, source pixel channels, window offset) of every launch the full-size sub-mobile GauGAN lowering emits: all read a
# stack, through the torch.split window of mlp_shared's output (tests/test_separable_conv.py::_lower_on_sim("full"))
SUB_MOBILE_LAYERS = [(48, 256, 144, 96), (48, 48, 144, 48), (48, 96, 144, 96), (64, 256, 192, 64), (64, 32, 192, 64), (64, 48, 192, 128),
                     (64, 512, 192, 128), (96, 512, 192, 0), (96, 768, 192, 96)]

SEP_CASES = (
    [SepSpec("sm%d_%d_b%d" % (ci, co, b), B=b, Cin=ci, Cout=co, src_stack=True, pre=c0, post=sc - c0 - ci, H=22, W=30, real=13, lead=6,
             pad_run=16, tail=3, seed=ci * 7 + co + b)
     for (ci, co, sc, c0) in SUB_MOBILE_LAYERS for b in (1, 3)]
    + [
        # buffer source, tiles on all four borders (negative origins at the top-left, ragged outputs at the bottom-right), the
        # source the last channel window of a wider pixel, B = 3, a whole CTA of padding
        SepSpec("borders_lastwin_b3", B=3, Cin=48, Cout=96, H=22, W=30, real=20, lead=8, pad_run=16, tail=5, pre=96, seed=101),
        SepSpec("cin256_cout1024", B=1, Cin=256, Cout=1024, H=20, W=20, real=12, lead=4, pad_run=8, tail=1, seed=102),
        SepSpec("cin16_cout8", B=2, Cin=16, Cout=8, H=18, W=26, real=15, lead=3, pad_run=9, tail=2, pre=16, post=16, seed=103),
        SepSpec("cin16_cout40", B=1, Cin=16, Cout=40, H=18, W=26, real=15, lead=8, pad_run=16, seed=104),
        SepSpec("cout72_partial_block", B=2, Cin=32, Cout=72, H=14, W=17, real=10, lead=2, pad_run=3, seed=105),
        SepSpec("stack_src_b2", B=2, Cin=64, Cout=128, src_stack=True, pre=64, H=20, W=24, real=14, lead=7, pad_run=10, tail=2, seed=106),
        # branch 0 writes a stack, branch 1 a channel window of a buffer; the padded list must write nothing to either
        SepSpec("mixed_stack_buf", B=2, Cin=32, Cout=48, H=17, W=21, real=11, lead=3, pad_run=16, tail=2,
                dsts=(("stack", 16, 8), ("buf", 24, 16)), seed=107),
        SepSpec("mixed_buf_stack_stacksrc", B=1, Cin=48, Cout=64, src_stack=True, post=48, real=9, lead=4, pad_run=8,
                dsts=(("buf", 64, 64), ("stack", 0, 0)), seed=108),
        SepSpec("offH2_offW0_dst_extent", B=2, Cin=32, Cout=64, H=19, W=23, dH=21, dW=18, offH=2, offW=0, real=16, lead=8, pad_run=8,
                seed=109),
        SepSpec("no_biases", B=1, Cin=64, Cout=96, H=16, W=16, real=10, dw_bias=False, pw_bias=False, dsts=(("buf", 0, 0),), seed=110),
        SepSpec("stack_to_stack_no_list", B=3, Cin=48, Cout=96, src_stack=True, no_list=True, real=7, lead=7,
                dsts=(("stack", 0, 0), ("stack", 8, 8)), seed=111),
    ]
)


@dataclass
class SepCase:
    spec: SepSpec
    dtype: torch.dtype
    src: torch.Tensor               # NHWC [B, H, W, src_C] or stack [B*N, 6, 6, src_C]
    idx: Optional[torch.Tensor]     # int32 [N, 2]
    dw_w: List[torch.Tensor]        # fp32 [Cin, 9] per branch
    dw_b: List[Optional[torch.Tensor]]
    pw_w: List[torch.Tensor]        # [Cout, Cin], launch dtype
    pw_b: List[Optional[torch.Tensor]]
    dst: List[Guarded]
    tile_img: Optional[torch.Tensor] = None     # per-image lists: the image of each row (default row // N)

    def buffers(self) -> Dict[str, Guarded]:
        return {"dst%d" % i: g for i, g in enumerate(self.dst)}

    def inputs(self) -> Dict[str, torch.Tensor]:
        out = {"src": self.src}
        if self.idx is not None:
            out["idx"] = self.idx
        for i in range(len(self.dst)):
            out.update({"dw_w%d" % i: self.dw_w[i], "pw_w%d" % i: self.pw_w[i]})
            for k, t in (("dw_b%d" % i, self.dw_b[i]), ("pw_b%d" % i, self.pw_b[i])):
                if t is not None:
                    out[k] = t
        return out


def sep_tile_list(spec: SepSpec, rng: np.random.Generator):
    """`real` distinct origins whose 4x4 outputs tile the destination (origin = 4i - off), always with the four corners."""
    hs = [4 * i - spec.offH for i in range(-(-spec.dh // 4))]
    ws = [4 * i - spec.offW for i in range(-(-spec.dw // 4))]
    grid = [(h, w) for h in hs for w in ws]
    corners = [(hs[0], ws[0]), (hs[0], ws[-1]), (hs[-1], ws[0]), (hs[-1], ws[-1])]
    rest = [g for g in grid if g not in corners]
    tiles = corners + [rest[i] for i in rng.choice(len(rest), spec.real - 4, replace=False)]
    rng.shuffle(tiles)
    none = [(TILE_NONE, TILE_NONE)]
    return tiles[:spec.lead] + none * spec.pad_run + tiles[spec.lead:] + none * spec.tail


def make_sep(spec: SepSpec, dtype: torch.dtype, device) -> SepCase:
    rng = np.random.default_rng(spec.seed)
    gen = torch.Generator(device=device)
    gen.manual_seed(spec.seed)
    B, N = spec.B, spec.N

    def randn(*shape, scale=1.0, dt=dtype):
        return (torch.randn(*shape, generator=gen, device=device, dtype=torch.float64) * scale).to(dt)

    rows = sep_tile_list(spec, rng)
    idx = None if spec.no_list else torch.tensor(rows, dtype=torch.int32, device=device)
    src = randn(B * N, 6, 6, spec.src_C) if spec.src_stack else randn(B, spec.H, spec.W, spec.src_C)
    dw_w, dw_b, pw_w, pw_b, dst = [], [], [], [], []
    for kind, extra, c0 in spec.dsts:
        dw_w.append(randn(spec.Cin, 9, scale=0.35, dt=torch.float32))
        dw_b.append(randn(spec.Cin, scale=0.2, dt=torch.float32) if spec.dw_bias else None)
        pw_w.append(randn(spec.Cout, spec.Cin, scale=spec.Cin ** -0.5))
        pw_b.append(randn(spec.Cout, scale=0.3, dt=torch.float32) if spec.pw_bias else None)
        shape = (B * N, 4, 4, spec.Cout + extra) if kind == "stack" else (B, spec.dh, spec.dw, spec.Cout + extra)
        dst.append(guarded(shape, dtype, device, gen, "nhwc"))
    return SepCase(spec, dtype, src, idx, dw_w, dw_b, pw_w, pw_b, dst)


def sep_descriptor(case: SepCase, flags: int = 0):
    """The sige_separable_conv_t of this case; d._keep holds the tensors."""
    from sige_b200 import _cabi

    s = case.spec
    d = _cabi.SeparableConv()
    d.dtype = {torch.float16: _cabi.F16, torch.bfloat16: _cabi.BF16, torch.float32: _cabi.F32}[case.dtype]
    d.src, d.src_is_stack, d.src_C, d.src_c0 = case.src.data_ptr(), int(s.src_stack), s.src_C, s.pre
    d.B, d.H, d.W = s.B, (6 if s.src_stack else s.H), (6 if s.src_stack else s.W)
    d.idx, d.N = _ptr(case.idx), s.N
    d.Cin, d.Cout, d.offH, d.offW = s.Cin, s.Cout, s.offH, s.offW
    d.nbranch = len(s.dsts)
    for i, (kind, extra, c0) in enumerate(s.dsts):
        br, g = d.branch[i], case.dst[i]
        br.dw_weight, br.dw_bias = case.dw_w[i].data_ptr(), _ptr(case.dw_b[i])
        br.pw_weight, br.pw_bias = case.pw_w[i].data_ptr(), _ptr(case.pw_b[i])
        br.dst, br.dst_is_stack = g.view.data_ptr(), int(kind == "stack")
        br.dH, br.dW = (4, 4) if kind == "stack" else (s.dh, s.dw)
        br.dst_C, br.dst_c0 = s.Cout + extra, c0
    d.flags = flags
    d._keep = case
    return d


def sep_images(case: SepCase) -> torch.Tensor:
    """The image of each of the launch's B*N tile rows: row t // N of B shared lists, or `tile_img` of per-image lists."""
    s = case.spec
    t = torch.arange(s.B * s.N, device=case.src.device)
    if s.per_image and case.tile_img is not None:
        assert case.tile_img.numel() == s.B * s.N, s.name
        return case.tile_img.long().to(t.device)
    return t // s.N


def sep_halo(case: SepCase):
    """float64 halo tiles [B*N, 6, 6, Cin] the launch reads (zero outside the source image and on padding tiles of a buffer
    source), the tile origins [B*N, 2] (None without a list) and the padding mask [B*N].  A shared list is read by every
    image; per-image lists hold B*N rows, row t a tile of image sep_images(case)[t]."""
    s = case.spec
    dev = case.src.device
    NT = s.B * s.N
    t = torch.arange(NT, device=dev)
    img, row = sep_images(case), (t if s.per_image else t % s.N)
    if s.per_image:
        assert not s.src_stack and case.idx is not None and case.idx.shape[0] == NT, s.name
    org = None if case.idx is None else case.idx.long()[row]
    none = torch.zeros(NT, dtype=torch.bool, device=dev) if org is None else org[:, 0] == TILE_NONE
    win = slice(s.pre, s.pre + s.Cin)
    if s.src_stack:
        return case.src[..., win].double(), org, none
    d = torch.arange(6, device=dev)
    hh, ww = org[:, :1] + d, org[:, 1:] + d
    valid = ((hh >= 0) & (hh < s.H))[:, :, None] & ((ww >= 0) & (ww < s.W))[:, None, :] & ~none[:, None, None]
    x = case.src[img[:, None, None], hh.clamp(0, s.H - 1)[:, :, None], ww.clamp(0, s.W - 1)[:, None, :]][..., win].double()
    return torch.where(valid[..., None], x, torch.zeros((), dtype=x.dtype, device=dev)), org, none


def sep_reference(case: SepCase) -> List[Expect]:
    s = case.spec
    dev = case.src.device
    u = ROUNDOFF[case.dtype]
    x, org, none = sep_halo(case)
    NT = s.B * s.N
    img = sep_images(case)
    d4 = torch.arange(4, device=dev)
    out = []
    for i, (kind, extra, c0) in enumerate(s.dsts):
        # depthwise in float64, staged once in the launch dtype
        w9 = case.dw_w[i].double().view(s.Cin, 1, 3, 3)
        a64 = F.conv2d(x.permute(0, 3, 1, 2), w9, None if case.dw_b[i] is None else case.dw_b[i].double(), groups=s.Cin)
        a64 = a64.permute(0, 2, 3, 1)                                                   # [NT, 4, 4, Cin]
        a = a64.to(case.dtype).double()
        pw = case.pw_w[i].double()
        v = a @ pw.t()
        mag = a.abs() @ pw.abs().t()
        if case.pw_b[i] is not None:
            v, mag = v + case.pw_b[i].double(), mag + case.pw_b[i].double().abs()
        bound = u * v.abs() + ACC * mag + PRE_ULPS * u * (a64.abs() @ pw.abs().t()) + ABS
        e, (want, written, bd, rnd) = expect_for("dst%d" % i, case.dst[i], u)
        sl = slice(c0, c0 + s.Cout)
        keep = ~none                                                                    # padding tiles write nothing
        if kind == "stack":
            tt = torch.arange(NT, device=dev)[keep]
            want[tt, :, :, sl], written[tt, :, :, sl] = v[keep], True
            bd[tt, :, :, sl], rnd[tt, :, :, sl] = bound[keep], (u * v.abs())[keep]
        else:
            oh, ow = org[:, :1] + s.offH + d4, org[:, 1:] + s.offW + d4                 # [NT, 4]
            ok = ((oh >= 0) & (oh < s.dh))[:, :, None] & ((ow >= 0) & (ow < s.dw))[:, None, :] & keep[:, None, None]
            OB = img[:, None, None].expand(NT, 4, 4)[ok]
            OH, OW = oh[:, :, None].expand(NT, 4, 4)[ok], ow[:, None, :].expand(NT, 4, 4)[ok]
            lin = (OB * s.dh + OH) * s.dw + OW
            assert lin.unique().numel() == lin.numel(), "case %s: two tiles write the same output pixel" % s.name
            want[OB, OH, OW, sl], written[OB, OH, OW, sl] = v[ok], True
            bd[OB, OH, OW, sl], rnd[OB, OH, OW, sl] = bound[ok], (u * v.abs())[ok]
        out.append(e)
    return out


# ----------------------------------------------------------------------------------------------------------------------
# sige_conv_in_nhwc / sige_conv_in_nhwc_tiles
# ----------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class ConvInSpec:
    """One stem launch: 3x3 pad-1 conv of a Cin <= 4 image.  aux: (affine, act, negative) per aux destination (negative: the
    scales are drawn around -1).  tiles: None (dense) or (per_image, counts, R, pad) — `counts` real R x R tiles per image
    (one entry: one shared list), lists padded to max(counts) + pad with SIGE_TILE_NONE entries."""
    name: str
    B: int
    H: int
    W: int
    Cin: int
    Cout: int
    aux: Tuple[Tuple[bool, int, bool], ...] = ()
    tiles: Optional[Tuple[bool, Tuple[int, ...], int, int]] = None
    bias: bool = True
    seed: int = 0


CONV_IN_CASES = [
    ConvInSpec("dense_cin3_cout128_b2", B=2, H=36, W=44, Cin=3, Cout=128, seed=1),
    ConvInSpec("dense_cin1_cout8", B=2, H=9, W=12, Cin=1, Cout=8, aux=((True, 1, False),), seed=2),
    ConvInSpec("dense_cin2_cout256_two_aux", B=2, H=20, W=16, Cin=2, Cout=256, aux=((True, 1, True), (True, 0, False)), seed=3),
    ConvInSpec("dense_cin4_cout128_aux_plain", B=1, H=31, W=40, Cin=4, Cout=128, aux=((False, 0, False),), bias=False, seed=4),
    ConvInSpec("dense_cin3_cout256_aux_swish_neg", B=2, H=16, W=24, Cin=3, Cout=256, aux=((True, 1, True),), seed=5),
    ConvInSpec("tiles_shared", B=2, H=37, W=45, Cin=3, Cout=128, tiles=(False, (23,), 6, 5), seed=6),
    ConvInSpec("tiles_shared_one_aux", B=1, H=30, W=26, Cin=4, Cout=8, aux=((True, 1, True),), tiles=(False, (17,), 6, 0), seed=7),
    ConvInSpec("tiles_per_image_two_aux", B=3, H=38, W=41, Cin=3, Cout=128, aux=((True, 1, False), (True, 1, True)),
               tiles=(True, (31, 12, 4), 6, 9), seed=8),
    ConvInSpec("tiles_per_image_cin1_cout256", B=2, H=22, W=19, Cin=1, Cout=256, aux=((False, 1, False),), tiles=(True, (9, 14), 4, 3), seed=9),
    # weights above 48 KB take the dynamic shared-memory opt-in (dense_glue.cu conv_in_smem_ok): Cin 4 from Cout 328, Cin 3 from
    # Cout 432; Cin 4, Cout 1544 is the largest stem that fits (231,600 B)
    ConvInSpec("dense_cin4_cout320_below_optin", B=1, H=14, W=20, Cin=4, Cout=320, seed=10),
    ConvInSpec("dense_cin4_cout328_optin", B=2, H=13, W=16, Cin=4, Cout=328, aux=((True, 1, False),), seed=11),
    ConvInSpec("tiles_shared_cin4_cout328_optin", B=1, H=20, W=22, Cin=4, Cout=328, tiles=(False, (11,), 6, 5), seed=12),
    ConvInSpec("dense_cin3_cout432_optin_aux", B=1, H=12, W=16, Cin=3, Cout=432, aux=((True, 1, True),), seed=13),
    ConvInSpec("tiles_shared_cin3_cout512_aux", B=2, H=18, W=21, Cin=3, Cout=512, aux=((True, 0, False),), tiles=(False, (9,), 6, 3), seed=14),
    ConvInSpec("tiles_per_image_cin4_cout512_sd_stem", B=2, H=24, W=20, Cin=4, Cout=512, aux=((True, 1, False),), tiles=(True, (7, 12), 6, 4),
               seed=15),
    ConvInSpec("dense_cin4_cout1544_largest", B=1, H=9, W=12, Cin=4, Cout=1544, seed=16),
    ConvInSpec("tiles_shared_cin4_cout1544_largest", B=1, H=16, W=16, Cin=4, Cout=1544, aux=((True, 1, False),), tiles=(False, (5,), 6, 2), seed=17),
]


@dataclass
class ConvInCase:
    spec: ConvInSpec
    dtype: torch.dtype
    x: torch.Tensor                 # NHWC [B, H, W, Cin]
    w: torch.Tensor                 # OIHW, launch dtype
    bias: Optional[torch.Tensor]    # launch dtype
    idx: Optional[torch.Tensor]     # int32 [n or B*n, 2]
    n_tiles: int
    out: Guarded
    aux: List[Guarded]
    scale: List[Optional[torch.Tensor]]
    shift: List[Optional[torch.Tensor]]

    def buffers(self):
        b = {"out": self.out}
        b.update({"aux%d" % i: g for i, g in enumerate(self.aux)})
        return b

    def inputs(self):
        out = {"x": self.x, "w": self.w}
        for k, t in (("bias", self.bias), ("idx", self.idx)):
            if t is not None:
                out[k] = t
        for i in range(len(self.aux)):
            if self.scale[i] is not None:
                out["scale%d" % i], out["shift%d" % i] = self.scale[i], self.shift[i]
        return out


def make_conv_in(spec: ConvInSpec, dtype: torch.dtype, device) -> ConvInCase:
    rng = np.random.default_rng(spec.seed)
    gen = torch.Generator(device=device)
    gen.manual_seed(spec.seed)

    def randn(*shape, scale=1.0, dt=dtype):
        return (torch.randn(*shape, generator=gen, device=device, dtype=torch.float64) * scale).to(dt)

    B = spec.B
    x = randn(B, spec.H, spec.W, spec.Cin)
    w = randn(spec.Cout, spec.Cin, 3, 3, scale=(9 * spec.Cin) ** -0.5)
    bias = randn(spec.Cout, scale=0.3) if spec.bias else None
    idx, n_tiles = None, 0
    if spec.tiles is not None:
        per_image, counts, R, pad = spec.tiles
        n_tiles = max(counts) + pad
        rows = []
        for n in counts:
            # origins anywhere from R - 1 above / left of the image to its last row / column: many stick out
            hs = rng.integers(-(R - 1), spec.H, size=n)
            ws = rng.integers(-(R - 1), spec.W, size=n)
            tiles = [(int(h), int(v)) for h, v in zip(hs, ws)] + [(TILE_NONE, TILE_NONE)] * (n_tiles - n)
            perm = rng.permutation(n_tiles)
            rows += [tiles[j] for j in perm]
        assert per_image or len(counts) == 1
        assert not per_image or len(counts) == B
        idx = torch.tensor(rows, dtype=torch.int32, device=device)
    out = guarded((B, spec.H, spec.W, spec.Cout), dtype, device, gen, "nhwc")
    aux, scale, shift = [], [], []
    for affine, act, neg in spec.aux:
        aux.append(guarded((B, spec.H, spec.W, spec.Cout), dtype, device, gen, "nhwc"))
        if affine:
            sign = torch.where(torch.rand(spec.Cout, generator=gen, device=device) < 0.5, -1.0, 1.0) if neg else 1.0
            scale.append(((1 + 0.3 * torch.randn(spec.Cout, generator=gen, device=device)) * sign).float())
            shift.append((0.4 * torch.randn(spec.Cout, generator=gen, device=device)).float())
        else:
            scale.append(None)
            shift.append(None)
    return ConvInCase(spec, dtype, x, w, bias, idx, n_tiles, out, aux, scale, shift)


def conv_in_call(case: ConvInCase, lib):
    """Calls sige_conv_in_nhwc[_tiles] for the case on `stream` 0 of the current device; returns the status."""
    from sige_b200 import _cabi

    s = case.spec
    arr = (_cabi.ConvAux * 2)()
    for i, g in enumerate(case.aux):
        a = arr[i]
        a.ptr, a.C, a.c0 = g.view.data_ptr(), s.Cout, 0
        a.scale, a.shift, a.act = _ptr(case.scale[i]), _ptr(case.shift[i]), s.aux[i][1]
    dt = {torch.float16: _cabi.F16, torch.bfloat16: _cabi.BF16}[case.dtype]
    stream = torch.cuda.current_stream().cuda_stream
    common = (case.x.data_ptr(), case.w.data_ptr(), _ptr(case.bias), case.out.view.data_ptr(), dt, s.B, s.H, s.W, s.Cin, s.Cout)
    if s.tiles is None:
        return lib.sige_conv_in_nhwc(*common, len(case.aux), arr, stream)
    per_image, _, R, _ = s.tiles
    return lib.sige_conv_in_nhwc_tiles(*common, case.idx.data_ptr(), case.n_tiles, R, R, int(per_image), len(case.aux), arr, stream)


def conv_in_written(case: ConvInCase) -> torch.Tensor:
    """bool [B, H, W]: the pixels the launch writes (all of them, or the in-image pixels of each image's tiles)."""
    s = case.spec
    dev = case.x.device
    if s.tiles is None:
        return torch.ones(s.B, s.H, s.W, dtype=torch.bool, device=dev)
    per_image, _, R, _ = s.tiles
    n = case.n_tiles
    t = torch.arange(s.B * n, device=dev)
    img, row = t // n, (t if per_image else t % n)
    org = case.idx.long()[row]
    d = torch.arange(R, device=dev)
    hh, ww = org[:, :1] + d, org[:, 1:] + d
    ok = ((hh >= 0) & (hh < s.H))[:, :, None] & ((ww >= 0) & (ww < s.W))[:, None, :]    # TILE_NONE rows are never in-image
    m = torch.zeros(s.B, s.H, s.W, dtype=torch.bool, device=dev)
    IB = img[:, None, None].expand(-1, R, R)[ok]
    m[IB, hh[:, :, None].expand(-1, R, R)[ok], ww[:, None, :].expand(-1, R, R)[ok]] = True
    return m


def conv_in_reference(case: ConvInCase) -> List[Expect]:
    s = case.spec
    u = ROUNDOFF[case.dtype]
    x = case.x.double().permute(0, 3, 1, 2)
    w = case.w.double()
    v = F.conv2d(x, w, padding=1)
    mag = F.conv2d(x.abs(), w.abs(), padding=1)
    if case.bias is not None:
        v, mag = v + case.bias.double().view(1, -1, 1, 1), mag + case.bias.double().abs().view(1, -1, 1, 1)
    v, mag = v.permute(0, 2, 3, 1), mag.permute(0, 2, 3, 1)                           # NHWC
    bound = u * v.abs() + ACC * mag + ABS
    m = conv_in_written(case)

    def fill(name, g, val, bd):
        e, (want, written, b, rnd) = expect_for(name, g, u)
        want[m], written[m], b[m], rnd[m] = val[m], True, bd[m], (u * val.abs())[m]
        return e

    out = [fill("out", case.out, v, bound)]
    for i, g in enumerate(case.aux):
        sc = torch.ones(s.Cout, dtype=torch.float64, device=v.device) if case.scale[i] is None else case.scale[i].double()
        sh = torch.zeros(s.Cout, dtype=torch.float64, device=v.device) if case.shift[i] is None else case.shift[i].double()
        av = _act(v * sc + sh, s.aux[i][1])
        out.append(fill("aux%d" % i, g, av, SWISH_LIP * sc.abs() * bound + u * av.abs()))
    return out


# ----------------------------------------------------------------------------------------------------------------------
# sige_group_norm_fold
# ----------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class GNSpec:
    """x = mean * (1 + 0.25 b) + std * N(0, 1) per image b (so the images' statistics differ), plus a small per-channel
    offset; gamma / beta in the launch dtype or NULL."""
    name: str
    B: int
    H: int
    W: int
    C: int
    G: int
    mean: float = 0.3
    std: float = 1.5
    affine: bool = True
    eps: float = 1e-6
    seed: int = 0


GN_CASES = [
    GNSpec("c128_g32", B=2, H=40, W=52, C=128, G=32, seed=1),
    GNSpec("c64_g1", B=2, H=24, W=40, C=64, G=1, seed=2),
    GNSpec("c96_g3", B=1, H=33, W=35, C=96, G=3, seed=3),
    GNSpec("c24_g8", B=3, H=20, W=21, C=24, G=8, seed=4),
    GNSpec("c1024_g32", B=1, H=24, W=24, C=1024, G=32, seed=5),
    GNSpec("c160_g32_hw_lt_64", B=2, H=7, W=9, C=160, G=32, seed=6),
    GNSpec("c128_g32_no_affine_hw_lt_64", B=1, H=5, W=5, C=128, G=32, affine=False, seed=7),
    GNSpec("c128_g32_512", B=1, H=512, W=512, C=128, G=32, seed=8),
    GNSpec("offset_c128_256", B=1, H=256, W=256, C=128, G=32, mean=8.0, std=0.25, seed=9),
    GNSpec("offset_c128_512", B=1, H=512, W=512, C=128, G=32, mean=8.0, std=0.25, seed=10),
]


def gn_nblk(HW: int, sms: int) -> int:
    """Partial-sum blocks per image: sige_group_norm_fold's min(2 * SMs, HW / 64), at least 1."""
    return min(2 * sms, max(1, HW // 64))


def gn_cpb(C: int, G: int) -> int:
    """Channels per finalize CTA: 32 when that is a whole number of groups, else all C."""
    return 32 if (C % 32 == 0 and 32 % (C // G) == 0) else C


def gn_slots(C: int) -> int:
    """Pixel slots of a partial CTA (256 threads = slots x C/8 channel octets); 256 % (C/8) threads idle."""
    return 256 // (C // 8)


def gn_chain(HW: int, C: int, sms: int) -> int:
    """The longest chain of fp32 additions behind one partial (sum, sumsq): a thread's pixels, then the slots."""
    nblk = gn_nblk(HW, sms)
    per = -(-HW // nblk)
    return -(-per // gn_slots(C)) + gn_slots(C)


@dataclass
class GNCase:
    spec: GNSpec
    dtype: torch.dtype
    x: torch.Tensor                 # NHWC [B, H, W, C]
    gamma: Optional[torch.Tensor]
    beta: Optional[torch.Tensor]
    scale: Guarded                  # fp32 [B, C]
    shift: Guarded
    ws: Guarded                     # fp32 workspace (exactly the floats the call needs)
    sms: int

    def buffers(self):
        return {"scale": self.scale, "shift": self.shift, "workspace": self.ws}

    def inputs(self):
        out = {"x": self.x}
        if self.gamma is not None:
            out["gamma"], out["beta"] = self.gamma, self.beta
        return out


def make_gn(spec: GNSpec, dtype: torch.dtype, device, sms: Optional[int] = None) -> GNCase:
    gen = torch.Generator(device=device)
    gen.manual_seed(spec.seed)
    if sms is None:
        sms = torch.cuda.get_device_properties(torch.device(device)).multi_processor_count if torch.device(device).type == "cuda" else H100_SMS
    B, C = spec.B, spec.C
    per_img = spec.mean * (1 + 0.25 * torch.arange(B, device=device, dtype=torch.float64)).view(B, 1, 1, 1)
    per_ch = 0.05 * spec.std * torch.randn(C, generator=gen, device=device, dtype=torch.float64)
    x = (per_img + per_ch + spec.std * torch.randn(B, spec.H, spec.W, C, generator=gen, device=device, dtype=torch.float64)).to(dtype)
    gamma = (1 + 0.2 * torch.randn(C, generator=gen, device=device)).to(dtype) if spec.affine else None
    beta = (0.2 * torch.randn(C, generator=gen, device=device)).to(dtype) if spec.affine else None
    need = B * gn_nblk(spec.H * spec.W, sms) * C * 2
    return GNCase(spec, dtype, x, gamma, beta, guarded((B, C), torch.float32, device, gen, "bc"),
                  guarded((B, C), torch.float32, device, gen, "bc"), guarded((need,), torch.float32, device, gen, "bc"), sms)


def gn_call(case: GNCase, lib, workspace_floats: Optional[int] = None):
    from sige_b200 import _cabi

    s = case.spec
    dt = {torch.float16: _cabi.F16, torch.bfloat16: _cabi.BF16}[case.dtype]
    n = case.ws.view.numel() if workspace_floats is None else workspace_floats
    return lib.sige_group_norm_fold(case.x.data_ptr(), dt, s.B, s.H, s.W, s.C, s.G, float(s.eps), _ptr(case.gamma), _ptr(case.beta),
                                    case.scale.view.data_ptr(), case.shift.view.data_ptr(), case.ws.view.data_ptr(), n,
                                    torch.cuda.current_stream().cuda_stream)


def gn_stats(case: GNCase):
    """float64 two-pass statistics per (b, channel) of the channel's group: mean, var, E|x|, E[x^2]."""
    s = case.spec
    x = case.x.double().view(s.B, s.H * s.W, s.G, s.C // s.G)
    mean = x.mean(dim=(1, 3))
    var = ((x - mean[:, None, :, None]) ** 2).mean(dim=(1, 3))
    eabs, esq = x.abs().mean(dim=(1, 3)), (x * x).mean(dim=(1, 3))
    rep = lambda t: t.repeat_interleave(s.C // s.G, dim=1)                             # noqa: E731
    return rep(mean), rep(var), rep(eabs), rep(esq)


def gn_reference(case: GNCase):
    """Expectations for scale and shift, and their bounds (for the folded check).

    The kernel sums x and x*x (fmaf: one rounding) per channel in fp32 along chains of at most `gn_chain` additions (a
    thread's pixels, then the slots of its CTA), then in float64.  Every term of sumsq is >= 0, so sumsq carries a relative
    error <= gamma = gn_chain * 2^-24 (first order), and sum an absolute error <= gamma * sum|x|.  With n values per group:
      |d mean| <= dm = gamma * E|x|,      |d var| <= dv = gamma * E[x^2] + 2 |mean| dm + dm^2 (+ float64 rounding)
    since the kernel's var = E[x^2] - mean^2 equals the two-pass variance in exact arithmetic.  rstd = 1/sqrt(var + eps) then
    lies in [1/sqrt(var + dv + eps), 1/sqrt(max(var - dv, 0) + eps)], widened by its rounding to fp32; scale = gamma_c * rstd
    and shift = beta_c - mean * rstd * gamma_c add one and four fp32 roundings."""
    s = case.spec
    mean, var, eabs, esq = gn_stats(case)
    g = gn_chain(s.H * s.W, s.C, case.sms) * U32
    dm = g * eabs
    dv = g * esq + 2 * mean.abs() * dm + dm * dm + 4 * 2.0 ** -53 * (esq + mean * mean)
    eps = float(np.float32(s.eps))
    rstd = 1 / torch.sqrt(var + eps)
    hi = 1 / torch.sqrt((var - dv).clamp(min=0) + eps) * (1 + U32)
    lo = 1 / torch.sqrt(var + dv + eps) * (1 - U32)
    drs = torch.maximum(hi - rstd, rstd - lo)
    ga = torch.ones_like(mean) if case.gamma is None else case.gamma.double().expand_as(mean)
    be = torch.zeros_like(mean) if case.beta is None else case.beta.double().expand_as(mean)
    want_scale, want_shift = ga * rstd, be - mean * rstd * ga
    b_scale = ga.abs() * drs + U32 * ga.abs() * hi + 1e-30
    b_shift = ga.abs() * (mean.abs() * drs + hi * dm) + 4 * U32 * (be.abs() + (mean.abs() + dm) * hi * ga.abs()) + 1e-30
    out = []
    for name, g_, want, bd in (("scale", case.scale, want_scale, b_scale), ("shift", case.shift, want_shift, b_shift)):
        e, (w, wr, b, rnd) = expect_for(name, g_, U32)
        w[:], wr[:], b[:], rnd[:] = want, True, bd, U32 * want.abs()
        out.append(e)
    e, _ = expect_for("workspace", case.ws, U32)
    e.scratch = torch.zeros_like(e.written)
    e.scratch[case.ws.off:case.ws.off + case.ws.view.numel()] = True                  # partial sums: any value
    out.append(e)
    return out, (b_scale, b_shift)


def gn_folded_check(label: str, case: GNCase, bounds) -> float:
    """x*scale + shift (with the kernel's scale / shift) against float64 F.group_norm, element by element, within
    |x| * bound(scale) + bound(shift).  Returns the worst error / bound ratio."""
    s = case.spec
    b_scale, b_shift = bounds
    sc, sh = case.scale.view.double(), case.shift.view.double()
    x = case.x.double()                                                                  # NHWC
    gn = F.group_norm(x.permute(0, 3, 1, 2), s.G, None if case.gamma is None else case.gamma.double(),
                      None if case.beta is None else case.beta.double(), float(np.float32(s.eps))).permute(0, 2, 3, 1)
    y = x * sc[:, None, None, :] + sh[:, None, None, :]
    bound = x.abs() * b_scale[:, None, None, :] + b_shift[:, None, None, :]
    ratio = torch.nan_to_num((y - gn).abs() / bound, nan=float("inf"))
    r = float(ratio.max())
    if r > 1:
        b, h, w, c = (int(z) for z in (ratio == ratio.max()).nonzero()[0])
        raise AssertionError("%s: x*scale + shift at (b, c, h, w) = (%d, %d, %d, %d): got %r, group_norm %r, bound %.3g"
                             % (label, b, c, h, w, float(y[b, h, w, c]), float(gn[b, h, w, c]), float(bound[b, h, w, c])))
    return r


# ----------------------------------------------------------------------------------------------------------------------
# sige_conv_out_nhwc
# ----------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class ConvOutSpec:
    """out (NCHW) = conv3x3_pad1(act(x*scale[b] + shift[b])) + bias.  pre: which of scale / shift are passed ("both",
    "scale", "shift", "none"); scale and shift differ between images."""
    name: str
    B: int
    H: int
    W: int
    C: int
    Cout: int
    act: int = 1
    pre: str = "both"
    bias: bool = True
    seed: int = 0


CONV_OUT_CASES = [
    ConvOutSpec("c16_cout3", B=2, H=19, W=37, C=16, Cout=3, seed=1),
    ConvOutSpec("c48_cout8", B=2, H=13, W=45, C=48, Cout=8, seed=2),
    ConvOutSpec("c96_cout1", B=1, H=21, W=35, C=96, Cout=1, seed=3),
    ConvOutSpec("c128_cout4", B=2, H=27, W=70, C=128, Cout=4, seed=4),
    ConvOutSpec("c160_cout7", B=2, H=17, W=33, C=160, Cout=7, seed=5),
    ConvOutSpec("c272_cout3", B=1, H=11, W=29, C=272, Cout=3, seed=6),
    ConvOutSpec("c96_identity_scale_only", B=2, H=9, W=41, C=96, Cout=5, act=0, pre="scale", seed=7),
    ConvOutSpec("c128_swish_shift_only", B=1, H=15, W=20, C=128, Cout=2, pre="shift", seed=8),
    ConvOutSpec("c48_no_preop", B=2, H=10, W=34, C=48, Cout=6, act=0, pre="none", bias=False, seed=9),
    ConvOutSpec("c128_swish_no_affine", B=1, H=12, W=12, C=128, Cout=3, pre="none", seed=10),
    ConvOutSpec("c160_no_preop", B=1, H=9, W=9, C=160, Cout=8, act=0, pre="none", seed=11),
    ConvOutSpec("c128_no_preop", B=1, H=10, W=33, C=128, Cout=4, act=0, pre="none", seed=12),
]


def conv_out_per_element(C: int) -> bool:
    """The staging path of conv_out_kernel: per element unless every thread of the 256 keeps one channel octet."""
    return 256 % (C // 8) != 0


@dataclass
class ConvOutCase:
    spec: ConvOutSpec
    dtype: torch.dtype
    x: torch.Tensor                 # NHWC [B, H, W, C]
    scale: Optional[torch.Tensor]   # fp32 [B, C]
    shift: Optional[torch.Tensor]
    w: torch.Tensor                 # OIHW launch dtype
    bias: Optional[torch.Tensor]
    out: Guarded                    # NCHW [B, Cout, H, W]

    def buffers(self):
        return {"out": self.out}

    def inputs(self):
        out = {"x": self.x, "w": self.w}
        for k, t in (("scale", self.scale), ("shift", self.shift), ("bias", self.bias)):
            if t is not None:
                out[k] = t
        return out


def make_conv_out(spec: ConvOutSpec, dtype: torch.dtype, device) -> ConvOutCase:
    gen = torch.Generator(device=device)
    gen.manual_seed(spec.seed)
    B, C = spec.B, spec.C

    def randn(*shape, scale=1.0, dt=dtype):
        return (torch.randn(*shape, generator=gen, device=device, dtype=torch.float64) * scale).to(dt)

    x = (0.5 + randn(B, spec.H, spec.W, C, scale=1.5, dt=torch.float64)).to(dtype)
    scale = (randn(B, C, scale=0.3, dt=torch.float64) + torch.linspace(0.6, 1.2, B, device=device, dtype=torch.float64)[:, None]).float() \
        if spec.pre in ("both", "scale") else None
    shift = (randn(B, C, scale=0.3, dt=torch.float64) - 0.4 * torch.arange(B, device=device, dtype=torch.float64)[:, None]).float() \
        if spec.pre in ("both", "shift") else None
    w = randn(spec.Cout, C, 3, 3, scale=(9 * C) ** -0.5)
    bias = randn(spec.Cout, scale=0.3) if spec.bias else None
    return ConvOutCase(spec, dtype, x, scale, shift, w, bias, guarded((B, spec.Cout, spec.H, spec.W), dtype, device, gen, "nchw"))


def conv_out_call(case: ConvOutCase, lib, C: Optional[int] = None, Cout: Optional[int] = None):
    from sige_b200 import _cabi

    s = case.spec
    dt = {torch.float16: _cabi.F16, torch.bfloat16: _cabi.BF16}[case.dtype]
    return lib.sige_conv_out_nhwc(case.x.data_ptr(), _ptr(case.scale), _ptr(case.shift), s.act, case.w.data_ptr(), _ptr(case.bias),
                                  case.out.view.data_ptr(), dt, s.B, s.H, s.W, s.C if C is None else C, s.Cout if Cout is None else Cout,
                                  torch.cuda.current_stream().cuda_stream)


def conv_out_reference(case: ConvOutCase) -> List[Expect]:
    s = case.spec
    u = ROUNDOFF[case.dtype]
    a = case.x.double()
    pre = case.scale is not None or case.shift is not None or s.act != 0
    if pre:
        if case.scale is not None:
            a = a * case.scale.double()[:, None, None, :]
        if case.shift is not None:
            a = a + case.shift.double()[:, None, None, :]
        a = _act(a, s.act).to(case.dtype).double()                                     # staged in the launch dtype
    a = a.permute(0, 3, 1, 2)
    w = case.w.double()
    v = F.conv2d(a, w, padding=1)                                                       # zero padding after the pre-op
    mag = F.conv2d(a.abs(), w.abs(), padding=1)
    if case.bias is not None:
        v, mag = v + case.bias.double().view(1, -1, 1, 1), mag + case.bias.double().abs().view(1, -1, 1, 1)
    bound = u * v.abs() + ACC * mag + ABS
    if pre:
        bound = bound + PRE_ULPS * u * (w.abs().amax(dim=(1, 2, 3)) * a.abs().max()).view(1, -1, 1, 1)
    e, (want, written, b, rnd) = expect_for("out", case.out, u)
    want[:], written[:], b[:], rnd[:] = v, True, bound, u * v.abs()
    return [e]


# ----------------------------------------------------------------------------------------------------------------------
# sige_attention_tokens
# ----------------------------------------------------------------------------------------------------------------------
ATTN_SHAPES = [(64, 256), (128, 256), (256, 256), (64, 512), (128, 512), (256, 512)]
KPC = 64                        # keys per cluster CTA (one key slice)
C_P = 1.0
EXP_REL = 2.0 ** -21            # __expf: ex2.approx (about 2^-22 relative) of an fp32 product x * log2(e)
ETA = {torch.float16: 2.0 ** -25, torch.bfloat16: 0.0, torch.float32: 0.0, torch.float64: 0.0}   # half an f16 subnormal step


@dataclass(frozen=True)
class AttnSpec:
    """mode: "random" (peaked logits, q ~ 2 C^-1/2 N(0, 1)), "flat" (q = 0), "dominant" (one key, in key slice r, ~12 above the
    rest for every query), "low_slice" (key slice r ~30 below the global maximum), "large" (logits up to about +-80)."""
    name: str
    B: int
    N: int
    C: int
    mode: str
    r: int = 0
    seed: int = 0


def _attn_cases():
    cases = []
    for (N, C) in ATTN_SHAPES:
        ks = N // KPC
        for B in (1, 3):
            tag = "n%d_c%d_b%d" % (N, C, B)
            seed = N + C + B
            cases += [AttnSpec(tag + "_random", B, N, C, "random", seed=seed), AttnSpec(tag + "_flat", B, N, C, "flat", seed=seed + 1),
                      AttnSpec(tag + "_large", B, N, C, "large", seed=seed + 2)]
            cases += [AttnSpec(tag + "_dominant%d" % r, B, N, C, "dominant", r=r, seed=seed + 3 + r) for r in range(ks)]
            if ks > 1:
                cases.append(AttnSpec(tag + "_low_slice%d" % (ks - 1), B, N, C, "low_slice", r=ks - 1, seed=seed + 9))
    return cases


ATTN_CASES = _attn_cases()


@dataclass
class AttnCase:
    spec: AttnSpec
    dtype: torch.dtype
    qkv: torch.Tensor               # [B, N, 3C]
    out: Guarded                    # [B, N, C]

    def buffers(self):
        return {"out": self.out}

    def inputs(self):
        return {"qkv": self.qkv}


def make_attn(spec: AttnSpec, dtype: torch.dtype, device) -> AttnCase:
    gen = torch.Generator(device=device)
    gen.manual_seed(spec.seed)
    B, N, C = spec.B, spec.N, spec.C

    def randn(*shape):
        return torch.randn(*shape, generator=gen, device=device, dtype=torch.float64)

    q, k, v = randn(B, N, C), randn(B, N, C), randn(B, N, C)
    d = torch.where(randn(C) < 0, -1.0, 1.0)                                             # a +-1 direction, |d|^2 = C
    if spec.mode == "random":
        q = q * 2 * C ** -0.5
    elif spec.mode == "flat":
        q = torch.zeros_like(q)
    elif spec.mode in ("dominant", "low_slice"):
        # logits: q_i . k_j ~ 0.1 for ordinary keys; key j* (slice r) ~ 12; in low_slice, every key of slice r ~ -30 and
        # the maximum (~12) lies in another slice
        q = 0.1 * d + 0.05 * q
        k = 0.05 * k
        if spec.mode == "dominant":
            k[:, spec.r * KPC + 17] = (12 / (0.1 * C)) * d
        else:
            other = (spec.r + 1) % (N // KPC)
            k[:, other * KPC + 5] = (12 / (0.1 * C)) * d
            k[:, spec.r * KPC:(spec.r + 1) * KPC] -= (18 / (0.1 * C)) * d      # ~12 - 18 - 12 = 30 below the maximum
    elif spec.mode == "large":
        # q_i = a_i d / sqrt(C), k_j = t_j d / sqrt(C): logits a_i t_j with |a|, |t| <= sqrt(80)
        a = (torch.rand(B, N, 1, generator=gen, device=device, dtype=torch.float64) * 2 - 1) * 80 ** 0.5
        t = (torch.rand(B, N, 1, generator=gen, device=device, dtype=torch.float64) * 2 - 1) * 80 ** 0.5
        q = a * d / C ** 0.5 + 0.01 * q
        k = t * d / C ** 0.5 + 0.01 * k
    else:
        raise ValueError(spec.mode)
    qkv = torch.cat([q, k, v], dim=2).to(dtype).contiguous()
    return AttnCase(spec, dtype, qkv, guarded((B, N, C), dtype, device, gen, "bnc", lead_bytes=48))


def attn_call(case: AttnCase, lib, flags: int = 0):
    from sige_b200 import _cabi

    s = case.spec
    dt = {torch.float16: _cabi.F16, torch.bfloat16: _cabi.BF16}[case.dtype]
    return lib.sige_attention_tokens(case.qkv.data_ptr(), case.out.view.data_ptr(), s.B, s.N, s.C, dt, flags,
                                     torch.cuda.current_stream().cuda_stream)


def attn_reference(case: AttnCase) -> List[Expect]:
    """out = sum_j s_j v_j, s = softmax(q k^T), in float64 on the 16-bit q, k, v.

    How the kernel computes it: per key slice r (64 keys, one cluster CTA) the fp32 logits l_j, their maximum m_r, the
    numerators p_j = __expf(l_j - m_r) rounded to 16 bits, and l_r = the fp32 sum of the ROUNDED numerators; then
    out = sum_r w_r (P_r V_r) / sum_r w_r l_r with w_r = __expf(m_r - M) (fp32).  Numerator and denominator use the same
    rounded numerators and the same weights, so a relative error d_j on key j's effective weight moves the result by
    sum_j s_j d_j (v_j - want) to first order — it is centred on `want`.  Hence the c_e term, with per key
        c_e[j] = u                                    the numerator's rounding to 16 bits
               + 2 * EXP_REL                          __expf of the numerator and of the slice weight
               + 2^-23 * (|l_j - m_r| + |m_r - M|)    the fp32 rounding of their arguments times log2(e)
               + 4 * dl                               logit errors of l_j, m_r (numerator) and m_r, M (weight)
    where dl = ACC * max_j sum_c |q_c k_jc| is the fp32 error of a logit, estimated like the accumulation term of the convs;
    it grows with the logits' magnitude.  Numerators below the 16-bit normal range have an absolute error up to ETA (half an
    f16 subnormal step) rather than a relative one: the term eta * w_r / L per key, L = sum_r w_r l_r, covers them.  The
    P.V products and both sums are fp32 (ACC * mag, mag = sum_j s_j |v_j|); the output is rounded once (u * |want|).
    C_P = 1 unit of sum_j s_j |v_j| is slack for the rest of the fp32 combine (the reciprocal of L, the fmaf over slices):
    those need ~2^-23 of it; the margin keeps the bound from resting on an exact count of them."""
    s = case.spec
    u = ROUNDOFF[case.dtype]
    C, N = s.C, s.N
    q, k, v = (t.double() for t in case.qkv.split(C, dim=2))
    logits = q @ k.transpose(1, 2)                                                        # [B, N, N]
    M = logits.amax(dim=2, keepdim=True)
    sl = logits.view(s.B, N, N // KPC, KPC)
    m_r = sl.amax(dim=3, keepdim=True)                                                    # [B, N, KS, 1]
    e = torch.exp(logits - M)
    L = e.sum(dim=2, keepdim=True)
    sm = e / L
    want = sm @ v
    dl = ACC * (q.abs() @ k.abs().transpose(1, 2)).amax(dim=2, keepdim=True)            # [B, N, 1]
    ce = u + 2 * EXP_REL + 2.0 ** -23 * ((sl - m_r).abs() + (m_r - M[..., None]).abs()).view(s.B, N, N) + 4 * dl
    wr = torch.exp(m_r - M[..., None]).expand(-1, -1, -1, KPC).reshape(s.B, N, N)        # w_r(j)
    coef = ce * sm + ETA[case.dtype] * wr / L                                          # [B, Nq, Nk]
    cen = torch.empty_like(want)
    for b in range(s.B):                                                                 # [64, Nk, C] at a time
        for i0 in range(0, N, 64):
            dev_j = (v[b][None, :, :] - want[b, i0:i0 + 64, None, :]).abs()
            cen[b, i0:i0 + 64] = torch.einsum("qk,qkc->qc", coef[b, i0:i0 + 64], dev_j)
    mag = sm @ v.abs()
    bound = u * want.abs() + C_P * u * mag + cen + ACC * mag + ABS
    ex, (w, wr_, b, rnd) = expect_for("out", case.out, u)
    w[:], wr_[:], b[:], rnd[:] = want, True, bound, u * want.abs()
    return [ex]
