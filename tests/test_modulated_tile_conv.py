"""Modulated tile convs: sige_tile_conv with `modulation` set applies SPADE's modulation leaky((x*scale + shift) * (1 + gamma) + beta)
in the tile conv's gather stage, so the sub-mobile GauGAN generator's SPADE layers lower to one launch each and nothing is
materialised.

CPU: the C-ABI's refusals and predicate; the float64 contract's modulated gather against the C oracle's gather -> modulate -> conv ->
scatter composite; the sub-mobile generator lowered on the descriptor simulator with a CPU restatement of the modulated launch; the
DDPM step unchanged by the new rule; rebinding the compiled miniature to a second edit on the simulator.
GPU: the mma.sync kernel's modulated instantiations against the float64 contract; gamma = beta = 0 equals the plain launch bitwise;
the miniature generator as a fused fp16 step; rebind and set_masks_async on the GPU."""
import copy
import ctypes
import os
import sys
import types
from collections import Counter
from dataclasses import dataclass

import numpy as np
import pytest
import torch
from torch.nn import functional as F

from conftest import REPO

sys.path.insert(0, os.path.join(REPO, "tests"))

import tile_conv_contract as TC  # noqa: E402


# ---------------------------------------------------------------------------------------------------------------- C-ABI (CPU)
def _host_desc(cin=64, cout=64, k=3, stride=1, N=16):
    """Descriptor pointing at its modulation, whose pointers are not device memory: only argument checks may look at them."""
    from sige_b200 import _cabi

    d = _cabi.TileConv()
    d.dtype = _cabi.F16
    d.n_src, d.src[0].ptr, d.src[0].C = 1, 0x10000, cin
    d.B, d.H, d.W, d.idx, d.N = 1, 64, 64, 0x20000, N
    d.R = d.S = 6 if (k == 3 and stride == 1) else (4 if k == 1 else 5)
    d.w_packed, d.bias = 0x30000, 0x40000
    d.Cin, d.Cout, d.kH, d.kW, d.stride = cin, cout, k, k, stride
    d.dst, d.dH, d.dW, d.dC = 0x50000, 64 // stride, 64 // stride, cout
    d.offH = d.offW = 1 if (k == 3 and stride == 1) else 0
    m = _cabi.ConvModulation()
    m.gamma, m.gamma_C, m.beta, m.beta_C, m.negative_slope = 0x60000, cin, 0x70000, cin, 0.2
    d.modulation = ctypes.pointer(m)
    return d, m


def test_modulation_field_refusals_come_before_any_cuda_call(cabi_lib):
    """Each refusal returns non-zero with its own message (a descriptor that passed the checks would fail at the device
    instead, with a different message: there is no device here)."""
    from sige_b200 import _cabi

    lib = _cabi.lib()

    def refused(change, what):
        d, m = _host_desc()
        change(d, m)
        assert lib.sige_tile_conv(ctypes.byref(d), None) != 0
        assert what in lib.sige_last_error(), (what, lib.sige_last_error())

    def two_sources(d, m):
        d.n_src, d.src[1].ptr, d.src[1].C, d.Cin = 2, 0x18000, 64, 128

    def setter(**kw):
        def f(d, m):
            for k, v in kw.items():
                setattr(m if k in ("gamma", "beta", "gamma_C", "gamma_c0", "beta_C", "beta_c0", "negative_slope") else d, k, v)
        return f

    refused(two_sources, b"one source segment")
    refused(setter(src_is_stack=1), b"not a stack")
    refused(setter(act=1), b"act must be identity")
    refused(lambda d, m: (setattr(d, "n_src2", 1), setattr(d.src2[0], "C", 64), setattr(d, "Cin2", 64)), b"no fused shortcut")
    refused(setter(idx_per_image=1), b"per-image")
    refused(setter(negative_slope=float("nan")), b"finite")
    refused(setter(negative_slope=float("inf")), b"finite")
    refused(setter(gamma_C=56), b"gamma channel window")
    refused(setter(gamma_C=128, gamma_c0=72), b"gamma channel window")
    refused(setter(gamma_C=132, gamma_c0=4), b"gamma channel window")
    refused(setter(beta_C=96, beta_c0=40), b"beta channel window")
    refused(setter(beta_c0=-8, beta_C=64), b"beta channel window")
    refused(setter(gamma=0x60008), b"16-byte aligned")
    refused(setter(beta=None), b"null gamma / beta")
    refused(setter(src_pixel_stride=128), b"a source window cannot be modulated")
    assert lib.sige_tile_conv(None, None) != 0 and b"null" in lib.sige_last_error()
    d, m = _host_desc(N=0)
    m.beta = None
    assert lib.sige_tile_conv(ctypes.byref(d), None) == 0       # N == 0: no-op


def test_tile_conv_supported_and_the_refusal_of_what_it_rejects(cabi_lib):
    """ops.tile_conv_supported takes every modulated conv of the table, and sige_tile_conv refuses, before any CUDA call, each
    modulated descriptor the predicate rejects."""
    import test_cabi_symbols as TS
    from sige_b200 import _cabi, ops

    lib = _cabi.lib()
    assert lib.sige_abi_version() == 3 and set(_cabi.PROTOTYPES) == TS._declared()
    ok = ops.tile_conv_supported
    for cin in (8, 16, 40, 64, 96, 136, 256, 512, 768):
        for k, s in ((3, 1), (1, 1), (3, 2)):
            assert ok(cin, 64, k, s, torch.float16) and ok(cin, 48, k, s, torch.bfloat16)
    for cin, cout, dtype, code, why in ((36, 64, torch.float16, _cabi.F16, b"source 0 has 36 channels"),
                                        (64, 60, torch.float16, _cabi.F16, b"Cout (60) must be a multiple of 8"),
                                        (64, 64, torch.float32, _cabi.F32, b"needs f16/bf16")):
        assert not ok(cin, cout, 3, 1, dtype)
        d, m = _host_desc(cin=cin, cout=cout)
        d.dtype, m.gamma_C, m.beta_C = code, 64, 64
        assert lib.sige_tile_conv(ctypes.byref(d), None) != 0 and why in lib.sige_last_error(), lib.sige_last_error()


# ---------------------------------------------------------------------------------------------------------------- contract (CPU)
# A modulated launch is a launch of the descriptor contract (tests/tile_conv_contract.py) plus a Mod: gamma / beta buffers of Cin + extra
# channels read from channel c0 on, and the slope.  Its float64 restatement is the plain contract of the same launch on the modulated
# source image, rounded to the launch dtype once: gather, zero outside the image, conv, scatter and the error bound are the contract's.
@dataclass(frozen=True)
class Mod:
    gamma_extra: int = 0
    gamma_c0: int = 0
    beta_extra: int = 0
    beta_c0: int = 0
    slope: float = 0.2


@dataclass
class ModCase:
    case: "TC.Case"
    mod: Mod
    gamma: torch.Tensor          # NHWC [B, H, W, Cin + gamma_extra] at the source's logical extent
    beta: torch.Tensor


def make_mod_case(spec, mod: Mod, dtype, device) -> ModCase:
    case = TC.make_case(spec, dtype, device)
    gen = torch.Generator(device=device)
    gen.manual_seed(spec.seed + 7919)
    gamma, beta = ((torch.randn(spec.B, spec.H, spec.W, spec.Cin + extra, generator=gen, device=device) * 0.5).to(dtype)
                   for extra in (mod.gamma_extra, mod.beta_extra))
    return ModCase(case, mod, gamma, beta)


def modulation(mc: ModCase):
    """The sige_conv_modulation_t of a modulated case."""
    from sige_b200 import _cabi

    m = _cabi.ConvModulation()
    m.gamma, m.gamma_C, m.gamma_c0 = mc.gamma.data_ptr(), mc.gamma.shape[3], mc.mod.gamma_c0
    m.beta, m.beta_C, m.beta_c0 = mc.beta.data_ptr(), mc.beta.shape[3], mc.mod.beta_c0
    m.negative_slope = mc.mod.slope
    m._keep = mc
    return m


def modulated_source(mc: ModCase) -> torch.Tensor:
    """float64 NHWC [B, H, W, Cin]: leaky((x*scale + shift) * (1 + gamma) + beta), x up-sampled to the logical extent, rounded once to
    the launch dtype (what the kernel stages in shared memory)."""
    case, s, mod = mc.case, mc.case.spec, mc.mod
    x = torch.cat([t.double().repeat_interleave(1 << up, 1).repeat_interleave(1 << up, 2) for t, (_, up) in zip(case.srcs, s.srcs)], -1)
    assert s.act == 0
    if s.preop:
        sel = torch.arange(s.B, device=x.device) if s.preop == "per_sample" else torch.zeros(s.B, dtype=torch.long, device=x.device)
        x = x * case.scale.double()[sel][:, None, None, :] + case.shift.double()[sel][:, None, None, :]
    g = mc.gamma.double()[..., mod.gamma_c0:mod.gamma_c0 + s.Cin]
    b = mc.beta.double()[..., mod.beta_c0:mod.beta_c0 + s.Cin]
    a = x * (1 + g) + b
    return torch.where(a > 0, a, a * mod.slope).to(case.dtype).double()


def mod_reference(mc: ModCase):
    """TC.reference of the same launch on the modulated source: a single plain segment with an identity shared pre-op, so the
    contract's bound keeps its term for an operand staged in 16 bits from fp32 arithmetic."""
    import dataclasses

    case, s = mc.case, mc.case.spec
    dev = case.idx.device
    spec = dataclasses.replace(s, srcs=((s.Cin, 0),), preop="shared", act=0)
    plain = dataclasses.replace(case, spec=spec, srcs=[modulated_source(mc)], scale=torch.ones(1, s.Cin, dtype=torch.float32, device=dev),
                                shift=torch.zeros(1, s.Cin, dtype=torch.float32, device=dev))
    return TC.reference(plain)


ORACLE_CASES = [
    (TC.Spec("mod3x3", B=1, H=22, W=22, srcs=((64, 0),), Cout=64, counts=(20,), preop="shared", seed=41), Mod()),
    (TC.Spec("mod1x1_identity", B=1, H=18, W=18, k=1, srcs=((64, 0),), Cout=72, counts=(15,), residual=(0, 0), seed=42), Mod(slope=1.0)),
    (TC.Spec("mod_upsampled_windows", B=1, H=20, W=20, srcs=((64, 1),), Cout=64, counts=(18,), preop="shared", seed=43), Mod(64, 64, 8, 8)),
]


def _nchw(t):
    return np.ascontiguousarray(t.permute(0, 3, 1, 2).float().numpy())


@pytest.mark.parametrize("spec,mod", ORACLE_CASES, ids=lambda c: getattr(c, "name", ""))
def test_modulated_reference_matches_oracle(oracle, spec, mod):
    """The reference's composite on the C oracle: three Gathers (x with the folded batch norm, gamma, beta), the modulation as
    pointwise math on the tiles, conv, scatter."""
    mc = make_mod_case(spec, mod, torch.float32, "cpu")
    case = mc.case
    (dst,) = mod_reference(mc)
    s = case.spec
    gc0, bc0, slope = mod.gamma_c0, mod.beta_c0, mod.slope
    x = np.concatenate([_nchw(t).repeat(1 << up, 2).repeat(1 << up, 3) for t, (_, up) in zip(case.srcs, s.srcs)], 1)
    idx = case.idx.numpy()
    sc = sh = None
    if s.preop:
        sc, sh = case.scale.numpy().reshape(1, -1, 1, 1), case.shift.numpy().reshape(1, -1, 1, 1)
    gx = oracle.gather(x, s.R, s.R, idx, sc, sh, "identity", False)
    gg = oracle.gather(np.ascontiguousarray(_nchw(mc.gamma)[:, gc0:gc0 + s.Cin]), s.R, s.R, idx)
    gb = oracle.gather(np.ascontiguousarray(_nchw(mc.beta)[:, bc0:bc0 + s.Cin]), s.R, s.R, idx)
    z = gx * (1 + gg) + gb
    z = np.ascontiguousarray(np.where(z > 0, z, z * slope).astype(np.float32))
    tiles = oracle.conv2d_tiles(z, case.w.numpy(), case.bias.numpy(), (s.stride, s.stride))
    res = None if case.residual is None else _nchw(case.residual)
    want = oracle.scatter(tiles, _nchw(case.dst), s.off, s.off, s.stride, s.stride, idx, res)
    got = dst.want.permute(0, 3, 1, 2).numpy()
    assert float(np.abs(got - want).max()) <= 1e-5 * float(np.abs(want).max())
    assert np.array_equal(want != _nchw(case.dst), dst.written.permute(0, 3, 1, 2).numpy())


# ---------------------------------------------------------------------------------------------------------------- lowering (CPU)
def _mod_sim():
    """(ModulatedSim, NarrowSim): the descriptor simulator of test_narrow_tile_conv.py with and without a CPU restatement of
    the modulated sige_tile_conv launch."""
    import test_narrow_tile_conv as TN

    NarrowSim, _ = TN._narrow_sim()

    class ModulatedSim(NarrowSim):
        def modulated_conv_supported(self, cin, cout, k, stride):
            """ops.tile_conv_supported(): Cin and Cout multiples of 8."""
            return cin % 8 == 0 and cout % 8 == 0

        def prepare_conv(self, fc):
            """The modulated launch: leaky((x*scale + shift) * (1 + gamma) + beta) at the source's logical extent, then the plain
            launch on that (zero outside the image, as the simulator pads after the pre-op)."""
            s = fc.spec
            if s.modulation is None:
                return super().prepare_conv(fc)
            gamma, beta, slope = s.modulation
            assert len(s.srcs) == 1 and not s.src_is_stack and s.act == "identity" and s.shortcut is None and s.tile_img is None
            assert s.slot is not None, "a modulated launch reads the fixed-capacity tile list"
            x, up = s.srcs[0]
            z = torch.empty(tuple(gamma.shape), dtype=torch.float32)
            inner = copy.copy(s)
            inner.srcs, inner.scale, inner.shift, inner.modulation = [(z, 0)], None, None, None
            shim = types.SimpleNamespace(spec=inner, launch_fn=None)
            super().prepare_conv(shim)

            def run(stream):
                a = x.float()
                if up:
                    a = F.interpolate(a, scale_factor=2.0, mode="nearest")
                B = a.shape[0]
                if s.scale is not None:
                    a = a * (s.scale.view(1, -1, 1, 1) if s.scale.dim() == 1 else s.scale.view(B, -1, 1, 1))
                if s.shift is not None:
                    a = a + (s.shift.view(1, -1, 1, 1) if s.shift.dim() == 1 else s.shift.view(B, -1, 1, 1))
                m = a * (1 + gamma.float()) + beta.float()
                z.copy_(torch.where(m > 0, m, m * slope))
                shim.launch_fn(stream)

            fc.launch_fn = run

    return ModulatedSim, NarrowSim


def _lower(size):
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import dilate_mask, downsample_mask
    from sige_b200.fused import FusedStep
    from sige_b200.workloads import gaugan_gc as G

    ModulatedSim, NarrowSim = _mod_sim()
    net = G.build_gaugan_gc(size)
    with reference_cpu_runtime():
        _, ref = G.run_gaugan_gc(net, downsample_mask, dilate_mask, size=size, fused=lambda n: n.set_fused(False))
        args = (G.gaugan_gc_inputs(size)[1],)
        with torch.no_grad():
            step = FusedStep(net, *args, executor=ModulatedSim())
            before = FusedStep(net, *args, executor=NarrowSim())
    return step, before, ref


def _counts(step):
    e = Counter(step.eager_nodes)
    return (sum(v for k, v in e.items() if k.startswith("gather(")), [k for k, _ in step.steps].count("spade"), len(step.fused),
            sum(1 for f in step.fused if f.spec.modulation is not None), len(step.eager_nodes))


@pytest.mark.parametrize("size,before,after", [
    # (gather( eager nodes, spade steps, tile-conv launches, modulated launches, recorded calls)
    ("full", (42, 14, 31, 0, 112), (0, 0, 31, 14, 70)),
    # the miniature's three dense blocks keep their six modulation launches (dense SPADE layers have no tile list)
    ("mini", (36, 18, 28, 0, 112), (0, 6, 28, 12, 76)),
])
def test_sub_mobile_generator_modulates_in_the_gather_stage(size, before, after):
    """Sub-mobile GauGAN on the simulator: every sparse SPADE layer's modulation becomes the gather stage of the conv that reads it,
    so no operand stack is materialised (gather) and no sparse modulation launch is left (spade); the launch count is unchanged and the
    output stays the operator modules'.  In the learned-shortcut blocks conv_1 and conv_s stay two launches."""
    step, prev, ref = _lower(size)
    assert _counts(prev) == before
    assert _counts(step) == after
    mods = [f for f in step.fused if f.spec.modulation is not None]
    assert {f.spec.modulation[2] for f in mods} == {0.2, 1.0}
    assert all(f.spec.shortcut is None for f in step.fused)
    assert not any(n.startswith(("sige.", "gather(")) for n in step.eager_nodes)
    scale = ref.abs().max().item()
    assert (step.output - ref).abs().max().item() <= 2e-5 * scale
    assert (prev.output - ref).abs().max().item() <= 2e-5 * scale


@pytest.mark.parametrize("kind", ["intree", "reference"])
def test_ddpm_step_is_unchanged_by_the_modulation_rule(kind):
    """The DDPM U-Net has no SPADE layer: the same launches with and without the modulated launch."""
    import test_fused_cpu as TF
    from sige_b200.fused import FusedStep
    from sige_b200.workloads.ddpm import DDPMConfig

    ModulatedSim, NarrowSim = _mod_sim()
    model, x1, t = TF._prepared(kind, DDPMConfig.small(), 0.05)
    out = []
    for ex in (NarrowSim(), ModulatedSim()):
        with torch.no_grad():
            step = FusedStep(model, x1, t, executor=ex)
        out.append(([k for k, _ in step.steps], [(f.name, f.spec.Cin, f.spec.Cout, f.spec.k, f.spec.modulation is None, f.spec.shortcut is None)
                                                for f in step.fused], list(step.eager_nodes), step.output.clone()))
    assert out[0][:3] == out[1][:3]
    assert torch.equal(out[0][3], out[1][3])


def _edit_b(size="mini"):
    """A second, smaller edit of the miniature's label map elsewhere: (edited label map, its mask)."""
    from sige_b200.workloads import gaugan_gc as G

    s0, _, _ = G.gaugan_gc_inputs(size)
    lab = s0.argmax(1)[0].clone()
    lab[40:48, 16:28] = 3
    s1 = torch.zeros_like(s0)
    s1.scatter_(1, lab[None, None], 1.0)
    return s1, (s1 != s0).any(1)[0]


def _pyramid(mask):
    from sige.utils import dilate_mask, downsample_mask

    return downsample_mask(dilate_mask(mask, 1), min_res=(4, 8), dilation=0)


def test_rebind_installs_the_next_edit_of_the_miniature_on_the_simulator():
    """With nothing holding a tile list of its own, the compiled step takes a second, smaller edit by `rebind` (no re-trace):
    equal to a fresh compile of that edit exactly, and back on edit A it reproduces the first output."""
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige_b200.fused import FusedStep
    from sige_b200.workloads import gaugan_gc as G

    ModulatedSim, _ = _mod_sim()
    net = G.build_gaugan_gc("mini")
    s0, s1, mask_a = G.gaugan_gc_inputs("mini")
    s1_b, mask_b = _edit_b()
    assert 0 < int(mask_b.sum()) < int(mask_a.sum())
    with reference_cpu_runtime(), torch.no_grad():
        net.set_mode("full")
        net(s0)
        net.set_masks(_pyramid(mask_a))
        net.set_mode("sparse")
        step = FusedStep(net, s1, executor=ModulatedSim(), headroom=0.5)
        assert sum(1 for f in step.fused if f.spec.modulation is not None) == 12
        out_a = step(s1).clone()
        net.set_masks(_pyramid(mask_b))
        assert step.rebind()
        out_b = step(s1_b).clone()
        fresh_b = FusedStep(net, s1_b, executor=ModulatedSim(), headroom=0.5)(s1_b).clone()
        net.set_masks(_pyramid(mask_a))
        assert step.rebind()
        again_a = step(s1).clone()
    assert not torch.equal(out_a, out_b)
    assert torch.equal(out_b, fresh_b)
    assert torch.equal(again_a, out_a)


# ---------------------------------------------------------------------------------------------------------------- kernel (GPU)
def _mod_specs():
    """Cin x geometry x features; each (spec, Mod) is one modulated launch of the contract (3x3 on 6x6 tiles, 1x1 on 4x4 tiles; border
    tiles always, SIGE_TILE_NONE padding, gamma / beta channel windows, up-sampled sources, identity slope)."""
    specs, seed = [], 300
    cins = (8, 16, 24, 40, 48, 96, 136, 64, 256, 512, 768)
    for i, cin in enumerate(cins):
        for j, k in enumerate((3, 1)):
            v = (i + j) % 4
            if v == 0:
                kw, mod = dict(preop="shared", counts=(37,), pad_to=48, padded=True), Mod()
            elif v == 1:
                kw, mod = dict(B=2, preop="per_sample", counts=(21,), pad_to=24, residual=(8, 8)), Mod(16, 8, 8, 0)
            elif v == 2:
                kw, mod = dict(preop="shared", counts=(33,), dst=(16, 8), aux=((8, 0, False, 0),)), Mod(cin, cin, 0, 0, 1.0)
            else:
                kw, mod = dict(counts=(27,), pad_to=32), Mod(0, 0, 24, 16)
            up = 1 if (i % 3 == 1 and k == 3) else 0
            cout = (48, 64, 96, 144)[(i + j) % 4]
            B = kw.pop("B", 1)
            seed += 1
            specs.append((TC.Spec("m%d_c%d_k%d_v%d%s" % (cin, cout, k, v, "_up" if up else ""), B=B, H=30, W=38, srcs=((cin, up),), Cout=cout,
                                  k=k, seed=seed, **kw), mod))
    return specs


def _pad64(c):
    return (c + 63) // 64 * 64


def _mod_case(spec, mod, dtype, dev) -> ModCase:
    from sige_b200 import ops

    mc = make_mod_case(spec, mod, dtype, dev)
    mc.case.wp = ops.pack_conv_weight(F.pad(mc.case.w, (0, 0, 0, 0, 0, _pad64(spec.Cin) - spec.Cin)), dtype)
    return mc


def _launch(mc: ModCase, ksplit, flags, mod=True):
    """The modulated launch of `mc`, or (mod=False) the plain launch of the same descriptor."""
    from sige_b200 import _cabi

    d = TC.descriptor(mc.case, ksplit=ksplit, flags=flags)
    if mod:
        d.modulation = ctypes.pointer(modulation(mc))
    _cabi.check(_cabi.lib().sige_tile_conv(ctypes.byref(d), torch.cuda.current_stream().cuda_stream), "sige_tile_conv")
    torch.cuda.synchronize()


def _ksplits(spec):
    J = -(-spec.Cin // 64) * spec.k * spec.k
    return [0] + [ks for ks in (1, 2, 4, 8) if ks <= J]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_modulation_field_against_the_float64_contract(dtype):
    """Every modulated case, at every split the plan allows, with and without PDL: within the contract's bound and every element
    it does not write bitwise unchanged."""
    dev = torch.device("cuda:0")
    worst = excess = 0.0
    n = 0
    for spec, mod in _mod_specs():
        mc = _mod_case(spec, mod, dtype, dev)
        case = mc.case
        init = {k: v.clone() for k, v in case.buffers().items()}
        expects = mod_reference(mc)
        for ks in _ksplits(spec):
            for flags in (TC.TC5, TC.TC5 | TC.PDL | (TC.PADDED if spec.padded else 0)):
                for name, buf in case.buffers().items():
                    buf.copy_(init[name])
                _launch(mc, ks, flags)
                got = {k: v.clone() for k, v in case.buffers().items()}
                w_, e_ = TC.check("%s %s ksplit=%d flags=%d" % (spec.name, TC.DTYPE_NAME[dtype], ks, flags), expects, got, init)
                worst, excess, n = max(worst, w_), max(excess, e_), n + 1
    print("modulated contract %s: %d launches, worst error/bound %.3f, accumulation headroom used %.3f" % (TC.DTYPE_NAME[dtype], n, worst, excess))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("cin,k", [(40, 3), (64, 3), (512, 3), (96, 1), (256, 1)])
def test_zero_modulation_field_equals_the_plain_launch(dtype, cin, k):
    """gamma = beta = 0 and slope 1: bitwise the existing mma.sync launch with the same scale / shift pre-op."""
    dev = torch.device("cuda:0")
    spec = TC.Spec("zero%d_k%d" % (cin, k), B=1, H=30, W=38, srcs=((cin, 0),), Cout=64, k=k, counts=(40,), preop="shared", seed=cin + k)
    mc = _mod_case(spec, Mod(slope=1.0), dtype, dev)
    mc.gamma.zero_()
    mc.beta.zero_()
    case = mc.case
    init = case.dst.clone()
    for ks in _ksplits(spec):
        case.dst.copy_(init)
        _launch(mc, ks, 0)
        got = case.dst.clone()
        case.dst.copy_(init)
        _launch(mc, ks, 0, mod=False)
        assert torch.equal(got.view(torch.int16), case.dst.view(torch.int16)), ks


# ---------------------------------------------------------------------------------------------------------------- fused steps (GPU)
@pytest.mark.gpu
def test_sub_mobile_miniature_fused_fp16_with_modulated_launches():
    from sige.utils import dilate_mask, downsample_mask
    from sige_b200.workloads import gaugan_gc as G

    import test_separable_conv as TS

    saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        net = G.build_gaugan_gc("mini").to("cuda:0")
        _, via_modules = G.run_gaugan_gc(net, downsample_mask, dilate_mask, device="cuda:0", fused=lambda n: n.set_fused(False))
        _, fused = G.run_gaugan_gc(net, downsample_mask, dilate_mask, device="cuda:0", fused=lambda n: n.set_fused(True, dtype=torch.float16))
        step = net.fused_step
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved
    assert sum(1 for f in step.fused if f.spec.modulation is not None) == 12
    assert not any(n.startswith(("sige.", "gather(")) for n in step.eager_nodes)
    assert [k for k, _ in step.steps].count("spade") == 0
    ref = via_modules.float().cpu().numpy()
    G_ = TS._golden_or_none()
    if G_ is not None:
        ref = G_["sparse1"]
    e = np.abs(fused.float().cpu().numpy() - ref).max() / np.abs(ref).max()
    print("sub-mobile mini with modulated launches: fused fp16 vs %s %.3g" % ("golden" if G_ is not None else "fp32 operator modules", e))
    assert e <= 1e-2
    a = step.replay().clone()
    b = step.replay().clone()
    assert torch.equal(a, b), "graph replay must be idempotent"


@pytest.mark.gpu
def test_next_edit_reuses_the_compiled_generator_step():
    """The whole sub-mobile miniature step takes the next label edit without recompiling: `rebind` and `set_masks_async` (the
    latter with no host synchronisation) install a second edit with the same compiled step, bitwise equal to a fresh compile."""
    from sige.utils import dilate_mask, downsample_mask
    from sige_b200.workloads import gaugan_gc as G

    dev = torch.device("cuda:0")
    net = G.build_gaugan_gc("mini").to(dev)
    s0, s1, mask_a = (t.to(dev) for t in G.gaugan_gc_inputs("mini"))
    s1_b, mask_b = (t.to(dev) for t in _edit_b())

    def pyr(m):
        return downsample_mask(dilate_mask(m, 1), min_res=(4, 8), dilation=0)

    with torch.no_grad():
        net.set_mode("full")
        net(s0)
        net.set_masks(pyr(mask_a))
        net.set_mode("sparse")
        net.set_fused(True, dtype=torch.float16, headroom=0.5)
        out_a = net(s1)
        step = net.fused_step
        assert sum(1 for f in step.fused if f.spec.modulation is not None) == 12
        pyr_b, pyr_a = pyr(mask_b), pyr(mask_a)
        net.set_masks(pyr_b)
        out_b = net(s1_b)
        assert net.fused_step is step, "rebind: the second edit re-uses the compiled step"
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            assert net.set_masks_async(pyr_a) is True
        finally:
            torch.cuda.set_sync_debug_mode("default")
        out_a_async = net(s1)
        assert net.fused_step is step and net.masks_async_ok()
        net.set_fused(True, dtype=torch.float16, headroom=0.5)           # fresh compiles
        net.set_masks(pyr_b)
        fresh_b = net(s1_b)
        assert net.fused_step is not step
        net.set_fused(True, dtype=torch.float16, headroom=0.5)
        net.set_masks(pyr_a)
        fresh_a = net(s1)
    assert torch.equal(out_b, fresh_b) and torch.equal(out_a_async, fresh_a) and torch.equal(out_a, fresh_a)
