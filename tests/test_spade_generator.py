"""The SPADE GauGAN generator's sparse SPADE layers as modulated tile convs on channel windows.

The full SPADE (reference gaugan/models/sige_normalization.py:51,75-86) has ONE gamma/beta conv whose input is a torch.split window of
the block's shared activation and whose output is split into gamma and beta.  sige_tile_conv_strided reads such a window in place;
the lowering runs `mlp_gamma_beta` on it and hands the conv that reads the SPADE gamma / beta as windows of one buffer
(sige_tile_conv_modulated), so nothing is materialised and the compiled step takes the next label edit in place.

CPU: the in-tree generator against the reference's golden; launch counts before / after on the descriptor simulator (the in-tree file
and, when installed, the reference's); the DDPM and sub-mobile steps unchanged by the new rule; rebind on the simulator; the new entry
point's refusals and predicate.
GPU: the strided launch bitwise equal to the plain launch on a compacted copy (wgmma and mma.sync geometries, every split, PDL,
padded lists, NaN outside the window); the modulated launch with gamma / beta windows bitwise equal to compacted copies; the fused
fp16 miniature against the golden; the next edit by rebind and set_masks_async."""
import ctypes
import os
import sys
from collections import Counter

import numpy as np
import pytest
import torch
from torch.nn import functional as F

from conftest import REPO, golden

sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "baseline"))

import consumers  # noqa: E402
import tile_conv_contract as TC  # noqa: E402

def _sims():
    """(StridedSim, ModulatedSim): the descriptor simulator of test_modulated_tile_conv.py with and without the strided launch.  A
    window source or gamma / beta window reaches the simulator as a channel-slice view, which its torch math reads as it is."""
    import test_modulated_tile_conv as TM

    ModulatedSim, _ = TM._mod_sim()

    class StridedSim(ModulatedSim):
        def strided_conv_supported(self, cin, cout, k, stride):
            """sige_tile_conv_strided: a window of cin % 8 == 0 channels, Cout % 8 == 0."""
            return cin % 8 == 0 and cout % 8 == 0

    return StridedSim, ModulatedSim


def _generator(size, which):
    from sige_b200.workloads import gaugan_spade as GS

    if which == "reference":
        if not consumers.available():
            pytest.skip("baseline/_ref absent (python baseline/build_ref.py)")
        return consumers.build_gaugan(size)
    return GS.build_gaugan_spade(size)


def _counts(step):
    e = Counter(step.eager_nodes)
    return {"launches": len(step.fused), "modulated": sum(1 for f in step.fused if f.spec.modulation is not None),
            "gather": sum(v for k, v in e.items() if k.startswith("gather(")), "spade": [k for k, _ in step.steps].count("spade"),
            "to_nhwc": e["to_nhwc"], "recorded": len(step.eager_nodes)}


def _windowed(step):
    return [f.name for f in step.fused if not f.spec.src_is_stack and not f.spec.srcs[0][0].is_contiguous(memory_format=torch.channels_last)]


# ---------------------------------------------------------------------------------------------------------------- workload (CPU)
def test_in_tree_generator_matches_the_reference_golden():
    """The in-tree miniature, on the oracle runtime, reproduces the output the reference's own class produced."""
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import dilate_mask, downsample_mask

    G = golden("gaugan_mini_golden.npz")
    net = _generator("mini", "intree")
    with reference_cpu_runtime():
        full0, sparse1 = consumers.run_gaugan(net, downsample_mask, dilate_mask)
    for name, got in (("full0", full0), ("sparse1", sparse1)):
        assert np.abs(got.numpy() - G[name]).max() <= 1e-6 * max(1.0, np.abs(G[name]).max()), name
    if consumers.available():
        assert list(consumers.build_gaugan("mini").state_dict()) == list(net.state_dict())


# ---------------------------------------------------------------------------------------------------------------- lowering (CPU)
# (launches, modulated, gather( nodes, spade steps, to_nhwc copies, recorded calls) before and after the new rules
EXPECTED = {
    "full": ({"launches": 41, "modulated": 0, "gather": 33, "spade": 14, "to_nhwc": 30, "recorded": 101},
             {"launches": 41, "modulated": 14, "gather": 0, "spade": 0, "to_nhwc": 16, "recorded": 54}),
    "mini": ({"launches": 36, "modulated": 0, "gather": 28, "spade": 12, "to_nhwc": 34, "recorded": 116},
             {"launches": 36, "modulated": 12, "gather": 0, "spade": 0, "to_nhwc": 22, "recorded": 76}),
}


@pytest.mark.parametrize("which", ["intree", "reference"])
@pytest.mark.parametrize("size", ["mini", "full"])
def test_spade_layers_lower_to_strided_and_modulated_launches(size, which):
    """Every sparse SPADE layer: `mlp_gamma_beta` reads its torch.split window of the shared activation in place, and the conv that
    reads the SPADE takes gamma / beta as the two halves of that launch's buffer.  No operand stack is materialised, no modulation
    launch is left, the launch count is unchanged and the output stays the operator modules'."""
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import dilate_mask, downsample_mask
    from sige_b200.fused import FusedStep

    StridedSim, ModulatedSim = _sims()
    net = _generator(size, which)
    with reference_cpu_runtime():
        _, ref = consumers.run_gaugan(net, downsample_mask, dilate_mask, fused=lambda n: n.set_fused(False), size=size)
        args = (consumers.gaugan_inputs(size)[1],)
        with torch.no_grad():
            before = FusedStep(net, *args, executor=ModulatedSim())
            after = FusedStep(net, *args, executor=StridedSim())
    want_before, want_after = EXPECTED[size]
    assert _counts(before) == want_before
    assert _counts(after) == want_after
    assert not any(n.startswith(("sige.", "gather(")) for n in after.eager_nodes)
    mods = [f for f in after.fused if f.spec.modulation is not None]
    assert {f.spec.modulation[2] for f in mods} == {0.2, 1.0}
    # one strided launch per sparse SPADE layer: its window is an nhidden-wide part of a 2- or 3-part buffer
    assert len(_windowed(after)) == len(mods)
    for f in after.fused:
        if f.name in _windowed(after):
            t = f.spec.srcs[0][0]
            assert t.stride(3) in (2 * t.shape[1], 3 * t.shape[1]) and f.spec.Cin == t.shape[1]
    for f in mods:
        g, b, _ = f.spec.modulation
        assert g.shape == b.shape and g.shape[1] == f.spec.Cin and g.stride(3) == b.stride(3) == 2 * f.spec.Cin
        assert b.data_ptr() - g.data_ptr() == f.spec.Cin * g.element_size()
    scale = ref.abs().max().item()
    assert (after.output - ref).abs().max().item() <= 2e-5 * scale
    assert (before.output - ref).abs().max().item() <= 2e-5 * scale


def _signature(step):
    def src(t):
        return (tuple(t.shape), tuple(t.stride()))

    return ([k for k, _ in step.steps],
            [(f.name, f.spec.Cin, f.spec.Cout, f.spec.k, f.spec.stride, [src(t) for t, _ in f.spec.srcs],
              None if f.spec.modulation is None else (src(f.spec.modulation[0]), src(f.spec.modulation[1]), f.spec.modulation[2]),
              f.spec.shortcut is None) for f in step.fused],
            list(step.eager_nodes))


@pytest.mark.parametrize("kind", ["intree", "reference"])
def test_ddpm_step_is_unchanged_by_the_window_rules(kind):
    """The DDPM U-Net has no channel windows: the same steps, launches and output with and without the strided launch."""
    import test_fused_cpu as TF
    from sige_b200.fused import FusedStep
    from sige_b200.workloads.ddpm import DDPMConfig

    StridedSim, ModulatedSim = _sims()
    model, x1, t = TF._prepared(kind, DDPMConfig.small(), 0.05)
    out = []
    for ex in (ModulatedSim(), StridedSim()):
        with torch.no_grad():
            step = FusedStep(model, x1, t, executor=ex)
        out.append((_signature(step), step.output.clone()))
    assert out[0][0] == out[1][0]
    assert torch.equal(out[0][1], out[1][1])


def test_sub_mobile_step_is_unchanged_by_the_window_rules():
    """The sub-mobile generator's SPADE has separate gamma and beta convs and separable launches read its windows: the same steps,
    launches and output with and without the strided launch."""
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import dilate_mask, downsample_mask
    from sige_b200.fused import FusedStep
    from sige_b200.workloads import gaugan_gc as G

    StridedSim, ModulatedSim = _sims()
    net = G.build_gaugan_gc("mini")
    with reference_cpu_runtime():
        G.run_gaugan_gc(net, downsample_mask, dilate_mask, fused=lambda n: n.set_fused(False))
        args = (G.gaugan_gc_inputs("mini")[1],)
        out = []
        with torch.no_grad():
            for ex in (ModulatedSim(), StridedSim()):
                step = FusedStep(net, *args, executor=ex)
                out.append((_signature(step), step.output.clone()))
    assert out[0][0] == out[1][0]
    assert torch.equal(out[0][1], out[1][1])


def _edit_b():
    """A second, smaller edit of the miniature's label map elsewhere: (edited label map, its mask)."""
    s0, _, _ = consumers.gaugan_inputs("mini")
    lab = s0.argmax(1)[0].clone()
    lab[40:48, 16:28] = 3
    s1 = torch.zeros_like(s0)
    s1.scatter_(1, lab[None, None], 1.0)
    return s1, (s1 != s0).any(1)[0]


def _pyramid(mask):
    from sige.utils import dilate_mask, downsample_mask

    return downsample_mask(dilate_mask(mask, 1), min_res=(4, 8), dilation=0)


def test_rebind_installs_the_next_edit_of_the_miniature_on_the_simulator():
    """The compiled miniature takes a second, smaller edit by `rebind` (no re-trace), equal to a fresh compile of that edit exactly,
    and back on the first edit reproduces its output."""
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige_b200.fused import FusedStep

    StridedSim, _ = _sims()
    net = _generator("mini", "intree")
    s0, s1, mask_a = consumers.gaugan_inputs("mini")
    s1_b, mask_b = _edit_b()
    assert 0 < int(mask_b.sum()) < int(mask_a.sum())
    with reference_cpu_runtime(), torch.no_grad():
        net.set_mode("full")
        net(s0)
        net.set_masks(_pyramid(mask_a))
        net.set_mode("sparse")
        step = FusedStep(net, s1, executor=StridedSim(), headroom=0.5)
        assert _counts(step)["modulated"] == 12
        out_a = step(s1).clone()
        net.set_masks(_pyramid(mask_b))
        assert step.rebind()
        out_b = step(s1_b).clone()
        fresh_b = FusedStep(net, s1_b, executor=StridedSim(), headroom=0.5)(s1_b).clone()
        net.set_masks(_pyramid(mask_a))
        assert step.rebind()
        again_a = step(s1).clone()
    assert not torch.equal(out_a, out_b)
    assert torch.equal(out_b, fresh_b)
    assert torch.equal(again_a, out_a)


# ---------------------------------------------------------------------------------------------------------------- C-ABI (CPU)
def _host_desc(cin=128, cout=256, k=3, N=16):
    """Descriptor whose pointers are not device memory: only argument checks may look at them."""
    from sige_b200 import _cabi

    d = _cabi.TileConv()
    d.dtype = _cabi.F16
    d.n_src, d.src[0].ptr, d.src[0].C = 1, 0x10000, cin
    d.B, d.H, d.W, d.idx, d.N = 1, 64, 64, 0x20000, N
    d.R = d.S = 6 if k == 3 else 4
    d.w_packed, d.bias = 0x30000, 0x40000
    d.Cin, d.Cout, d.kH, d.kW, d.stride = cin, cout, k, k, 1
    d.dst, d.dH, d.dW, d.dC = 0x50000, 64, 64, cout
    d.offH = d.offW = 1 if k == 3 else 0
    d.flags = _cabi.CONV_TC5
    return d


def test_strided_refusals_come_before_any_cuda_call(cabi_lib):
    """Each refusal returns non-zero with its own message (a descriptor that passed the checks would fail at the device instead,
    with a different message: there is no device here)."""
    from sige_b200 import _cabi

    lib = _cabi.lib()

    def refused(change, what, pitch=384):
        d = _host_desc()
        change(d)
        assert lib.sige_tile_conv_strided(ctypes.byref(d), pitch, None) != 0
        assert what in lib.sige_last_error(), (what, lib.sige_last_error())

    def two_sources(d):
        d.n_src, d.src[1].ptr, d.src[1].C, d.Cin = 2, 0x18000, 64, 192

    def shortcut(d):
        d.n_src2, d.src2[0].ptr, d.src2[0].C, d.Cin2 = 1, 0x19000, 64, 64

    refused(two_sources, b"one source segment")
    refused(lambda d: setattr(d, "src_is_stack", 1), b"not a stack")
    refused(shortcut, b"no fused shortcut")
    refused(lambda d: setattr(d, "idx_per_image", 1), b"per-image")
    refused(lambda d: None, b"pixel stride", pitch=120)
    refused(lambda d: None, b"pixel stride", pitch=132)
    refused(lambda d: None, b"pixel stride", pitch=0)
    refused(lambda d: setattr(d.src[0], "ptr", 0x10008), b"16-byte aligned")
    assert lib.sige_tile_conv_strided(None, 256, None) != 0 and b"null" in lib.sige_last_error()
    d = _host_desc(N=0)
    assert lib.sige_tile_conv_strided(ctypes.byref(d), 256, None) == 0          # N == 0: no-op
    d = _host_desc()
    d.src[0].C = 12
    assert lib.sige_tile_conv_strided(ctypes.byref(d), 256, None) != 0           # and otherwise sige_tile_conv's contract
    assert b"multiple of 8" in lib.sige_last_error()


def test_strided_predicate_and_channel_windows(cabi_lib):
    import test_cabi_symbols as TS
    from sige_b200 import _cabi, ops
    from sige_b200.fused import CudaExecutor

    assert _cabi.lib().sige_abi_version() == 2
    assert set(_cabi.PROTOTYPES) == TS._declared() and "sige_tile_conv_strided" in _cabi.PROTOTYPES
    ex = CudaExecutor(torch.device("cpu"), torch.float16)
    for cin in (8, 40, 64, 128, 192):
        for k, s in ((3, 1), (1, 1), (3, 2)):
            assert ex.strided_conv_supported(cin, 256, k, s) and ops.tile_conv_strided_supported(cin, 48, k, s, torch.bfloat16)
    assert not ex.strided_conv_supported(36, 256, 3, 1) and not ex.strided_conv_supported(128, 60, 3, 1)
    assert not ops.tile_conv_strided_supported(128, 256, 3, 1, torch.float32)
    buf = torch.empty(2, 384, 5, 7, dtype=torch.float16).contiguous(memory_format=torch.channels_last)
    for c0, c1 in ((0, 384), (0, 128), (128, 256), (256, 384)):
        base, pitch, first = ops.channel_window(buf[:, c0:c1])
        assert (base, pitch, first) == (buf.data_ptr(), 384, c0)
    with pytest.raises(ValueError):
        ops.channel_window(torch.empty(2, 16, 5, 7, dtype=torch.float16))           # NCHW: channels are not innermost


# ---------------------------------------------------------------------------------------------------------------- kernels (GPU)
STRIDED_SPECS = [
    # (spec, (pitch, c0) of the window the source becomes)
    (TC.Spec("g3_copy", B=1, H=46, W=46, srcs=((128, 0),), Cout=256, counts=(120,), pad_to=136, padded=True, seed=501), (384, 128)),
    (TC.Spec("g3_preop", B=1, H=46, W=46, srcs=((128, 0),), Cout=128, counts=(100,), preop="shared", act=1, residual=(0, 0), seed=502),
     (256, 0)),
    (TC.Spec("g3_wide", B=1, H=90, W=90, srcs=((128, 0),), Cout=256, counts=(300,), seed=503), (384, 256)),
    (TC.Spec("g3_up", B=2, H=40, W=44, srcs=((64, 1),), Cout=64, counts=(60,), preop="per_sample", seed=504), (136, 72)),
    (TC.Spec("g1_copy", B=1, H=50, W=50, k=1, srcs=((128, 0),), Cout=128, counts=(150,), pad_to=160, padded=True, seed=505), (256, 128)),
    (TC.Spec("g1_preop", B=1, H=38, W=42, k=1, srcs=((64, 0),), Cout=64, counts=(70,), preop="shared", aux=((8, 8, True, 1),), seed=506),
     (192, 64)),
    (TC.Spec("s2_copy", B=1, H=34, W=30, stride=2, srcs=((64, 0),), Cout=128, counts=(40,), c_div_tile=True, seed=507), (128, 64)),
    (TC.Spec("n40", B=1, H=30, W=38, srcs=((40, 0),), Cout=64, counts=(50,), preop="shared", seed=508), (120, 40)),
    (TC.Spec("n24_k1", B=1, H=30, W=38, k=1, srcs=((24, 0),), Cout=48, counts=(40,), pad_to=48, padded=True, seed=509), (32, 8)),
    (TC.Spec("n16_up", B=1, H=32, W=40, srcs=((16, 1),), Cout=32, counts=(30,), seed=510), (48, 32)),
]


def _strided_case(spec, pitch, c0, dtype, dev):
    """The contract case of `spec` (compacted source) plus a wider buffer holding the same source at channels [c0, c0 + Cin) of
    `pitch`, NaN everywhere else."""
    from sige_b200 import ops

    case = TC.make_case(spec, dtype, dev)
    if spec.Cin % 64:
        case.wp = ops.pack_conv_weight(F.pad(case.w, (0, 0, 0, 0, 0, (spec.Cin + 63) // 64 * 64 - spec.Cin)), dtype)
    src = case.srcs[0]
    wide = torch.full((*src.shape[:3], pitch), float("nan"), dtype=dtype, device=dev)
    wide[..., c0:c0 + spec.Cin] = src
    return case, wide


def _ksplits(spec):
    J = -(-spec.Cin // 64) * spec.k * spec.k
    return [0] + [ks for ks in (1, 2, 4, 8) if ks <= J]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_strided_launch_equals_the_plain_launch_on_a_compacted_copy(dtype):
    """Every window case on the wgmma kernel (cp.async copy gather and register-staged gather) and on the mma.sync kernel (narrow
    sources included), at every split, with and without PDL and padded lists: bitwise the plain launch on the compacted window.
    The channels outside the window are NaN, so a read of any of them would show; every element the launch does not write keeps
    its initial bits."""
    from sige_b200 import _cabi

    dev = torch.device("cuda:0")
    lib = _cabi.lib()
    stream = torch.cuda.current_stream().cuda_stream
    n = 0
    for spec, (pitch, c0) in STRIDED_SPECS:
        case, wide = _strided_case(spec, pitch, c0, dtype, dev)
        init = {k: v.clone() for k, v in case.buffers().items()}
        written = {e.name: e.written for e in TC.reference(case)}
        for ks in _ksplits(spec):
            for flags in (0, TC.TC5, TC.TC5 | TC.PDL | (TC.PADDED if spec.padded else 0)):
                label = "%s %s ksplit=%d flags=%d" % (spec.name, TC.DTYPE_NAME[dtype], ks, flags)
                outs = []
                for strided in (False, True):
                    for name, buf in case.buffers().items():
                        buf.copy_(init[name])
                    d = TC.descriptor(case, ksplit=ks, flags=flags)
                    if strided:
                        d.src[0].ptr = wide[..., c0:].data_ptr()
                        _cabi.check(lib.sige_tile_conv_strided(ctypes.byref(d), pitch, stream), "sige_tile_conv_strided")
                    else:
                        _cabi.check(lib.sige_tile_conv(ctypes.byref(d), stream), "sige_tile_conv")
                    torch.cuda.synchronize()
                    outs.append({k: v.clone() for k, v in case.buffers().items()})
                for name in init:
                    plain, got = outs[0][name].view(torch.int16), outs[1][name].view(torch.int16)
                    assert torch.equal(plain, got), (label, name)
                    keep = ~written[name].to(dev)
                    assert torch.equal(got[keep], init[name].view(torch.int16)[keep]), (label, name)
                    assert not torch.isnan(outs[1][name].float()[~keep]).any(), (label, name)
                n += 1
    print("strided launches %s: %d configurations bitwise equal to the compacted launch" % (TC.DTYPE_NAME[dtype], n))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("cin,k,slope", [(128, 3, 0.2), (64, 3, 0.2), (256, 1, 1.0), (40, 3, 0.2)])
def test_modulated_launch_with_gamma_beta_windows_equals_compacted_copies(dtype, cin, k, slope):
    """gamma and beta as the two channel halves of ONE buffer (torch.split(gamma_beta, C)), passed as views: bitwise the same launch
    with gamma and beta copied into buffers of their own."""
    import test_modulated_tile_conv as TM
    from sige_b200 import _cabi, ops

    dev = torch.device("cuda:0")
    spec = TC.Spec("modwin%d_k%d" % (cin, k), B=1, H=30, W=38, srcs=((cin, 0),), Cout=128, k=k, counts=(40,), pad_to=48, padded=True,
                   preop="shared", seed=600 + cin + k)
    mc = TM._mod_case(spec, TM.Mod(slope=slope), dtype, dev)
    case = mc.case
    gb = torch.randn(1, 2 * cin, spec.H, spec.W, device=dev).mul_(0.5).to(dtype).contiguous(memory_format=torch.channels_last)
    gamma_w, beta_w = torch.split(gb, cin, dim=1)
    gamma_c, beta_c = (t.contiguous(memory_format=torch.channels_last) for t in (gamma_w, beta_w))
    init = case.dst.clone()
    stream = torch.cuda.current_stream().cuda_stream
    outs = []
    for ks in _ksplits(spec):
        for g, b in ((gamma_c, beta_c), (gamma_w, beta_w)):
            case.dst.copy_(init)
            d = TC.descriptor(case, ksplit=ks, flags=TC.PDL | TC.PADDED)
            m = ops.conv_modulation(g, b, slope)
            _cabi.check(_cabi.lib().sige_tile_conv_modulated(ctypes.byref(d), ctypes.byref(m), stream), "sige_tile_conv_modulated")
            torch.cuda.synchronize()
            outs.append(case.dst.clone())
        assert torch.equal(outs[-2].view(torch.int16), outs[-1].view(torch.int16)), ks
    assert not torch.equal(outs[-1], init)


# ---------------------------------------------------------------------------------------------------------------- fused steps (GPU)
@pytest.mark.gpu
def test_miniature_fused_fp16_with_strided_and_modulated_launches():
    from sige.utils import dilate_mask, downsample_mask

    saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        net = _generator("mini", "intree").to("cuda:0")
        consumers.run_gaugan(net, downsample_mask, dilate_mask, device="cuda:0", fused=lambda n: n.set_fused(False))
        _, fused = consumers.run_gaugan(net, downsample_mask, dilate_mask, device="cuda:0", fused=lambda n: n.set_fused(True, dtype=torch.float16))
        step = net.fused_step
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved
    c = _counts(step)
    assert c["modulated"] == 12 and c["gather"] == 0 and c["spade"] == 0 and len(_windowed(step)) == 12
    assert not any(n.startswith(("sige.", "gather(")) for n in step.eager_nodes)
    ref = golden("gaugan_mini_golden.npz")["sparse1"]
    e = np.abs(fused.float().cpu().numpy() - ref).max() / np.abs(ref).max()
    print("SPADE generator mini, strided + modulated launches: fused fp16 vs the reference's golden %.3g" % e)
    assert e <= 1e-2
    a = step.replay().clone()
    b = step.replay().clone()
    assert torch.equal(a, b), "graph replay must be idempotent"


@pytest.mark.gpu
def test_next_edit_reuses_the_compiled_spade_generator_step():
    """The miniature's compiled step takes the next label edit without recompiling: `rebind` and `set_masks_async` (the latter with
    no host synchronisation) install a second edit with the same compiled step, bitwise equal to fresh compiles."""
    dev = torch.device("cuda:0")
    net = _generator("mini", "intree").to(dev)
    s0, s1, mask_a = (t.to(dev) for t in consumers.gaugan_inputs("mini"))
    s1_b, mask_b = (t.to(dev) for t in _edit_b())
    with torch.no_grad():
        net.set_mode("full")
        net(s0)
        net.set_masks(_pyramid(mask_a))
        net.set_mode("sparse")
        net.set_fused(True, dtype=torch.float16, headroom=0.5)
        out_a = net(s1).clone()
        step = net.fused_step
        assert _counts(step)["modulated"] == 12
        pyr_b, pyr_a = _pyramid(mask_b), _pyramid(mask_a)
        net.set_masks(pyr_b)
        out_b = net(s1_b).clone()
        assert net.fused_step is step, "rebind: the second edit re-uses the compiled step"
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            assert net.set_masks_async(pyr_a) is True
        finally:
            torch.cuda.set_sync_debug_mode("default")
        out_a_async = net(s1).clone()
        assert net.fused_step is step and net.masks_async_ok()
        net.set_fused(True, dtype=torch.float16, headroom=0.5)           # fresh compiles
        net.set_masks(pyr_b)
        fresh_b = net(s1_b).clone()
        assert net.fused_step is not step
        net.set_fused(True, dtype=torch.float16, headroom=0.5)
        net.set_masks(pyr_a)
        fresh_a = net(s1).clone()
    assert not torch.equal(out_a, out_b)
    assert torch.equal(out_b, fresh_b) and torch.equal(out_a_async, fresh_a) and torch.equal(out_a, fresh_a)
