"""Narrow tile convs: sige_tile_conv on one source whose channel count is a multiple of 8 but not of 64 (the layers of pruned /
compressed models, e.g. the 16...96-channel convs of GAN Compression's sub-mobile GauGAN), and the fused ReLU epilogue
(SIGE_ACT_RELU on an aux destination).

CPU: the C-ABI's refusals and launch plan; the sub-mobile generator lowered on the descriptor simulator with a CPU restatement of
the narrow launch and of the ReLU epilogue; the DDPM step is unchanged by the new rules.
GPU: the mma.sync kernel on narrow sources against the float64 restatement of the descriptor (tests/tile_conv_contract.py),
bitwise against the same launch on the source zero-padded to a multiple of 64 channels; the ReLU epilogue; the miniature
generator as a fused fp16 step; re-binding a compiled step to the next edit."""
import ctypes
import os
import sys
from collections import Counter

import numpy as np
import pytest
import torch
from torch.nn import functional as F

from conftest import REPO

sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "baseline"))

import mma_tile_conv_contract as MC  # noqa: E402
import tile_conv_contract as TC  # noqa: E402

ACT_RELU = 2


# ---------------------------------------------------------------------------------------------------------------- C-ABI (CPU)
def _host_desc(srcs=((40, 0),), cout=48, k=3, stride=1, n_src2=0):
    """A descriptor whose pointers are not device memory: only argument checks and the plan may look at it."""
    from sige_b200 import _cabi

    d = _cabi.TileConv()
    d.dtype = _cabi.F16
    d.n_src = len(srcs)
    for i, (c, up) in enumerate(srcs):
        d.src[i].ptr, d.src[i].C, d.src[i].up = 0x10000 + 0x1000 * i, c, up
    d.B, d.H, d.W, d.idx, d.N = 1, 64, 64, 0x20000, 16
    d.R = d.S = 6 if (k == 3 and stride == 1) else (4 if k == 1 else 5)
    d.w_packed, d.bias = 0x30000, 0x40000
    d.Cin, d.Cout, d.kH, d.kW, d.stride = sum(c for c, _ in srcs), cout, k, k, stride
    d.dst, d.dH, d.dW, d.dC = 0x50000, 64 // stride, 64 // stride, cout
    d.offH = d.offW = 1 if (k == 3 and stride == 1) else 0
    d.flags = TC.TC5
    if n_src2:
        d.n_src2, d.src2[0].ptr, d.src2[0].C, d.Cin2, d.w2_packed = 1, 0x60000, 64, 64, 0x70000
    return d


def test_narrow_launch_refusals_come_before_any_cuda_call(cabi_lib):
    from sige_b200 import _cabi

    lib = _cabi.lib()

    def refused(d, what):
        assert lib.sige_tile_conv(ctypes.byref(d), None) != 0
        assert what in lib.sige_last_error(), lib.sige_last_error()

    refused(_host_desc(srcs=((40, 0), (64, 0))), b"concatenated")
    refused(_host_desc(srcs=((64, 0), (24, 0))), b"concatenated")
    refused(_host_desc(srcs=((36, 0),)), b"multiple of 8")
    refused(_host_desc(srcs=((64, 0), (36, 0))), b"multiple of 8")
    refused(_host_desc(srcs=((96, 0),), n_src2=1), b"fused shortcut")
    d = _host_desc()
    d.act = ACT_RELU                        # ReLU is an epilogue activation only, never the gather stage's pre-op
    refused(d, b"unknown activation")
    d = _host_desc()
    d.n_aux, d.aux[0].ptr, d.aux[0].C, d.aux[0].act = 1, 0x80000, 48, 3
    refused(d, b"aux 0 unknown activation")
    # the other entry points keep the activations they take: identity and swish
    assert lib.sige_gather(0x10000, _cabi.F16, _cabi.NHWC, 1, 64, 8, 8, 6, 6, 0x20000, 4, None, None, ACT_RELU, 0, 0x30000, None) != 0
    aux = _cabi.ConvAux()
    aux.ptr, aux.C, aux.c0, aux.act = 0x50000, 64, 0, ACT_RELU
    assert lib.sige_conv_in_nhwc(0x10000, 0x20000, None, 0x30000, _cabi.F16, 1, 8, 8, 3, 64, 1, ctypes.byref(aux), None) != 0
    assert b"unknown activation" in lib.sige_last_error()


def test_narrow_launches_plan_on_the_mma_sync_kernel(cabi_lib):
    for cin in range(8, 137, 8):
        if cin % 64 == 0:
            continue
        for k, stride in ((3, 1), (1, 1), (3, 2)):
            p = TC.plan_of(_host_desc(srcs=((cin, 0),), cout=64, k=k, stride=stride))
            R = 6 if (k == 3 and stride == 1) else (4 if k == 1 else 5)
            want = MC.plan(16, R, R, k, k, stride, cin, 64, 0)       # 16 tiles: the S configuration, K split while a slice keeps 4 steps
            assert p.path == 0 and MC.plan_tuple(p) == MC.expected_plan_tuple(want) and want.config == "S", (cin, k, stride)


# ---------------------------------------------------------------------------------------------------------------- lowering (CPU)
def _narrow_sim():
    """The descriptor simulator with the separable launch (test_separable_conv.py) and the narrow launch restated."""
    import test_separable_conv as TS

    SeparableSim, _ = TS._sim_executors()

    class NarrowSim(SeparableSim):
        def narrow_conv_supported(self, cin, cout, k, stride):
            """sige_tile_conv on one source of cin % 8 == 0 channels (the weight is zero-padded like the source: exact)."""
            return cin % 8 == 0 and cin % 64 != 0 and cout % 8 == 0

        def prepare_conv(self, fc):
            """The ReLU epilogue: relu(conv + bias [+ residual]) where the launch writes.  Every element it does not write is a
            cached post-ReLU value (>= 0, checked), so ReLU over the whole destination after the launch is the same thing."""
            super().prepare_conv(fc)
            s, inner = fc.spec, fc.launch_fn
            assert s.Cin == sum(int(t.shape[1]) for t, _ in s.srcs) and (s.Cin % 64 == 0 or len(s.srcs) == 1)
            if s.epilogue_act == "identity":
                return
            assert s.epilogue_act == "relu" and not s.aux and s.shortcut is None

            def run(stream):
                out = s.dst_stack if s.dst_stack is not None else s.dst.raw
                assert s.dst_stack is not None or bool((out >= 0).all())
                inner(stream)
                out.clamp_(min=0)

            fc.launch_fn = run

    return NarrowSim, SeparableSim


def _lower(size):
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import dilate_mask, downsample_mask
    from sige_b200.fused import FusedStep
    from sige_b200.workloads import gaugan_gc as G

    NarrowSim, SeparableSim = _narrow_sim()
    net = G.build_gaugan_gc(size)
    with reference_cpu_runtime():
        _, ref = G.run_gaugan_gc(net, downsample_mask, dilate_mask, size=size, fused=lambda n: n.set_fused(False))
        args = (G.gaugan_gc_inputs(size)[1],)
        with torch.no_grad():
            step = FusedStep(net, *args, executor=NarrowSim())
            before = FusedStep(net, *args, executor=SeparableSim())
    return step, before, ref


def _kinds(step):
    e = Counter(step.eager_nodes)
    return {k: e[k] for k in ("sige.conv", "sige.scatter_block_residual", "relu", "sige.gather", "sige.scatter_gather", "to_nhwc")}, len(step.eager_nodes)


@pytest.mark.parametrize("size,before_kinds,after_kinds", [
    ("full", ({"sige.conv": 12, "sige.scatter_block_residual": 3, "relu": 7, "sige.gather": 5, "sige.scatter_gather": 7, "to_nhwc": 28}, 150),
             ({"sige.conv": 0, "sige.scatter_block_residual": 0, "relu": 2, "sige.gather": 0, "sige.scatter_gather": 0, "to_nhwc": 20}, 112)),
    ("mini", ({"sige.conv": 8, "sige.scatter_block_residual": 2, "relu": 7, "sige.gather": 4, "sige.scatter_gather": 5, "to_nhwc": 26}, 148),
             ({"sige.conv": 0, "sige.scatter_block_residual": 0, "relu": 3, "sige.gather": 0, "sige.scatter_gather": 0, "to_nhwc": 20}, 112)),
])
def test_sub_mobile_generator_lowers_its_narrow_convs(size, before_kinds, after_kinds):
    """Sub-mobile GauGAN on the simulator: with the narrow launch every sparse conv is fused (the 36-channel label map is gathered
    from a zero-padded 40-channel copy, mlp_shared's ReLU is its launch's epilogue, conv_1 and the shortcut of a learned-shortcut
    block scatter as two launches); the ReLUs left belong to the dense blocks.  The output stays the operator modules'."""
    step, before, ref = _lower(size)
    assert _kinds(before) == before_kinds
    assert _kinds(step) == after_kinds
    relu_launches = [f for f in step.fused if f.spec.epilogue_act == "relu"]
    assert len(relu_launches) == {"full": 5, "mini": 4}[size]
    assert all(f.spec.Cin == 40 and int(f.spec.srcs[0][0].shape[1]) == 40 for f in relu_launches)
    assert all(float(f.spec.weight[:, 36:].abs().max()) == 0.0 for f in relu_launches)
    assert any(f.spec.Cin % 64 for f in step.fused if f.spec.epilogue_act == "identity")
    scale = ref.abs().max().item()
    assert (step.output - ref).abs().max().item() <= 2e-5 * scale
    assert (before.output - ref).abs().max().item() <= 2e-5 * scale


def _ddpm_launches(kind):
    import test_fused_cpu as TF
    from sige_b200.fused import FusedStep
    from sige_b200.workloads.ddpm import DDPMConfig
    from sim_executor import SimExecutor

    NarrowSim, _ = _narrow_sim()
    model, x1, t = TF._prepared(kind, DDPMConfig.small(), 0.05)
    out = []
    for ex in (SimExecutor(), NarrowSim()):
        with torch.no_grad():
            step = FusedStep(model, x1, t, executor=ex)
        out.append(([k for k, _ in step.steps], [(f.name, f.spec.Cin, f.spec.Cout, f.spec.k, f.spec.epilogue_act, f.spec.shortcut is None)
                                                for f in step.fused], list(step.eager_nodes), step.output.clone()))
    return out


@pytest.mark.parametrize("kind", ["intree", "reference"])
def test_ddpm_step_is_unchanged_by_the_narrow_rules(kind):
    """Every width of the DDPM U-Net is a multiple of 64: the same launches with and without the narrow launch."""
    plain, narrow = _ddpm_launches(kind)
    assert plain[:3] == narrow[:3]
    assert torch.equal(plain[3], narrow[3])


# ---------------------------------------------------------------------------------------------------------------- kernel (GPU)
def _pad64(c):
    return (c + 63) // 64 * 64


def _narrow_specs():
    """Cin x Cout x geometry x features; each spec is one narrow launch of the contract."""
    specs, seed = [], 100
    cins, couts = (8, 16, 24, 32, 40, 48, 96, 136), (16, 32, 48, 96, 144)
    geoms = ((3, 1), (1, 1), (3, 2))
    for i, cin in enumerate(cins):
        for j, (k, stride) in enumerate(geoms):
            cout = couts[(i + j) % len(couts)]
            variant = (i + j) % 4
            kw = {}
            if variant == 0:
                kw = dict(preop="shared", act=1, residual=(8, 8), counts=(37,), pad_to=48, padded=True)
            elif variant == 1:
                kw = dict(B=2, per_image=True, preop="per_sample", act=1, counts=(30, 19), pad_to=32, aux=((0, 0, True, 1),))
            elif variant == 2:
                kw = dict(dst=(16, 8), aux=((8, 0, False, 0),), counts=(41,))
            else:
                kw = dict(B=2, residual=(0, 0), dst=None, aux=((0, 0, True, 0),), counts=(23,))
            B = kw.pop("B", 1)
            H, W = (34, 30) if stride == 2 else (30, 38)
            seed += 1
            specs.append(TC.Spec("n%d_c%d_k%ds%d_v%d" % (cin, cout, k, stride, variant), B=B, H=H, W=W, srcs=((cin, 0),), Cout=cout, k=k,
                                 stride=stride, c_div_tile=stride == 2, seed=seed, **kw))
    return specs


def _ksplits(spec):
    J = -(-spec.Cin // 64) * spec.k * spec.k
    return [0] + [ks for ks in (1, 2, 4, 8) if ks <= J]


def _narrow_case(spec, dtype, dev):
    from sige_b200 import ops

    case = TC.make_case(spec, dtype, dev)
    cp = _pad64(spec.Cin)
    case.wp = ops.pack_conv_weight(F.pad(case.w, (0, 0, 0, 0, 0, cp - spec.Cin)), dtype)
    return case


def _padded_twin(case, dev):
    """The same launch on the source zero-padded to a multiple of 64 channels (scale 1 / shift 0 on the padding), writing into
    copies of the case's buffers: what the operator modules run for such a conv."""
    import dataclasses

    from sige_b200 import ops

    s = case.spec
    cp = _pad64(s.Cin)
    srcs = [F.pad(x, (0, cp - s.Cin)).contiguous() for x in case.srcs]
    scale = None if case.scale is None else F.pad(case.scale, (0, cp - s.Cin), value=1.0).contiguous()
    shift = None if case.shift is None else F.pad(case.shift, (0, cp - s.Cin)).contiguous()
    w = F.pad(case.w, (0, 0, 0, 0, 0, cp - s.Cin))
    spec = dataclasses.replace(s, srcs=((cp, 0),))
    aux = [TC.Aux(a.buf.clone(), a.c0, a.scale, a.shift, a.act) for a in case.aux]
    twin = TC.Case(spec, case.dtype, srcs, case.idx, scale, shift, w, case.bias, None if case.dst is None else case.dst.clone(),
                   case.residual, aux)
    twin.wp = ops.pack_conv_weight(w, case.dtype)
    return twin


def _launch(case, ksplit, flags):
    from sige_b200 import _cabi

    d = TC.descriptor(case, ksplit=ksplit, flags=flags)
    _cabi.check(_cabi.lib().sige_tile_conv(ctypes.byref(d), torch.cuda.current_stream().cuda_stream), "sige_tile_conv")
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_narrow_tile_conv_against_the_float64_contract(dtype):
    """Every narrow case, at every split the plan allows, with and without PDL: within the contract's bound, untouched elements
    bitwise unchanged, and bitwise equal to the launch on the source zero-padded to a multiple of 64 channels."""
    dev = torch.device("cuda:0")
    worst = excess = 0.0
    n = 0
    for spec in _narrow_specs():
        case = _narrow_case(spec, dtype, dev)
        assert TC.plan_of(TC.descriptor(case)).path == 0
        init = {k: v.clone() for k, v in case.buffers().items()}
        expects = TC.reference(case)
        twin = _padded_twin(case, dev)
        twin_init = {k: v.clone() for k, v in twin.buffers().items()}
        for ks in _ksplits(spec):
            for flags in (TC.TC5, TC.TC5 | TC.PDL | (TC.PADDED if spec.padded else 0)):
                for name, buf in case.buffers().items():
                    buf.copy_(init[name])
                _launch(case, ks, flags)
                got = {k: v.clone() for k, v in case.buffers().items()}
                w_, e_ = TC.check("%s %s ksplit=%d flags=%d" % (spec.name, TC.DTYPE_NAME[dtype], ks, flags), expects, got, init)
                worst, excess, n = max(worst, w_), max(excess, e_), n + 1
                for name, buf in twin.buffers().items():
                    buf.copy_(twin_init[name])
                _launch(twin, ks, flags)
                for name, buf in twin.buffers().items():
                    assert torch.equal(buf.view(torch.int16), got[name].view(torch.int16)), \
                        "%s ksplit=%d flags=%d: %s differs from the zero-padded launch" % (spec.name, ks, flags, name)
    print("narrow contract %s: %d launches, worst error/bound %.3f, accumulation headroom used %.3f" % (TC.DTYPE_NAME[dtype], n, worst, excess))


def _stack_conv(x, wp, bias, k, ksplit):
    """sige_tile_conv on a narrow tile stack (M, Cin, R, R) -> (M, Cout, Ro, Ro), the weight packed padded to a multiple of 64."""
    from sige_b200 import _cabi

    M, cin, R, _ = x.shape
    cout = wp.shape[1]
    ro = R - k + 1
    out = torch.empty(M, cout, ro, ro, dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
    d = _cabi.TileConv()
    d.dtype = {torch.float16: _cabi.F16, torch.bfloat16: _cabi.BF16}[x.dtype]
    d.n_src, d.src[0].ptr, d.src[0].C = 1, x.data_ptr(), cin
    d.B, d.H, d.W, d.src_is_stack, d.N, d.R, d.S = 1, R, R, 1, M, R, R
    d.w_packed, d.bias = wp.data_ptr(), bias.data_ptr()
    d.Cin, d.Cout, d.kH, d.kW, d.stride = cin, cout, k, k, 1
    d.dst, d.dst_is_stack, d.dH, d.dW, d.dC = out.data_ptr(), 1, ro, ro, cout
    d.flags, d.ksplit = TC.TC5, ksplit
    _cabi.check(_cabi.lib().sige_tile_conv(ctypes.byref(d), torch.cuda.current_stream().cuda_stream), "sige_tile_conv")
    torch.cuda.synchronize()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("cin,cout,k", [(40, 144, 3), (24, 48, 3), (96, 32, 1), (136, 96, 3)])
def test_narrow_stack_source_equals_the_zero_padded_stack(dtype, cin, cout, k):
    """Tile-stack source and destination (the sparse operator modules' layout): bitwise equal to the zero-padded launch, and
    within fp32-accumulation error of float64 torch."""
    from sige_b200 import ops

    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(cin + cout)
    R = 6 if k == 3 else 4
    x = torch.randn(53, cin, R, R, generator=gen, device=dev).to(dtype).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(cout, cin, k, k, generator=gen, device=dev) / (cin * k * k) ** 0.5).to(dtype)
    b = torch.randn(cout, generator=gen, device=dev)
    cp = _pad64(cin)
    wp = ops.pack_conv_weight(F.pad(w, (0, 0, 0, 0, 0, cp - cin)), dtype)
    xp = torch.zeros(53, cp, R, R, dtype=dtype, device=dev).contiguous(memory_format=torch.channels_last)
    xp[:, :cin] = x
    for ks in [0] + [s for s in (1, 2, 4, 8) if s <= -(-cin // 64) * k * k]:
        got = _stack_conv(x, wp, b, k, ks)
        want = ops.tile_conv_stack(xp, wp, b, (k, k), 1, ksplit=ks)
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), ks
    ref = F.conv2d(x.double(), w.double(), b.double())
    mag = F.conv2d(x.double().abs(), w.double().abs(), b.double().abs())
    u = TC.UNIT_ROUNDOFF[dtype]
    assert bool(((got.double() - ref).abs() <= u * ref.abs() + TC.ACC * mag + TC.ABS).all())


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("cin,residual", [(40, False), (48, True), (128, True)])
def test_relu_epilogue_is_the_clamped_destination(dtype, cin, residual):
    """dst = NULL and one ReLU aux with no affine writes relu(conv + bias [+ residual]): the plain launch's destination clamped at
    zero (equal as values; ReLU of a negative result that rounds to -0 is +0), on the narrow kernel and the wgmma kernel."""
    import dataclasses

    dev = torch.device("cuda:0")
    spec = TC.Spec("relu%d" % cin, B=1, H=30, W=38, srcs=((cin, 0),), Cout=64, counts=(40,), residual=(0, 0) if residual else None,
                   seed=cin)
    case = _narrow_case(spec, dtype, dev)
    init = case.dst.clone()
    written = TC.reference(case)[0].written
    _launch(case, 0, TC.TC5)
    plain = case.dst.clone()
    relu_spec = dataclasses.replace(spec, dst=None)
    rcase = TC.Case(relu_spec, dtype, case.srcs, case.idx, None, None, case.w, case.bias, None, case.residual,
                    [TC.Aux(init.clone(), 0, None, None, ACT_RELU)])
    rcase.wp = case.wp
    _launch(rcase, 0, TC.TC5)
    got = rcase.aux[0].buf
    assert torch.equal(got[~written], init[~written])
    assert torch.equal(got[written], plain[written].clamp_min(0))


# ---------------------------------------------------------------------------------------------------------------- fused steps (GPU)
@pytest.mark.gpu
def test_sub_mobile_miniature_fused_fp16_runs_every_sparse_conv_fused():
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
    assert not [n for n in step.eager_nodes if n in ("sige.conv", "sige.gather", "sige.scatter_gather", "sige.scatter_block_residual")]
    assert sum(1 for f in step.fused if f.spec.epilogue_act == "relu") == 4
    assert any(f.spec.Cin % 64 for f in step.fused)
    ref = via_modules.float().cpu().numpy()
    G_ = TS._golden_or_none()
    if G_ is not None:
        ref = G_["sparse1"]
    e = np.abs(fused.float().cpu().numpy() - ref).max() / np.abs(ref).max()
    print("sub-mobile mini with narrow launches: fused fp16 vs %s %.3g" % ("golden" if G_ is not None else "fp32 operator modules", e))
    assert e <= 1e-2
    a = step.replay().clone()
    b = step.replay().clone()
    assert torch.equal(a, b), "graph replay must be idempotent"


def _narrow_model():
    """Gather -> 40-channel 3x3 conv -> ReLU -> ScatterGather -> 48-channel 3x3 conv -> Scatter: two narrow launches, the first
    with the ReLU epilogue, on one tile set."""
    from sige.nn import Gather, Scatter, ScatterGather, SIGEConv2d, SIGEModel
    from sige_b200.workloads.ddpm import init_deterministic

    class Narrow(SIGEModel):
        def __init__(self):
            super().__init__()
            self.conv0 = SIGEConv2d(40, 48, 3, padding=1)
            self.conv1 = SIGEConv2d(48, 24, 3, padding=1)
            self.gather = Gather(self.conv0, 6)
            self.scatter_gather = ScatterGather(self.gather)
            self.scatter = Scatter(self.gather)

        def forward(self, x):
            h = torch.relu(self.conv0(self.gather(x)))
            return self.scatter(self.conv1(self.scatter_gather(h)), None)

    return init_deterministic(Narrow(), seed=4).eval()


@pytest.mark.gpu
def test_next_edit_reuses_the_compiled_narrow_step():
    """The narrow launches read the same fixed-capacity tile lists as the others: `rebind` and `set_masks_async` install a second
    edit without re-tracing and equal a fresh compile bitwise."""
    from sige.utils import downsample_mask

    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(2)
    net = _narrow_model().to(dev).half()
    x0 = torch.randn(1, 40, 32, 48, generator=gen).to(dev).half()
    edit = torch.randn(1, 40, 32, 48, generator=gen).to(dev).half()

    def edited(mask):
        return x0 + edit * mask.to(dev).half()

    mask_a = torch.zeros(32, 48, dtype=torch.bool)
    mask_a[4:14, 6:20] = True
    mask_b = torch.zeros(32, 48, dtype=torch.bool)
    mask_b[18:27, 30:41] = True
    with torch.no_grad():
        net.set_mode("full")
        net(x0)
        net.set_mode("sparse")
        net.set_fused(True, headroom=0.5)
        net.set_masks(downsample_mask(mask_a.to(dev), min_res=(4, 4), dilation=1))
        out_a = net(edited(mask_a))
        step = net.fused_step
        assert not any(n.startswith("sige.") or n == "relu" for n in step.eager_nodes), step.eager_nodes
        assert [f.spec.epilogue_act for f in step.fused] == ["relu", "identity"] and [f.spec.Cin for f in step.fused] == [40, 48]
        pyr_b = downsample_mask(mask_b.to(dev), min_res=(4, 4), dilation=1)
        net.set_masks(pyr_b)
        out_b = net(edited(mask_b))
        assert net.fused_step is step
        assert net.set_masks_async(downsample_mask(mask_a.to(dev), min_res=(4, 4), dilation=1)) is True
        out_a_async = net(edited(mask_a))
        assert net.fused_step is step and net.masks_async_ok()
        net.set_fused(True, headroom=0.5)
        net.set_masks(pyr_b)
        fresh_b = net(edited(mask_b))
        assert net.fused_step is not step
        net.set_masks(downsample_mask(mask_a.to(dev), min_res=(4, 4), dilation=1))
        fresh_a = net(edited(mask_a))
        net.set_fused(False)
        net.set_masks(pyr_b)
        want_b = net(edited(mask_b))
    assert torch.equal(out_b, fresh_b) and torch.equal(out_a_async, fresh_a) and torch.equal(out_a, fresh_a)
    assert float((out_b.float() - want_b.float()).abs().max() / want_b.float().abs().max()) <= 1e-2
