"""sige_tile_conv_generic (the CUDA-core tile conv) against the float64 restatement of its C-ABI contract
(tests/generic_conv_contract.py).

Every launch must be within the rigorous per-element bound on every output element, leave the guard bands around the output and
every input bitwise unchanged, and be bitwise equal on a repeat.  The kernels' fixed summation order (fmaf over the products of
an output from 0, then the bias) makes more hold bitwise: NCHW and NHWC give the same bits, the three depthwise forms give the
same bits, and a channel-multiplier conv equals the depthwise conv on the channels that share its weights.  A CUDA-graph replay
equals the stream launch, and SIGEConv2d in sparse mode returns what the C-ABI call returns.  The worst error / bound ratio of
each launch is printed (pytest -s).
"""
from dataclasses import replace

import pytest
import torch

import generic_conv_contract as gc
import kernel_contracts as kc
from kernel_contracts import _launch, _run_and_check

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NAME = {torch.float32: "f32", torch.float16: "f16", torch.bfloat16: "bf16"}
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT = pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "bf16"])


def _lib():
    from sige_b200 import _cabi

    return _cabi.lib()


def _sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def _out(case: gc.GenCase, flat: torch.Tensor) -> torch.Tensor:
    """The output window of a flat buffer, logical NCHW."""
    g = case.out
    return case.logical(flat[g.off:g.off + g.view.numel()].view(*g.view.shape))


def _run(case: gc.GenCase, lib) -> torch.Tensor:
    return _out(case, _launch(case, kc.snapshot(case.buffers()), lambda: gc.gen_call(case, lib))["out"])


def _label(spec: gc.GenSpec, dtype, misalign: bool) -> str:
    path = gc.generic_path(spec, dtype, misalign)
    if path.startswith("dw"):
        path += ", %d trips" % gc.dw_trips(spec, dtype, misalign, _sms())
    return "%s %s (%s)" % (spec.name, NAME[dtype], path)


# ---------------------------------------------------------------------------------------------------------------- contract
@DT
@pytest.mark.parametrize("spec", gc.GEN_CASES, ids=lambda s: s.name)
def test_generic_conv_matches_the_float64_contract(spec, dtype):
    case = gc.make_gen(spec, dtype, DEV)
    path = gc.generic_path(spec, dtype, spec.misalign)
    ptrs = (case.x.view.data_ptr(), case.out.view.data_ptr())
    if spec.depthwise and spec.layout == "nhwc":
        # the launcher's own predicate (tile_conv_simt.cu launch_depthwise) on the pointers it is given
        assert (path == "dw_vec") == (spec.Cin % gc.VEC[dtype] == 0 and all(p % 16 == 0 for p in ptrs)), spec.name
    expects = gc.gen_reference(case)
    lib = _lib()
    _run_and_check("generic", _label(spec, dtype, spec.misalign), case, expects, lambda flags: gc.gen_call(case, lib))


@DT
@pytest.mark.parametrize("path", gc.PATHS)
def test_the_launcher_runs_the_predicted_kernel(path, dtype):
    """One case of each path, profiled: the depthwise paths run tile_conv_depthwise_kernel, the others tile_conv_simt_kernel,
    both instantiated for the launch dtype."""
    from torch.profiler import ProfilerActivity, profile

    spec = next(s for s in gc.GEN_CASES if gc.generic_path(s, dtype, s.misalign) == path and gc.gen_cost(s) < 10 ** 7)
    case = gc.make_gen(spec, dtype, DEV)
    lib = _lib()
    assert gc.gen_call(case, lib) == 0                                                    # warm: the attribute set, the module loaded
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        assert gc.gen_call(case, lib) == 0
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if "tile_conv_" in e.name}
    kern = "tile_conv_depthwise_kernel" if path.startswith("dw") else "tile_conv_simt_kernel"
    tname = {torch.float32: "float", torch.float16: "__half", torch.bfloat16: "__nv_bfloat16"}[dtype]
    assert len(names) == 1 and "%s<%s>" % (kern, tname) in next(iter(names)), (path, names)


# ---------------------------------------------------------------------------------------------------------------- bitwise
@DT
@pytest.mark.parametrize("spec", [s for s in gc.GEN_CASES if not s.depthwise and gc.gen_cost(s) < 10 ** 7], ids=lambda s: s.name)
def test_layout_does_not_change_the_bits(spec, dtype):
    """The halo chunk is staged into the same shared-memory layout from NCHW and from NHWC (tile_conv_simt.cu): the same
    products in the same order, so the same bits."""
    lib = _lib()
    a, b = (_run(gc.make_gen(spec, dtype, DEV, layout=lay), lib) for lay in ("nchw", "nhwc"))
    assert torch.equal(kc.bits(a), kc.bits(b)), "%s %s: NCHW and NHWC differ" % (spec.name, NAME[dtype])


@DT
@pytest.mark.parametrize("spec", [s for s in gc.GEN_CASES if s.depthwise and gc.gen_cost(s) < 10 ** 7], ids=lambda s: s.name)
def test_depthwise_forms_give_the_same_bits(spec, dtype):
    """NCHW, NHWC with 16-byte vectors and NHWC scalar all compute fmaf over (ky, kx) from 0, then add the bias."""
    lib = _lib()
    outs = {}
    for lay, mis in (("nchw", False), ("nhwc", False), ("nhwc", True)):
        s = replace(spec, layout=lay, misalign=mis)
        outs[gc.generic_path(s, dtype, mis)] = _run(gc.make_gen(s, dtype, DEV), lib)
    assert {"dw_nchw", "dw_nhwc_scalar"} <= set(outs) and (spec.Cin % gc.VEC[dtype] or "dw_vec" in outs)
    ref = outs["dw_nchw"]
    for path, o in outs.items():
        assert torch.equal(kc.bits(o), kc.bits(ref)), "%s %s: %s differs from dw_nchw" % (spec.name, NAME[dtype], path)


@DT
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
def test_channel_multiplier_equals_depthwise_on_shared_weights(layout, dtype):
    """groups = Cin = 16, Cout = 32 runs the generic kernel; with w'[2c] = w[c] and b'[2c] = b[c] its channel 2c computes the same
    fmaf chain as channel c of the depthwise kernel, so the bits agree."""
    lib = _lib()
    dws = gc.GenSpec("dw_c16", 6, 16, 16, 6, 6, groups=16, layout=layout, seed=60)
    mul = gc.GenSpec("mult_c16_cout32", 6, 16, 32, 6, 6, groups=16, layout=layout, seed=61)
    assert gc.generic_path(dws, dtype, False).startswith("dw") and gc.generic_path(mul, dtype, False) == "simt"
    d, m = gc.make_gen(dws, dtype, DEV), gc.make_gen(mul, dtype, DEV)
    m.x.view.copy_(d.x.view)
    m.w.view[0::2] = d.w.view
    m.b.view[0::2] = d.b.view
    got_d, got_m = _run(d, lib), _run(m, lib)
    assert torch.equal(kc.bits(got_m[:, 0::2]), kc.bits(got_d)), "multiplier channel 2c differs from depthwise channel c"


# ---------------------------------------------------------------------------------------------------------------- CUDA graphs
@DT
def test_graph_replay_matches_the_stream_launch(dtype):
    lib = _lib()
    for name in ("k7_r12", "g2_cig20_cog70", "dw_c128_nhwc", "dw_c64_nhwc_dil2_r8_misaligned", "dw_c96_nchw"):
        spec = next(s for s in gc.GEN_CASES if s.name == name)
        case = gc.make_gen(spec, dtype, DEV)
        kc.graph_equals_stream(case, lambda: gc.gen_call(case, lib))


# ---------------------------------------------------------------------------------------------------------------- SIGEConv2d
def _module_inputs():
    """(label, module dtype, stack dtype, conv kwargs, stack maker) for every input form SIGEConv2d hands to ops.tile_conv_generic."""
    def nchw(t):
        return t.contiguous()

    def cl(t):
        return t.contiguous(memory_format=torch.channels_last)

    def strided(t):                      # a window of a larger stack: dense in neither layout
        big = torch.zeros(t.shape[0], t.shape[1] + 3, t.shape[2] + 2, t.shape[3] + 1, dtype=t.dtype, device=t.device)
        big[:, 2:2 + t.shape[1], 1:1 + t.shape[2], :t.shape[3]] = t
        return big[:, 2:2 + t.shape[1], 1:1 + t.shape[2], :t.shape[3]]

    f32, f16, bf16 = torch.float32, torch.float16, torch.bfloat16
    conv = dict(in_channels=12, out_channels=20, kernel_size=3)
    grouped = dict(in_channels=16, out_channels=24, kernel_size=3, groups=2)
    return [
        ("f32_nchw", f32, f32, conv, nchw),
        ("f32_channels_last", f32, f32, conv, cl),
        ("f32_strided", f32, f32, conv, strided),
        ("f32_depthwise_channels_last", f32, f32, dict(in_channels=16, out_channels=16, kernel_size=3, groups=16), cl),
        ("f32_rect_stride_dilation", f32, f32, dict(in_channels=8, out_channels=8, kernel_size=(3, 1), stride=(1, 2), dilation=(2, 1)), nchw),
        ("f16_grouped_nchw", f16, f16, grouped, nchw),
        ("bf16_dilated_channels_last", bf16, bf16, dict(in_channels=64, out_channels=64, kernel_size=3, dilation=2), cl),
        ("f16_depthwise_strided", f16, f16, dict(in_channels=32, out_channels=32, kernel_size=3, groups=32), strided),
        ("f16_stack_f32_weights_grouped", f32, f16, grouped, cl),
        ("bf16_stack_f32_weights_depthwise", f32, bf16, dict(in_channels=24, out_channels=24, kernel_size=3, groups=24), nchw),
    ]


@pytest.mark.parametrize("inp", _module_inputs(), ids=lambda v: v[0])
def test_sige_conv2d_returns_what_the_cabi_call_returns(inp, monkeypatch):
    """SIGEConv2d's sparse forward on a stack that reaches ops.tile_conv_generic: bitwise the C-ABI call on the same operands (the
    stack made dense in its own layout, or NCHW; the weights and bias cast to the stack's dtype), in the stack's layout."""
    from sige_b200 import _cabi, ops
    from sige_b200.nn import SIGEConv2d

    label, mdt, xdt, kw, form = inp
    torch.manual_seed(7)
    conv = SIGEConv2d(**kw).to(DEV).to(mdt)
    conv.set_mode("sparse")
    x = form(torch.randn(5, kw["in_channels"], 8, 9, device=DEV).to(xdt))
    calls = []
    real = ops.tile_conv_generic
    monkeypatch.setattr(ops, "tile_conv_generic", lambda *a, **k: calls.append(a) or real(*a, **k))
    with torch.no_grad():
        got = conv(x)
    torch.cuda.synchronize()
    assert len(calls) == 1, "%s: the stack did not reach ops.tile_conv_generic" % label
    lay = ops.layout_of(x)
    xd = x if lay >= 0 else x.contiguous()
    lay = max(lay, 0)
    w = conv.weight.detach().to(xdt).contiguous()
    b = conv.bias.detach().to(xdt).contiguous()
    M, Cin, R, S = xd.shape
    Cout, _, kH, kW = w.shape
    (sH, sW), (dH, dW) = conv.stride, conv.dilation
    Ro, So = (R - dH * (kH - 1) - 1) // sH + 1, (S - dW * (kW - 1) - 1) // sW + 1
    want = torch.empty((M, Cout, Ro, So), dtype=xdt, device=DEV,
                       memory_format=torch.channels_last if lay == _cabi.NHWC else torch.contiguous_format)
    rc = _cabi.lib().sige_tile_conv_generic(xd.data_ptr(), w.data_ptr(), b.data_ptr(), want.data_ptr(), ops._dt(xd), lay, M, Cin, R, S,
                                            Cout, kH, kW, sH, sW, dH, dW, conv.groups, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert rc == 0, _cabi.last_error()
    assert got.dtype == xdt and got.shape == want.shape and ops.layout_of(got) == lay, label
    assert torch.equal(kc.bits(got.contiguous()), kc.bits(want.contiguous())), "%s: SIGEConv2d differs from the C-ABI call" % label
