"""sige_tile_conv at the largest extents its ABI accepts, against the float64 restatement of the launch
(tests/extent_contract.py, tests/mma_tile_conv_contract.py).

Images of 65535 (or 65534, where a source is read up-sampled) rows by 16 columns, and the transpose, with tiles across row /
column 32768 and against the last row / column.  Every geometry and gather variant runs on both kernels, the mma.sync kernel
(no SIGE_CONV_TC5) and the wgmma kernel, and for each launch:
  * sige_tile_conv_plan names the kernel the case is meant for;
  * every element it writes is within the contract's bound, every other element of every writable buffer (guard bands
    included) and every input is bitwise unchanged;
  * a second launch is bitwise identical.
"""
import pytest
import torch

import extent_contract as ec
import kernel_contracts as kc
import mma_tile_conv_contract as mc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MAX_PEAK = 10 * ec.GiB

# written for a tall image; extent_contract.spec_at_edge sets the extents (and turns it wide)
BASES = [
    # destination and residual are the last 64 of 128 channels
    mc.Spec("3x3", B=1, srcs=((64, 0),), Cout=64, counts=(1,), R=6, dst=(64, 64), residual=(64, 64), seed=301),
    mc.Spec("1x1", B=1, srcs=((64, 0),), Cout=64, counts=(1,), R=4, k=(1, 1), seed=302),
    mc.Spec("3x3_s2", B=1, srcs=((64, 0),), Cout=64, counts=(1,), R=5, stride=2, seed=303),
    mc.Spec("shared_preop", B=1, srcs=((64, 0),), Cout=64, counts=(1,), R=6, preop="shared", act=1, seed=304),
    mc.Spec("per_sample_preop", B=2, srcs=((64, 0),), Cout=64, counts=(1,), R=6, preop="per_sample", act=1, seed=305),
    mc.Spec("modulated", B=1, srcs=((64, 0),), Cout=64, counts=(1,), R=6, preop="shared", mod=(8, 8, 0, 0, 0.2), seed=306),
    mc.Spec("upsampled_second", B=1, srcs=((64, 0), (64, 1)), Cout=64, counts=(1,), R=6, seed=307),
]
KERNELS = ("mma", "wgmma")


def _run(case, init, d):
    from sige_b200 import ops

    kc.restore(case.buffers(), init)
    ops.launch_tile_conv(d, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return kc.snapshot(case.buffers())


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("tall", [True, False], ids=["tall", "wide"])
@pytest.mark.parametrize("base", BASES, ids=lambda s: s.name)
def test_tile_conv_at_the_extent_limit(base, tall, kernel, dtype):
    spec = ec.spec_at_edge(base, tall)
    peak = ec.peak_bytes(spec, dtype)
    assert peak <= MAX_PEAK, "%s: %.1f GiB" % (spec.name, peak / ec.GiB)
    ec.need(peak, DEV)
    from sige_b200 import _cabi

    flags, path = (_cabi.CONV_TC5, 1) if kernel == "wgmma" else (0, 0)
    case = ec.make_edge_case(spec, tall, dtype, DEV)
    expects = mc.reference(case)
    init = kc.snapshot(case.buffers())
    inputs = case.inputs()
    inputs0 = {k: v.clone() for k, v in inputs.items()}
    d = mc.descriptor(case, 0, flags)
    label = "%s %s %s (%d x %d, %d tiles)" % (spec.name, kernel, mc.DTYPE_NAME[dtype], spec.H, spec.W, case.idx.shape[0])
    assert mc.plan_of(d).path == path, "%s: planned on the other kernel" % label
    first = _run(case, init, d)
    r = kc.check(label, expects, first, init, inputs, inputs0)
    assert all(torch.equal(kc.bits(a), kc.bits(b)) for a, b in zip(_run(case, init, d).values(), first.values())), \
        "%s: a second launch differs" % label
    print("[extent contract] %-56s worst |err| / bound %.3f, beyond rounding %.3f" % (label, r[0], r[1]))
    del case, expects, init, inputs, inputs0, first
    torch.cuda.empty_cache()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("bs", ec.BIG_CASES, ids=lambda s: s.name)
def test_tile_conv_on_a_buffer_of_2_to_the_31_elements(bs, dtype):
    """Source window, destination, residual and aux destination in one buffer of 2^31 elements (mma.sync) or 2048 fewer
    (wgmma, reading up to the buffer's last element)."""
    es = torch.empty((), dtype=dtype).element_size()
    peak = bs.elements * es + 2 * ec.CHUNK * 8
    assert peak <= MAX_PEAK
    ec.need(peak, DEV)
    from sige_b200 import ops

    bc = ec.make_big_case(bs, dtype, DEV)
    d = ec.big_descriptor(bc)
    label = "%s %s (%d elements, %d tiles)" % (bs.name, mc.DTYPE_NAME[dtype], bs.elements, bc.case.idx.shape[0])
    assert mc.plan_of(d).path == bs.path, "%s: planned on the other kernel" % label
    idx, want, bound = ec.big_reference(bc)
    stream = torch.cuda.current_stream().cuda_stream
    ops.launch_tile_conv(d, stream)
    torch.cuda.synchronize()
    r = ec.big_check(label, bc, idx, want, bound)
    first = bc.flat[idx].clone()
    ops.launch_tile_conv(d, stream)
    torch.cuda.synchronize()
    assert torch.equal(kc.bits(bc.flat[idx]), kc.bits(first)), "%s: a second launch differs" % label
    ec.big_check(label + " (second launch)", bc, idx, want, bound)
    print("[extent contract] %-56s worst |err| / bound %.3f" % (label, r))
    del bc, d, idx, want, bound, first
    torch.cuda.empty_cache()
