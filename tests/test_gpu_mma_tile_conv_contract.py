"""Every configuration and geometry of the mma.sync tile conv against the float64 restatement of its descriptor
(tests/mma_tile_conv_contract.py).

For each case of mc.CASES (those whose descriptor sets a source window or a modulation in a test of their own), in fp16 and bf16,
at every ksplit the case lists:
  * the plan the library reports on this device equals the restated heuristic's (configuration, tiles per CTA, K split, grid) and is
    the configuration the case is meant for — a mismatch fails: the case would test something else;
  * the launch, with and without programmatic dependent launch, is within the per-element bound on every element it writes, and
    leaves every other element of every writable buffer — guard bands included — and every input bitwise unchanged;
  * a second launch is bitwise identical; so is the launch without SIGE_CONV_PADDED (padded lists).
The worst error / bound ratios of every launch are printed (pytest -s) so the headroom on the device is on record.
"""
import pytest
import torch

import kernel_contracts as kc
import mma_tile_conv_contract as mc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _run(case, init, d):
    from sige_b200 import ops

    kc.restore(case.buffers(), init)
    ops.launch_tile_conv(d, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return kc.snapshot(case.buffers())


def _same(a, b):
    return all(torch.equal(kc.bits(a[k]), kc.bits(b[k])) for k in a)


PLAIN_CASES = [s for s in mc.CASES if not (s.mod or s.window)]
FIELD_CASES = [s for s in mc.CASES if s.mod or s.window]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("spec", PLAIN_CASES, ids=lambda s: s.name)
def test_mma_tile_conv_matches_the_float64_contract(spec, dtype):
    _sweep(spec, dtype)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("spec", FIELD_CASES, ids=lambda s: s.name)
def test_mma_tile_conv_window_and_modulation_fields_match_the_float64_contract(spec, dtype):
    """The cases whose descriptor sets src_pixel_stride or modulation."""
    _sweep(spec, dtype)


def _sweep(spec, dtype):
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    case = mc.make_case(spec, dtype, DEV)
    expects = mc.reference(case)
    init = kc.snapshot(case.buffers())
    inputs = case.inputs()
    inputs0 = {k: v.clone() for k, v in inputs.items()}
    padded = mc.PADDED if spec.padded else 0
    record = []
    for ks in spec.ksplits:
        d = mc.descriptor(case, ks, padded)
        want = spec.plan(ks, sms)
        got = mc.plan_of(d)
        label = "%s %s ksplit %d -> %s%s tpc %d grid %dx%dx%d" % ((spec.name, mc.DTYPE_NAME[dtype], ks, want.config, " MOD" if spec.mod else "",
                                                                  want.tpc) + want.grid)
        assert mc.plan_tuple(got) == mc.expected_plan_tuple(want), "%s: the library plans %s" % (label, mc.plan_tuple(got))
        assert want.config == spec.expect, "%s: the case is meant for %s (%d SMs)" % (label, spec.expect, sms)
        assert bool(spec.ambiguous(want, ks, sms)) == spec.single_cta, label
        first = None
        for pdl in (0, mc.PDL):
            d.flags = padded | pdl
            out = _run(case, init, d)
            name = label + (" pdl" if pdl else "")
            record.append((name, kc.check(name, expects, out, init, inputs, inputs0)))
            if first is None:
                first = out
            else:
                assert _same(out, first), "%s: programmatic dependent launch changed the result" % label
        d.flags = padded
        assert _same(_run(case, init, d), first), "%s: a second launch differs" % label
        if spec.padded:
            d.flags = 0
            assert _same(_run(case, init, d), first), "%s: the result depends on SIGE_CONV_PADDED" % label
    for name, (r, x) in record:
        print("[mma tile-conv contract] %-72s worst |err| / bound %.3f, beyond rounding %.3f" % (name, r, x))
