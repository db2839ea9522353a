"""wgmma tile-conv launches with early source groups (SIGE_CONV_EARLY_SRC0 / _SRC1 / _SHORTCUT) against the float64 restatement of their descriptor
(tests/tile_conv_contract.py): every case of tcc.CASES that has a second source or a fused shortcut, under every mask of those
groups, at every ksplit the case lists — within the per-element bound, every other element bitwise unchanged, with and without
programmatic dependent launch (and with SIGE_CONV_EARLY_RELEASE) bitwise identical, and both halo layouts bitwise identical.
The halo fills each rank's CTAs record (trace slot 12) are those of the restated K partition (tests/test_early_chunks.py)."""
import pytest
import torch

import tile_conv_contract as tcc
from test_early_chunks import halo_fills

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EARLY_RELEASE = 8
CASES = [s for s in tcc.CASES if (len(s.srcs) == 2 or s.shortcut) and s.stride == 1]


def _run(case, init, d):
    from sige_b200 import ops

    for name, buf in case.buffers().items():
        buf.copy_(init[name])
    ops.launch_tile_conv(d, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return {name: buf.clone() for name, buf in case.buffers().items()}


def _same(a, b):
    return all(torch.equal(a[k].view(torch.int16), b[k].view(torch.int16)) for k in a)


def _traced_fills(case, init, d, plan):
    """Most halo fills recorded by any CTA of each K rank (trace slot 12)."""
    from sige_b200 import _cabi

    n = plan.grid_x * plan.grid_y * plan.grid_z
    buf = torch.zeros(n * 16, dtype=torch.int64, device=DEV)
    _cabi.check(_cabi.lib().sige_debug_set_trace(buf.data_ptr()), "sige_debug_set_trace")
    try:
        _run(case, init, d)
    finally:
        _cabi.lib().sige_debug_set_trace(None)
    return [int(v) for v in buf.view(plan.grid_z, -1, 16)[:, :, 12].max(dim=1).values]


def _set_halo(n):
    from sige_b200 import _cabi

    _cabi.check(_cabi.lib().sige_debug_set_split_halo_buffers(n), "sige_debug_set_split_halo_buffers")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("spec", CASES, ids=lambda s: s.name)
def test_masked_launch_matches_the_float64_contract(spec, dtype):
    case = tcc.make_case(spec, dtype, DEV)
    expects = tcc.reference(case)
    init = {name: buf.clone() for name, buf in case.buffers().items()}
    padded = tcc.PADDED if spec.padded else 0
    groups = [g for g in range(3) if (g < len(spec.srcs)) or (g == 2 and spec.shortcut)]
    allowed = sum(1 << g for g in groups)
    masks = [m for m in range(1, 8) if m & ~allowed == 0]
    record = []
    for ks in spec.ksplits:
        for early in masks:
            d = tcc.descriptor(case, ks, tcc.TC5 | padded)
            d.flags = tcc.TC5 | padded | (early << 4)
            plan = tcc.plan_of(d)
            assert plan.path == 1
            label = "%s %s ksplit %d early %d -> %s" % (spec.name, tcc.DTYPE_NAME[dtype], ks, early, tcc.plan_str(plan))
            first = None
            for flags in (0, tcc.PDL, tcc.PDL | EARLY_RELEASE):
                flags |= tcc.TC5 | padded | (early << 4)
                d.flags = flags
                got = _run(case, init, d)
                if first is None:
                    first = got
                    record.append((label, tcc.check(label, expects, got, init)))
                else:
                    assert _same(got, first), "%s: flags %d changed the result" % (label, flags)
            if plan.deep_ring:
                d.flags = tcc.TC5 | padded | tcc.PDL | (early << 4)
                cin2 = sum(spec.shortcut) if spec.shortcut else 0
                assert _traced_fills(case, init, d, plan) == halo_fills(sum(c for c, _ in spec.srcs), spec.srcs[0][0], cin2, early,
                                                                        plan.ksplit), label
                try:
                    for n in (1, 2):
                        _set_halo(n)
                        assert _same(_run(case, init, d), first), "%s: halo layout x%d differs" % (label, n)
                finally:
                    _set_halo(0)
    for label, (r, x) in record:
        print("[early-chunk contract] %-64s worst |err| / bound %.3f, beyond rounding %.3f" % (label, r, x))
