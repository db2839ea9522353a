"""Every wgmma tile-conv configuration against the float64 restatement of its descriptor (tests/tile_conv_contract.py).

For each case of tcc.CASES, in fp16 and bf16, at every ksplit the case lists:
  * the plan on this device is the intended kernel instantiation (a mismatch fails: the case would test something else);
  * the launch, with and without programmatic dependent launch, is within the per-element bound of tcc.check on every
    element it writes, and leaves every other element of every buffer bitwise unchanged;
  * a second launch is bitwise identical; so is the launch without SIGE_CONV_PADDED (padded lists);
  * split narrow 3x3 launches run in both halo layouts, each within the bound and bitwise equal to each other;
  * the mma.sync kernel (SIGE_CONV_TC5 cleared) meets the same bound, or refuses the fused shortcut.
The worst error / bound ratios of every launch are printed (pytest -s) so the headroom on the device is on record.
"""
import numpy as np
import pytest
import torch

import tile_conv_contract as tcc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _set_halo(n):
    from sige_b200 import _cabi

    _cabi.check(_cabi.lib().sige_debug_set_split_halo_buffers(n), "sige_debug_set_split_halo_buffers")


def _run(case, init, d):
    from sige_b200 import ops

    for name, buf in case.buffers().items():
        buf.copy_(init[name])
    ops.launch_tile_conv(d, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return {name: buf.clone() for name, buf in case.buffers().items()}


def _same(a, b):
    return all(torch.equal(a[k].view(torch.int16), b[k].view(torch.int16)) for k in a)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("spec", tcc.CASES, ids=lambda s: s.name)
def test_tile_conv_matches_the_float64_contract(spec, dtype):
    from sige_b200._cabi import SigeError

    case = tcc.make_case(spec, dtype, DEV)
    expects = tcc.reference(case)
    init = {name: buf.clone() for name, buf in case.buffers().items()}
    padded = tcc.PADDED if spec.padded else 0
    record = []
    for i, ks in enumerate(spec.ksplits):
        d = tcc.descriptor(case, ks, tcc.TC5 | padded)
        plan = tcc.plan_of(d)
        key, want_key = tcc.instantiation(spec, dtype, plan), tcc.intended(spec, dtype, i)
        label = "%s %s ksplit %d -> %s" % (spec.name, tcc.DTYPE_NAME[dtype], ks, tcc.plan_str(plan))
        assert key == want_key, "%s: runs %s, the case is meant for %s" % (label, key, want_key)
        first = None
        for pdl in (0, tcc.PDL):
            d.flags = tcc.TC5 | padded | pdl
            got = _run(case, init, d)
            record.append((label + (" pdl" if pdl else ""), tcc.check(label + (" pdl" if pdl else ""), expects, got, init)))
            if first is None:
                first = got
            else:
                assert _same(got, first), "%s: programmatic dependent launch changed the result" % label
        d.flags = tcc.TC5 | padded
        assert _same(_run(case, init, d), first), "%s: a second launch differs" % label
        if spec.padded:
            d.flags = tcc.TC5
            assert _same(_run(case, init, d), first), "%s: the result depends on SIGE_CONV_PADDED" % label
            d.flags = tcc.TC5 | padded
        if plan.deep_ring:
            layouts = {}
            try:
                for n in (1, 2):
                    _set_halo(n)
                    layouts[n] = _run(case, init, d)
                    record.append(("%s halo x%d" % (label, n), tcc.check("%s halo x%d" % (label, n), expects, layouts[n], init)))
            finally:
                _set_halo(0)
            assert _same(layouts[1], layouts[2]), "%s: the two halo layouts differ" % label
            assert _same(layouts[1], first)
        mlabel = "%s %s ksplit %d mma.sync" % (spec.name, tcc.DTYPE_NAME[dtype], ks)
        d.flags = padded
        if spec.shortcut:      # the mma.sync kernel does not implement the fused shortcut: a loud error, not a wrong result
            with pytest.raises(SigeError, match="wgmma"):
                _run(case, init, d)
        else:
            record.append((mlabel, tcc.check(mlabel, expects, _run(case, init, d), init)))
    for label, (r, x) in record:
        print("[tile-conv contract] %-58s worst |err| / bound %.3f, beyond rounding %.3f" % (label, r, x))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_stem_per_image_tiles_match_the_dense_stem(dtype):
    """sige_conv_in_nhwc_tiles with per-image lists padded by SIGE_TILE_NONE: bit-identical to the dense stem inside each
    image's own tiles (dst and aux), every other element bitwise unchanged — no tile writes into another image."""
    from sige_b200 import ops

    g = torch.Generator(device=DEV)
    g.manual_seed(5)
    B, Cin, Cout, H, W = 3, 3, 128, 38, 44          # (the dense stem needs W % 4 == 0; the tiles overhang both extents)
    cl = torch.channels_last
    x = torch.randn(B, Cin, H, W, device=DEV, generator=g).to(dtype).contiguous(memory_format=cl)
    w = (torch.randn(Cout, Cin, 3, 3, device=DEV, generator=g) / (Cin * 9) ** 0.5).to(dtype)
    b = torch.randn(Cout, device=DEV, generator=g).to(dtype)
    sc, sh = torch.rand(Cout, device=DEV, generator=g) + 0.5, torch.randn(Cout, device=DEV, generator=g)
    dense_aux = torch.empty(B, Cout, H, W, device=DEV, dtype=dtype).contiguous(memory_format=cl)
    dense = ops.conv_in_nhwc(x, w, b, aux=[ops.conv_aux(dense_aux, sc, sh, "swish")])
    rng = np.random.default_rng(5)
    hs, ws = [4 * i - 1 for i in range(-(-H // 4))], [4 * i - 1 for i in range(-(-W // 4))]
    grid = [(h, v) for h in hs for v in ws]
    counts = (40, 17, 3)
    n_max = max(counts) + 5                          # padding in every image's list, a whole run of it in the longest
    lists = []
    corners = [(hs[0], ws[0]), (hs[-1], ws[-1])]    # overhang the top-left and bottom-right borders
    rest = [t for t in grid if t not in corners]
    for n in counts:
        lists.append(sorted(corners + [rest[i] for i in rng.choice(len(rest), n - 2, replace=False)]))
    rows = []
    for tiles in lists:
        rows += tiles + [(tcc.TILE_NONE, tcc.TILE_NONE)] * (n_max - len(tiles))
    idx = torch.tensor(rows, dtype=torch.int32, device=DEV)
    out0 = torch.randn(B, Cout, H, W, device=DEV, generator=g).to(dtype).contiguous(memory_format=cl)
    aux0 = torch.randn(B, Cout, H, W, device=DEV, generator=g).to(dtype).contiguous(memory_format=cl)
    out, aux = out0.clone(memory_format=cl), aux0.clone(memory_format=cl)
    ops.conv_in_nhwc(x, w, b, out=out, aux=[ops.conv_aux(aux, sc, sh, "swish")], tiles=idx, tile_size=6, tiles_per_image=True)
    torch.cuda.synchronize()
    inside = torch.zeros(B, H, W, dtype=torch.bool, device=DEV)
    for bi, tiles in enumerate(lists):
        for (y0, x0) in tiles:
            inside[bi, max(y0, 0):max(min(y0 + 6, H), 0), max(x0, 0):max(min(x0 + 6, W), 0)] = True
    assert bool(inside.any(dim=(1, 2)).all()) and not bool(inside.all())

    def nhwc(t):
        return t.permute(0, 2, 3, 1)

    for got, want, before in ((out, dense, out0), (aux, dense_aux, aux0)):
        assert torch.equal(nhwc(got)[inside], nhwc(want)[inside])
        assert torch.equal(nhwc(got)[~inside].view(torch.int16), nhwc(before)[~inside].view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------- stack destination
STACK_CASES = [
    # a fixed-capacity list (real tiles, then SIGE_TILE_NONE padding) read from an image, written as a stack of tile rows:
    # the q conv of the SD decoder's attention (1x1 on 4x4 tiles, 512 -> 512) and a 3x3 conv on 6x6 tiles of two images
    tcc.Spec("stack_k1_c512", B=1, H=20, W=24, k=1, srcs=((512, 0),), Cout=512, counts=(13,), pad_to=24, seed=951),
    tcc.Spec("stack_k3_c64_128_b2", B=2, H=22, W=26, srcs=((64, 0),), Cout=128, counts=(11,), pad_to=16, seed=952),
]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("kernel", ["wgmma", "mma.sync"])
@pytest.mark.parametrize("spec", STACK_CASES, ids=lambda s: s.name)
def test_stack_destination_rows_of_padding_keep_their_contents(spec, kernel, dtype):
    """dst_is_stack with a padded list: the row of each real tile within the float64 bound of its conv, the row of each
    SIGE_TILE_NONE entry still holding its NaN sentinel bitwise (include/sige_b200.h: such a tile writes nothing)."""
    import torch.nn.functional as F

    from sige_b200 import ops

    case = tcc.make_case(spec, dtype, DEV)
    B, N, Ro, Cout = spec.B, spec.N, spec.Ro, spec.Cout
    stack = torch.full((B * N, Ro, Ro, Cout), float("nan"), dtype=dtype, device=DEV)
    d = tcc.descriptor(case, flags=tcc.TC5 if kernel == "wgmma" else 0)
    d.dst, d.dst_is_stack, d.dH, d.dW, d.dC, d.dst_c0 = stack.data_ptr(), 1, Ro, Ro, Cout, 0
    assert (tcc.plan_of(d).path == 1) == (kernel == "wgmma"), kernel
    ops.launch_tile_conv(d, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()

    t = torch.arange(B * N, device=DEV)
    org = case.idx.long()[t % N]
    none = org[:, 0] == tcc.TILE_NONE
    assert bool(none.any()) and not bool(none.all())
    a, valid = tcc._gather([(case.srcs[0], 0)], torch.where(none[:, None], torch.zeros_like(org), org), t // N, spec.R, spec.H, spec.W)
    a = torch.where(valid[..., None], a, torch.zeros((), dtype=a.dtype, device=DEV)).permute(0, 3, 1, 2)
    w, b = case.w.double(), case.bias.double()
    v = F.conv2d(a, w, b).permute(0, 2, 3, 1)
    mag = F.conv2d(a.abs(), w.abs(), b.abs()).permute(0, 2, 3, 1)
    bound = tcc.UNIT_ROUNDOFF[dtype] * v.abs() + tcc.ACC * mag + tcc.ABS
    got = stack.double()
    ratio = ((got[~none] - v[~none]).abs() / bound[~none]).nan_to_num(nan=float("inf"))
    assert float(ratio.max()) <= 1.0, "%s %s: a real tile's row off by %.3g of its bound" % (spec.name, kernel, float(ratio.max()))
    pad = stack[none].view(torch.int16)
    assert torch.equal(pad, torch.full_like(stack[none], float("nan")).view(torch.int16)), "%s %s: a padding row was written" % (spec.name, kernel)
    print("[tile conv contract] stack destination %s %s %s: %d real rows worst |err| / bound %.3f, %d padding rows untouched"
          % (spec.name, kernel, tcc.DTYPE_NAME[dtype], int((~none).sum()), float(ratio.max()),
             int(none.sum())))
