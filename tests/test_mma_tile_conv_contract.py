"""CPU checks of the mma.sync tile-conv contract (tests/mma_tile_conv_contract.py), no GPU needed:

  * the float64 restatement agrees with the C oracle's gather -> conv2d_tiles -> scatter composite (fp32 arithmetic, so to 1e-6)
    on non-square tiles and kernels, stride 2 with a negative origin, channel windows and Cout 72, and with plain F.conv2d in
    float64 on stacks (to 1e-12);
  * the Python restatement of the launch plan equals sige_tile_conv_plan on random descriptors, modulated or not (without a device
    the library plans for 132 SMs), hand-worked points of every branch included;
  * the GPU sweep's case table reaches all 12 instantiations (f16 / bf16 x L / M / S x plain / MOD) and every required feature,
    and no case that claims a configuration could be mistaken for another from the plan's (bn, grid);
  * launches the kernel cannot run are refused before anything is launched, each with its own message;
  * `check` bites: a result computed from the contract fails against three deliberately wrong expectations.
"""
import ctypes
import dataclasses

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import kernel_contracts as kc
import mma_tile_conv_contract as mc

ORACLE_CASES = [
    mc.Spec("tile_6x10", B=2, H=24, W=40, srcs=((16, 0),), Cout=72, counts=(13,), R=6, S=10, preop="shared", act=1, residual=(8, 8),
            dst=(8, 0), seed=201),
    mc.Spec("kernel_1x3", B=1, H=16, W=24, srcs=((8, 0), (8, 1)), Cout=8, counts=(9,), R=4, S=8, k=(1, 3), seed=202),
    mc.Spec("kernel_3x2_off_1_0", B=1, H=20, W=20, srcs=((16, 0),), Cout=16, counts=(12,), R=6, S=5, k=(3, 2), off=(1, 0), seed=203),
    mc.Spec("stride2_7x7_negative_origin", B=1, H=36, W=30, srcs=((16, 0),), Cout=16, counts=(14,), R=7, stride=2, c_div_tile=True,
            residual=(0, 0), preop="shared", seed=204),
    mc.Spec("stride2_5x5", B=2, H=30, W=30, srcs=((16, 0),), Cout=16, counts=(19,), R=5, stride=2, dHW=(15, 15), c_div_tile=True, seed=205),
    mc.Spec("tile_5x5_no_bias", B=1, H=25, W=25, srcs=((16, 0),), Cout=16, counts=(18,), R=5, bias=False, seed=206),
]
# (No SIGE_TILE_NONE padding and no origin left of or above (-offH, -offW) - 1 here: the oracle's scatter, like the reference's,
# only clips at the bottom and right.  The restatement's own handling of padding is exercised by test_case_is_well_formed.)
STACK_CASES = [
    mc.Spec("stack_stack", B=1, srcs=((16, 0),), Cout=24, counts=(5,), R=7, src_stack=True, dst_stack=True, seed=211),
    mc.Spec("stack_stack_s2_3x1", B=1, srcs=((8, 0),), Cout=8, counts=(4,), R=7, S=5, k=(3, 1), stride=2, src_stack=True, dst_stack=True, seed=212),
]


def _nchw(t):
    return np.ascontiguousarray(t.permute(0, 3, 1, 2).float().numpy())


@pytest.mark.parametrize("spec", ORACLE_CASES, ids=lambda s: s.name)
def test_reference_matches_oracle(oracle, spec):
    case = mc.make_case(spec, torch.float32, "cpu")
    (e,) = mc.reference(case)
    s = spec
    x = np.concatenate([_nchw(t).repeat(1 << up, 2).repeat(1 << up, 3) for t, (_, up) in zip(case.srcs, s.srcs)], 1)
    idx = case.idx.numpy()
    sc = sh = None
    if s.preop:
        sc, sh = case.scale.numpy().reshape(1, -1, 1, 1), case.shift.numpy().reshape(1, -1, 1, 1)
    g = oracle.gather(x, s.R, s.Sx, idx, sc, sh, "swish" if s.act == 1 else "identity", False)
    tiles = oracle.conv2d_tiles(g, case.w.numpy(), None if case.bias is None else case.bias.numpy(), (s.stride, s.stride))
    c0 = s.dst[1]
    y0 = _nchw(case.dst.view)[:, c0:c0 + s.Cout]
    res = None if case.residual is None else _nchw(case.residual)[:, s.residual[1]:s.residual[1] + s.Cout]
    want = oracle.scatter(tiles, y0, s.offs[0], s.offs[1], s.stride, s.stride, idx, res)
    n = case.dst.view.numel()
    got = e.want[case.dst.off:case.dst.off + n].view(*case.dst.view.shape)
    written = e.written[case.dst.off:case.dst.off + n].view(*case.dst.view.shape)
    assert float(np.abs(_nchw(got)[:, c0:c0 + s.Cout] - want).max()) <= 1e-6 * float(np.abs(want).max())
    # the written set is exactly what the oracle changed, all of it inside the channel window
    assert np.array_equal(want != y0, written.permute(0, 3, 1, 2).numpy()[:, c0:c0 + s.Cout])
    assert int(written.sum()) == int(written[..., c0:c0 + s.Cout].sum()) == int(e.written.sum())
    if s.c_div_tile:        # the (-1, -1) tile writes outputs from (0, 0): C division of the origin
        assert bool(written[0, :s.Ro, :s.So, c0:c0 + s.Cout].all())


@pytest.mark.parametrize("spec", STACK_CASES, ids=lambda s: s.name)
def test_stack_reference_is_a_plain_convolution(spec):
    case = mc.make_case(spec, torch.float64, "cpu")
    (e,) = mc.reference(case)
    want = F.conv2d(case.srcs[0].permute(0, 3, 1, 2), case.w, case.bias.double(), stride=spec.stride).permute(0, 2, 3, 1)
    assert tuple(want.shape) == (spec.NT, spec.Ro, spec.So, spec.Cout)
    n = case.dst.view.numel()
    got = e.want[case.dst.off:case.dst.off + n].view(*case.dst.view.shape)
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())
    assert bool(e.written[case.dst.off:case.dst.off + n].all()) and int(e.written.sum()) == n      # every row written, no guard element


# ---------------------------------------------------------------------------------------------------------------- the plan
def _host_desc(NT=16, R=6, S=6, k=(3, 3), stride=1, cin=64, cout=64, ksplit=0, B=1, flags=0, modulated=False):
    """A descriptor whose pointers are not device memory: only argument checks and the plan may look at it."""
    from sige_b200 import _cabi

    d = _cabi.TileConv()
    d.dtype = _cabi.F16
    d.n_src, d.src[0].ptr, d.src[0].C = 1, 0x10000, cin
    d.B, d.H, d.W, d.idx, d.N = B, 64, 64, 0x20000, NT // B
    d.R, d.S = R, S
    d.w_packed, d.bias = 0x30000, 0x40000
    d.Cin, d.Cout, d.kH, d.kW, d.stride = cin, cout, k[0], k[1], stride
    d.dst, d.dH, d.dW, d.dC = 0x50000, 64, 64, cout
    d.ksplit, d.flags = ksplit, flags
    if modulated:
        d.modulation = ctypes.pointer(_cabi.ConvModulation())
    return d


def test_plan_branches_by_hand(cabi_lib):
    """One hand-worked point per branch of the selection at 132 SMs, the library and the restatement side by side."""
    def both(**kw):
        p = mc.plan(kw.get("NT", 16), kw.get("R", 6), kw.get("S", 6), *kw.get("k", (3, 3)), kw.get("stride", 1), kw.get("cin", 64),
                    kw.get("cout", 64), kw.get("ksplit", 0))
        assert mc.plan_tuple(mc.plan_of(_host_desc(**kw))) == mc.expected_plan_tuple(p), kw
        return p

    # 6x6 / 3x3: L packs 8 tiles, M 4, S 2.  2112 tiles: cL = 264 = 2 SMs -> L; one tile fewer: cM = 528 -> M
    assert both(NT=2112) == mc.Plan("L", 8, 1, (264, 1, 1))
    assert both(NT=2104) == mc.Plan("M", 4, 1, (526, 1, 1))
    # cM = 132 = SMs -> M, split once (264 CTAs = 2 per SM, 9 steps / 2 >= 4); cM = 131 -> S, whose 262 CTAs leave no room to split
    assert both(NT=528) == mc.Plan("M", 4, 2, (132, 1, 2))
    assert both(NT=524) == mc.Plan("S", 2, 1, (262, 1, 1))
    # a small grid splits K while a slice keeps 4 steps: 9 steps stop at 2 slices, 36 steps reach 8
    assert both(NT=16) == mc.Plan("S", 2, 2, (8, 1, 2))
    assert both(NT=16, cin=256) == mc.Plan("S", 2, 8, (8, 1, 8))
    # 10x10: 64 output pixels fit M and L only; 12x12: 100 fit L only; 14x14: 144 fit nothing
    assert both(NT=4, R=10, S=10) == mc.Plan("M", 1, 2, (4, 1, 2))
    assert both(NT=4, R=12, S=12, cout=200) == mc.Plan("L", 1, 2, (4, 2, 2))
    assert both(NT=4, R=14, S=14) is None
    # ksplit larger than the K loop has steps: one slice (1x1 on 64 channels is one step)
    assert both(NT=16, R=4, S=4, k=(1, 1), ksplit=8) == mc.Plan("S", 2, 1, (8, 1, 1))
    assert both(NT=16, ksplit=8) == mc.Plan("S", 2, 8, (8, 1, 8))
    # tiles per CTA bounded by the halo, not by the GEMM rows: 5x5 -> 9 pixels, 32 / 9 = 3 but 72 / 25 = 2
    assert both(NT=5, R=5, S=5) == mc.Plan("S", 2, 2, (3, 1, 2))


def test_plan_of_plain_and_modulated_descriptors_equals_its_restatement(cabi_lib):
    rng = np.random.default_rng(7)
    seen, filled = set(), 0
    for _ in range(600):
        kH, kW = (int(v) for v in rng.integers(1, 4, 2))
        stride = int(rng.integers(1, 3))
        R, S = int(rng.integers(kH, 16)), int(rng.integers(kW, 16))
        B = int(rng.integers(1, 4))
        NT = B * int(rng.choice([1, 2, 3, 7, 30, 100, 400, 1500]))
        cin, cout = 8 * int(rng.integers(1, 40)), 8 * int(rng.integers(1, 40))
        ks = int(rng.choice([0, 0, 1, 2, 4, 8]))
        p = mc.plan(NT, R, S, kH, kW, stride, cin, cout, ks)
        for modulated in (False, True):
            got = mc.plan_of(_host_desc(NT=NT, R=R, S=S, k=(kH, kW), stride=stride, cin=cin, cout=cout, ksplit=ks, B=B, flags=mc.PDL,
                                        modulated=modulated))
            assert mc.plan_tuple(got) == mc.expected_plan_tuple(p), (NT, R, S, kH, kW, stride, cin, cout, ks)
        seen.add(None if p is None else p.config)
        filled += p is not None
    assert seen == {None, "L", "M", "S"} and filled >= 300


def test_plan_of_descriptors_the_kernel_refuses_is_zero(cabi_lib):
    for kw in (dict(ksplit=3), dict(cin=36), dict(cout=36), dict(R=2), dict(R=14, S=14)):
        assert mc.plan_tuple(mc.plan_of(_host_desc(**kw))) == (0,) * 7, kw
    d = _host_desc()
    d.dtype = 0                                 # fp32 launches take the CUDA-core path
    assert mc.plan_tuple(mc.plan_of(d)) == (0,) * 7
    with pytest.raises(ValueError):
        mc.plan(16, 6, 6, 3, 3, 1, 64, 64, 3)


def test_refusals_come_before_any_launch(cabi_lib):
    from sige_b200 import _cabi

    lib = _cabi.lib()

    def refused(d, what):
        assert lib.sige_tile_conv(ctypes.byref(d), None) != 0
        assert what in lib.sige_last_error(), lib.sige_last_error()

    refused(_host_desc(R=14, S=14), b"14x14 (144 output pixels) does not fit")
    refused(_host_desc(ksplit=3), b"ksplit must be 1, 2, 4 or 8 (got 3)")
    refused(_host_desc(R=2), b"tile smaller than the kernel")
    refused(_host_desc(R=6, S=2), b"tile smaller than the kernel")


# ---------------------------------------------------------------------------------------------------------------- the case table
def _rows():
    for spec in mc.CASES:
        for ks in spec.ksplits:
            yield spec, ks, spec.plan(ks)


def test_every_case_runs_the_configuration_it_is_meant_for():
    for spec, ks, p in _rows():
        assert p is not None and p.config == spec.expect, (spec.name, ks, p)
        J = -(-spec.Cin // mc.KC) * spec.kH * spec.kW
        assert p.ksplit == (ks if 0 < ks <= J else 1) or ks == 0, (spec.name, ks, p)


def test_every_case_keeps_its_configuration_on_any_h100():
    """114 SMs (PCIe) to 144: the case sizes leave room on both sides of each threshold."""
    for spec, ks, _ in _rows():
        for sms in (114, 132, 144):
            assert spec.plan(ks, sms).config == spec.expect, (spec.name, sms)


def test_no_case_is_ambiguous():
    """M and S both report bn 64: a case stands for its configuration only if no other one would give the same (bn, grid).  Grids of
    one CTA (fewer tiles than S packs) look the same under both; those cases are marked single_cta and do not count below."""
    for spec, ks, p in _rows():
        for sms in (114, 132, 144):
            p = spec.plan(ks, sms)
            assert bool(spec.ambiguous(p, ks, sms)) == spec.single_cta, (spec.name, ks, sms, p, spec.ambiguous(p, ks, sms))
        if spec.single_cta:
            assert p.grid[0] == 1 and spec.expect == "S"


def test_case_table_reaches_every_instantiation():
    reached = {(dt, spec.expect, int(spec.mod is not None)) for spec in mc.CASES if not spec.single_cta for dt in ("f16", "bf16")}
    assert len(mc.ALL_INSTANTIATIONS) == 12
    assert sorted(reached) == mc.ALL_INSTANTIATIONS, "missing: %s" % sorted(set(mc.ALL_INSTANTIATIONS) - reached)


def test_case_table_covers_every_feature():
    seen = set().union(*(mc.features(s) for s in mc.CASES))
    assert mc.REQUIRED_FEATURES <= seen, "not covered: %s" % sorted(mc.REQUIRED_FEATURES - seen)
    assert {s.Cout for s in mc.CASES} >= {8, 72, 136, 200}
    # every requested split on each K-loop shape the kernel treats differently
    for name in ("S_rows4", "K_27_over_4", "K_cin40", "K_cin96", "K_cin200", "K_1x1_cin64"):
        (spec,) = [s for s in mc.CASES if s.name == name]
        assert spec.ksplits == mc.ALL_KS
    # whole CTAs of padding in the SIGE_CONV_PADDED case
    (spec,) = [s for s in mc.CASES if s.padded]
    assert spec.B == 1 and (spec.N - spec.counts[0]) // spec.plan(0).tpc >= 2


@pytest.mark.parametrize("spec", mc.CASES, ids=lambda s: s.name)
def test_case_is_well_formed(spec):
    """The tensors build, the descriptor passes its own invariants, no two tiles write one pixel (reference() asserts it), padding
    sits at the tail of each list, and something is written next to something that is not."""
    big = spec.NT > 700
    case = mc.make_case(dataclasses.replace(spec, srcs=tuple((8, up) for _, up in spec.srcs), Cout=8, dst=None if spec.dst is None else (0, 0),
                                            residual=None if spec.residual is None else (0, 0), window=None, mod=None,
                                            aux=tuple((0, 0, a, b) for _, _, a, b in spec.aux)) if big else spec, torch.float32, "cpu")
    expects = mc.reference(case)
    assert len(expects) == len(case.buffers())
    for e in expects:
        assert bool(e.written.any())
        assert not bool(e.written[:e.g.off].any()) and not bool(e.written[e.g.off + e.g.view.numel():].any())
        assert spec.dst_stack or not bool(e.written.all())
    if case.idx is not None:
        idx = case.idx.numpy().reshape(spec.B if spec.per_image else 1, spec.N, 2)
        for b, n in enumerate(spec.counts if spec.per_image else spec.counts[:1]):
            assert len({tuple(r) for r in idx[b, :n]}) == n and (idx[b, n:] == mc.TILE_NONE).all()
    if spec.mod:
        assert not spec.src_stack and not spec.per_image and spec.act == 0 and len(spec.srcs) == 1
    if spec.window:
        assert not spec.src_stack and not spec.per_image and len(spec.srcs) == 1
    if spec.per_image or spec.padded:
        assert not spec.src_stack and not spec.dst_stack


# ---------------------------------------------------------------------------------------------------------------- check() bites
def _exact(spec):
    case = mc.make_case(spec, torch.float16, "cpu")
    expects = mc.reference(case)
    init = kc.snapshot(case.buffers())
    got = mc.rounded_result(case, expects)
    kc.check(spec.name, expects, got, init)            # the contract accepts its own result
    return case, expects, got, init


def _roll(e, shift):
    """The expectation with its written values, mask and bounds moved by `shift` elements of the flat buffer."""
    base = e.g.flat.double()
    written = torch.roll(e.written, shift)
    want = torch.where(written, torch.roll(e.want, shift), base)
    return dataclasses.replace(e, want=want, written=written, bound=torch.roll(e.bound, shift), rounding=torch.roll(e.rounding, shift))


def test_check_rejects_a_pixel_decoded_into_the_next_tile():
    """5x5 / 3x3 tiles (9 pixels, idle rows): the expectation of one output pixel swapped with the same pixel of the next tile."""
    spec = mc.Spec("idle_rows", B=1, srcs=((16, 0),), Cout=8, counts=(6,), R=5, src_stack=True, dst_stack=True, seed=221)
    case, expects, got, init = _exact(spec)
    (e,) = expects
    want = e.want.clone()
    v = want[e.g.off:e.g.off + e.g.view.numel()].view(*e.g.view.shape)
    v[[2, 3], 1, 2] = v[[3, 2], 1, 2]
    with pytest.raises(AssertionError, match=r"\(b, c, h, w\) = \([23], \d, 1, 2\)"):
        kc.check(spec.name, [dataclasses.replace(e, want=want)], got, init)


def test_check_rejects_floor_division_of_a_negative_origin():
    spec = mc.Spec("neg", B=1, H=20, W=20, srcs=((16, 0),), Cout=8, counts=(8,), R=5, stride=2, dHW=(10, 10), c_div_tile=True, seed=222)
    case, expects, got, init = _exact(spec)
    with pytest.raises(AssertionError):
        kc.check(spec.name, mc.reference(case, floor_division=True), got, init)


def test_check_rejects_a_channel_vector_past_a_72_channel_window():
    spec = mc.Spec("window72", B=1, H=12, W=12, srcs=((16, 0),), Cout=72, counts=(5,), R=6, dst=(16, 8), seed=223)
    case, expects, got, init = _exact(spec)
    (e,) = expects
    # a kernel that wrote channels [16, 88) instead of [8, 80): eight elements past the window at every written pixel
    wrong = _roll(e, 8)
    moved = {"dst": torch.where(wrong.written, torch.roll(got["dst"], 8), init["dst"])}
    kc.check(spec.name, [wrong], moved, init)          # consistent with the wrong contract ...
    with pytest.raises(AssertionError):
        kc.check(spec.name, [wrong], got, init)        # ... which rejects the right result ...
    with pytest.raises(AssertionError, match="outside the written set"):
        kc.check(spec.name, expects, moved, init)      # ... and the right contract catches the shifted one
    # and the last pixel of the buffer: a vector past its window lands in the guard band
    stack = mc.Spec("guard", B=1, srcs=((16, 0),), Cout=72, counts=(3,), R=6, src_stack=True, dst_stack=True, seed=224)
    case, expects, got, init = _exact(stack)
    (e,) = expects
    wrong = _roll(e, 8)
    moved = {"dst": torch.where(wrong.written, torch.roll(got["dst"], 8), init["dst"])}
    with pytest.raises(AssertionError, match="guard element"):
        kc.check(stack.name, expects, moved, init)
