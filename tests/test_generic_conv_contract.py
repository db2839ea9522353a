"""CPU checks of tests/generic_conv_contract.py: the float64 restatement of sige_tile_conv_generic against independent computations
(F.conv2d, the in-tree C oracle, a float32 conv of another summation order), mutants of the kernel that the bound must reject,
the case table against the launcher's predicate, and the C-ABI refusals that come before any CUDA call."""
import pytest
import torch
import torch.nn.functional as F

import generic_conv_contract as gc
import kernel_contracts as kc

F64 = torch.float64
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT = pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "bf16"])
P = 0x10000                     # not device memory: a launch would fault, so these calls must fail on their arguments
CPU_MACS = 2 * 10 ** 7          # float64 restatements the CPU finishes in well under a second
SMALL = [s for s in gc.GEN_CASES if gc.gen_cost(s) <= CPU_MACS]


def _window(e: kc.Expect, t: torch.Tensor) -> torch.Tensor:
    return t[e.g.off:e.g.off + e.g.view.numel()].view(*e.g.view.shape)


def _logical(case: gc.GenCase, e: kc.Expect, t: torch.Tensor) -> torch.Tensor:
    return case.logical(_window(e, t))


def _within(case: gc.GenCase, e: kc.Expect, val: torch.Tensor, label: str):
    """`val` (logical NCHW, already in the launch dtype) passes `check` as the launch's output."""
    got = gc.gen_written(case, val)
    kc.check(label, [e], {"out": got}, {"out": case.out.flat})


# ---------------------------------------------------------------------------------------------------------------- restatement
@pytest.mark.parametrize("spec", SMALL, ids=lambda s: s.name)
def test_restatement_matches_conv2d(spec):
    """float64 operands: the restatement's values are F.conv2d(x, w, b, stride, 0, dilation, groups) to 1e-12, in the case's
    layout; it writes the whole output window and nothing outside it; its bound is positive everywhere."""
    case = gc.make_gen(spec, F64, "cpu")
    (e,) = gc.gen_reference(case)
    want = F.conv2d(case.x_nchw, case.w.view, case.bias, spec.stride, 0, spec.dilation, spec.groups)
    assert tuple(want.shape) == (spec.M, spec.Cout, spec.Ro, spec.So)
    torch.testing.assert_close(_logical(case, e, e.want), want, rtol=1e-12, atol=1e-12)
    assert bool(_window(e, e.written).all()) and int(e.written.sum()) == case.out.view.numel()
    assert bool((_window(e, e.bound) > 0).all())
    assert torch.equal(e.want[~e.written], case.out.flat[~e.written])


@pytest.mark.parametrize("spec", SMALL, ids=lambda s: s.name)
def test_oracle_lies_within_the_f32_bound(spec, oracle):
    """The in-tree C oracle (float64 accumulation, one rounding to fp32) on the f32 operands is within the f32 bound."""
    case = gc.make_gen(spec, torch.float32, "cpu")
    (e,) = gc.gen_reference(case)
    b = None if case.bias is None else case.bias.numpy()
    got = oracle.conv2d_tiles(case.x_nchw.contiguous().numpy(), case.w.view.numpy(), b, spec.stride, spec.dilation, spec.groups)
    _within(case, e, torch.from_numpy(got), "%s oracle" % spec.name)


@DT
@pytest.mark.parametrize("spec", SMALL, ids=lambda s: s.name)
def test_a_float32_conv_of_another_summation_order_lies_within_the_bound(spec, dtype):
    """torch's float32 CPU conv of the stored operands (its own summation order, rounded products where it does not fuse them),
    rounded to the dtype: the bound holds for any order of the K products, not just the kernel's."""
    case = gc.make_gen(spec, dtype, "cpu")
    (e,) = gc.gen_reference(case)
    b = None if case.bias is None else case.bias.float()
    got = F.conv2d(case.x_nchw.float(), case.w.view.float(), b, spec.stride, 0, spec.dilation, spec.groups)
    _within(case, e, got, "%s float32 conv" % spec.name)


def test_bound_is_rigorous_where_it_is_tight():
    """The f32 bound is gamma_{K+1} mag: small enough that a single product of a typical size exceeds it (the mutants below),
    and yet never smaller than the one rounding the C oracle's float64 sum takes (u |want| <= gamma_2 mag)."""
    assert gc.gamma(1) > gc.U32 and gc.gamma(10) < 10.01 * gc.U32
    for spec in SMALL:
        case = gc.make_gen(spec, torch.float32, "cpu")
        (e,) = gc.gen_reference(case)
        w = e.written
        assert bool((e.bound[w] >= gc.U32 * e.want[w].abs()).all()), spec.name
        assert not bool(e.rounding.any()), "f32 stores the fp32 result as it is: no rounding of its own"
        # a typical product: the bound is below it on the median element
        v, mag = gc.gen_values(case)
        assert float((e.bound[w] / (mag.flatten() / spec.K)).median()) < 0.05, spec.name


# ---------------------------------------------------------------------------------------------------------------- sensitivity
@DT
@pytest.mark.parametrize("mutant", gc.MUTANTS)
def test_the_bound_rejects_every_mutant_where_it_changes_the_math(mutant, dtype):
    """A kernel with one mistake, computed in float64 and rounded to the dtype: `check` rejects it on at least one written
    element of every case the mutation applies to (and passes the correct values of the same case)."""
    applied = 0
    for spec in gc.GEN_CASES:
        if not gc.mutant_applies(spec, dtype, mutant):
            continue
        case = gc.make_gen(spec, dtype, "cpu")
        (e,) = gc.gen_reference(case)
        label = "%s %s %s" % (spec.name, mutant, dtype)
        _within(case, e, _logical(case, e, e.want), label)
        bad = gc.gen_mutant(case, mutant)
        assert not torch.equal(bad, _logical(case, e, e.want)), "%s: the mutation does not change the math" % label
        with pytest.raises(AssertionError, match="> bound"):
            _within(case, e, bad, label)
        applied += 1
    assert applied > 0 or (mutant == "other16" and dtype != torch.float16), (mutant, dtype)


def test_bf16_weights_survive_the_round_trip_through_f16():
    """Why the other16 mutant applies to f16 only: bf16's 8-bit significand fits f16's 11 bits, so the round trip moves only
    the weights below f16's normal range (2^-14)."""
    for spec in gc.GEN_CASES:
        w = gc.make_gen(spec, torch.bfloat16, "cpu").w.view
        moved = w.to(torch.float16).to(torch.bfloat16) != w
        assert not bool(moved[w.abs() >= 2.0 ** -14].any()), spec.name


# ---------------------------------------------------------------------------------------------------------------- coverage
def test_case_table_reaches_every_path_in_every_dtype():
    for dt in DTYPES:
        assert {gc.generic_path(s, dt, s.misalign) for s in gc.GEN_CASES} == set(gc.PATHS), dt
        for form in ("dw_vec", "dw_nhwc_scalar", "dw_nchw"):
            trips = [gc.dw_trips(s, dt, s.misalign) for s in gc.GEN_CASES if gc.generic_path(s, dt, s.misalign) == form]
            assert max(trips) >= 2, "a second grid-stride trip of %s at 132 SMs (%s)" % (form, dt)
    for m in gc.MUTANTS:
        assert any(gc.mutant_applies(s, torch.float16, m) for s in gc.GEN_CASES), m


def test_case_table_contains_every_edge():
    C = gc.GEN_CASES
    simt = [s for s in C if not s.depthwise]
    dw = [s for s in C if s.depthwise]
    geo = {(s.kH, s.kW, s.R, s.S) for s in C}
    # chunk and block edges
    assert any(s.cig < gc.SIMT_CI for s in simt) and any(s.cig == 36 and gc.k_chunks(s) == 3 for s in simt)
    assert any(s.cog == 70 and gc.cout_blocks(s) == 2 for s in simt) and any(s.Cin == 3 for s in simt)
    # pixel passes and shared memory
    assert {(3, 3, 10, 10), (1, 1, 8, 8)} <= {(s.kH, s.kW, s.R, s.S) for s in simt if s.P == 64 and gc.pixel_passes(s) == 2}
    assert {(5, 5, 9, 9), (3, 3, 14, 14)} <= {(s.kH, s.kW, s.R, s.S) for s in simt if gc.simt_smem(s) > gc.SMEM_DEFAULT}
    assert (7, 7, 12, 12) in geo and any(s.M >= 1500 for s in simt)
    # anisotropic geometry
    assert any(s.R != s.S for s in C) and {(1, 3), (3, 1)} <= {(s.kH, s.kW) for s in C}
    assert any(s.strideH != s.strideW for s in C) and any(s.dilH != s.dilW for s in C)
    assert any(s.strideH == s.strideW == 2 and s.R == s.S == 5 for s in simt)
    # groups
    assert any(s.groups == 2 and s.cig == 20 and s.cog == 70 for s in C)
    assert any(s.groups == 4 and s.dilH == s.dilW == 2 for s in C)
    mult = [s for s in C if s.groups == s.Cin == 16 and s.Cout == 32]
    assert mult and all(gc.generic_path(s, dt, s.misalign) == "simt" for s in mult for dt in DTYPES)
    # depthwise forms
    f32, f16, bf16 = DTYPES
    path = lambda s, dt: gc.generic_path(s, dt, s.misalign)                              # noqa: E731
    assert {"dw_nchw", "dw_vec"} <= {path(s, f16) for s in dw if s.Cin == 128}
    assert any(s.Cin == 6 and all(path(s, dt) == "dw_nhwc_scalar" for dt in DTYPES) for s in dw)
    assert any(s.Cin == 12 and path(s, f32) == "dw_vec" and path(s, f16) == path(s, bf16) == "dw_nhwc_scalar" for s in dw)
    assert any(s.misalign and s.Cin % 8 == 0 and path(s, f32) == "dw_nhwc_scalar" for s in dw)
    assert any(s.strideH == s.strideW == 2 for s in dw) and any(s.dilH == s.dilW == 2 for s in dw)
    assert gc.dw_trips(gc.GenSpec("t", 2112, 128, 128, 6, 6, groups=128, layout="nhwc"), f16, False) == 1
    assert gc.dw_trips(gc.GenSpec("t", 2113, 128, 128, 6, 6, groups=128, layout="nhwc"), f16, False) == 2   # > 540,672 vectors
    # bias and values
    assert any(not s.bias for s in simt) and any(not s.bias for s in dw) and any(s.spread for s in C)
    assert len({s.name for s in C}) == len(C) and len({s.seed for s in C}) == len(C)


def test_misaligned_windows_are_one_element_off():
    """Misalignment is by whole elements (4 bytes for f32, 2 for 16-bit): never an address no element can have."""
    spec = next(s for s in gc.GEN_CASES if s.misalign)
    for dt in DTYPES:
        case = gc.make_gen(spec, dt, "cpu")
        es = case.out.flat.element_size()
        assert case.out.view.data_ptr() % 16 == es and case.out.view.data_ptr() % es == 0, dt
        assert all(t.data_ptr() % 16 == 0 for t in (case.x.view, case.w.view, case.b.view)), dt
        aligned = gc.make_gen(spec, dt, "cpu", misalign=False)
        assert aligned.out.view.data_ptr() % 16 == 0 and torch.equal(kc.bits(aligned.x.view), kc.bits(case.x.view))


def test_layouts_hold_the_same_values():
    spec = next(s for s in gc.GEN_CASES if s.name == "g4_dil2_nhwc")
    a, b = gc.make_gen(spec, torch.float16, "cpu", layout="nchw"), gc.make_gen(spec, torch.float16, "cpu", layout="nhwc")
    assert torch.equal(a.x_nchw, b.x_nchw) and torch.equal(a.w.view, b.w.view) and torch.equal(a.bias, b.bias)
    assert b.x.view.is_contiguous() and b.x_nchw.is_contiguous(memory_format=torch.channels_last)


# ---------------------------------------------------------------------------------------------------------------- refusals
def test_generic_conv_refuses_bad_arguments_before_any_cuda_call(cabi_lib):
    """The pointers here are not device memory: a launch would fault, so these calls must fail on their arguments."""
    from sige_b200 import _cabi

    lib = _cabi.lib()

    def call(dtype=_cabi.F32, layout=_cabi.NCHW, M=2, Cin=8, R=6, S=6, Cout=8, kH=3, kW=3, sH=1, sW=1, dH=1, dW=1, groups=1,
             x=P, w=P, out=P):
        return lib.sige_tile_conv_generic(x, w, None, out, dtype, layout, M, Cin, R, S, Cout, kH, kW, sH, sW, dH, dW, groups, None)

    for bad in (dict(M=-1), dict(Cin=0), dict(Cout=0), dict(R=0), dict(S=0), dict(kH=0), dict(kW=0), dict(sH=0), dict(sW=0),
                dict(dH=0), dict(dW=0), dict(groups=0)):
        assert call(**bad) != 0 and b"bad shape" in lib.sige_last_error(), bad
    for bad in (dict(Cin=8, groups=3, Cout=9), dict(Cin=6, groups=3, Cout=8)):
        assert call(**bad) != 0 and b"not divisible by groups" in lib.sige_last_error(), bad
    for bad in (2, -1):
        assert call(layout=bad) != 0 and b"bad layout" in lib.sige_last_error(), bad
    for bad in (dict(R=2), dict(S=2), dict(R=4, dH=2), dict(S=6, kW=4, dW=2), dict(kH=7)):
        assert call(**bad) != 0 and b"tile smaller than the (dilated) kernel" in lib.sige_last_error(), bad
    for dt in (3, -1):
        assert call(dtype=dt) != 0 and b"unsupported dtype" in lib.sige_last_error(), dt
        assert call(dtype=dt, Cin=8, Cout=8, groups=8) != 0 and b"unsupported dtype" in lib.sige_last_error(), ("depthwise", dt)
    assert call(x=None) != 0 and b"null pointer" in lib.sige_last_error()
    # M = 0: nothing to do, null pointers included
    assert call(M=0, x=None, w=None, out=None) == 0
    assert call(M=0, x=None, w=None, out=None, Cin=16, Cout=16, groups=16, layout=_cabi.NHWC) == 0
