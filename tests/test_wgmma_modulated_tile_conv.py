"""Modulated tile convs on the wgmma kernel: with SIGE_CONV_TC5, a modulated sige_tile_conv runs the stride-1 wgmma geometries (3x3 on
6x6 tiles, 1x1 on 4x4 tiles, Cin and Cout multiples of 64) on the MOD instantiations of tile_conv_tc5_kernel, whose register-staged
gather applies SPADE's modulation leaky((x*scale + shift) * (1 + gamma) + beta).  Everything else stays on the mma.sync kernel.

CPU (host-only planning: the plan of an H100 80GB HBM3, as in test_tile_conv_contract.py): sige_tile_conv_plan of a modulated
descriptor gives the intended instantiation for every case and split of the table below, the table reaches all 12 MOD
instantiations, and the launches that stay on mma.sync plan it.
GPU: every case against the float64 contract (tests/test_modulated_tile_conv.py's mod_reference), with the plan on the device checked;
gamma = beta = 0 with slope 1 equals the plain wgmma launch bitwise; the SPADE generator miniature runs its wide modulated launches on
wgmma."""
import ctypes
import dataclasses
import os
import sys

import pytest
import torch

from conftest import REPO

sys.path.insert(0, os.path.join(REPO, "tests"))

import mma_tile_conv_contract as MC  # noqa: E402
import tile_conv_contract as TC  # noqa: E402
import test_modulated_tile_conv as TM  # noqa: E402
from test_modulated_tile_conv import Mod  # noqa: E402

W = (128, 1, 0)          # wide tiles, never split
# (spec, Mod): spec.ksplits are the splits requested, spec.expect the intended plan of each, (BN, effective ksplit, double halo)
CASES = [
    # ---- BN = 128 (m_blocks * Cout/128 >= 132) ----
    (TC.Spec("MW3_up_windows", B=1, H=100, W=100, srcs=((256, 1),), Cout=256, counts=(560,), preop="shared", residual=(0, 0),
             ksplits=(0, 1, 4), expect=(W, W, W), seed=801), Mod(64, 64, 8, 8)),
    (TC.Spec("MW1_aux_only_slope1", B=1, H=74, W=74, k=1, srcs=((256, 0),), Cout=512, counts=(300,), dst=None, aux=((8, 8, True, 1),),
             ksplits=(0, 2), expect=(W, W), seed=802), Mod(slope=1.0)),
    # ---- BN = 64 (m_blocks * Cout/64 <= 100) ----
    # 128 -> 128 on 2 x 50 tiles: 6 ring steps; ksplit 8 > 6 falls back to one slice
    (TC.Spec("MN3_per_sample_residual", B=2, H=46, W=46, srcs=((128, 0),), Cout=128, counts=(50,), preop="per_sample", residual=(8, 8),
             ksplits=(0, 1, 2, 4, 8), expect=((64, 4, 0), (64, 1, 0), (64, 2, 0), (64, 4, 0), (64, 1, 0)), seed=803), Mod(16, 8, 8, 0)),
    # 256 -> 64 (the shape of a SPADE block's last conv_1): ksplit 2 spans two halo fills per slice, the double-buffered layout
    (TC.Spec("MN3d_up_padded", B=1, H=62, W=62, srcs=((256, 1),), Cout=64, counts=(203,), pad_to=232, padded=True, preop="shared",
             ksplits=(0, 1, 2, 4, 8), expect=((64, 4, 0), (64, 1, 0), (64, 2, 1), (64, 4, 0), (64, 8, 0)), seed=804), Mod()),
    (TC.Spec("MN1_per_sample_dst_window", B=2, H=50, W=50, k=1, srcs=((384, 0),), Cout=128, counts=(75,), preop="per_sample", dst=(16, 8),
             ksplits=(0, 1, 2, 4, 8), expect=((64, 2, 0), (64, 1, 0), (64, 2, 0), (64, 4, 0), (64, 1, 0)), seed=805), Mod(0, 0, 24, 16)),
]

# every MOD instantiation tc5_launch can reach: (dtype, BN, taps, S2, DEEP, DB, ASYNC), all register-staged
MOD_INSTANTIATIONS = sorted(
    [(dt, 128, taps, 0, 0, 0, 0) for dt in ("f16", "bf16") for taps in (9, 1)]
    + [(dt, 64, 9, 0, deep, db, 0) for dt in ("f16", "bf16") for (deep, db) in ((0, 0), (1, 0), (1, 1))]
    + [(dt, 64, 1, 0, 0, 0, 0) for dt in ("f16", "bf16")]
)


def modulated_plan(d):
    """sige_tile_conv_plan of a copy of `d` whose modulation is set (the plan never reads it)."""
    from sige_b200 import _cabi

    m = type(d).from_buffer_copy(d)
    m.modulation = ctypes.pointer(_cabi.ConvModulation())
    return TC.plan_of(m)


def instantiation(spec, dtype, plan):
    """The MOD instantiation a modulated plan launches (the register-staged gather: ASYNC = 0), or None for mma.sync."""
    key = TC.instantiation(spec, dtype, plan)
    return None if key is None else key[:6] + (0,)


def intended(spec, dtype, i):
    key = TC.intended(spec, dtype, i)
    return None if key is None else key[:6] + (0,)


def mod_features(spec, mod):
    f = TC.features(spec) & {"per_sample_affine", "shared_affine", "residual", "aux_only", "upsampled_source", "channel_windows", "padded"}
    if spec.preop is None:
        f.add("no_affine")
    if mod.gamma_c0 or mod.beta_c0 or mod.gamma_extra or mod.beta_extra:
        f.add("gamma_beta_windows")
    if mod.slope == 1.0:
        f.add("slope1")
    return f


# ---------------------------------------------------------------------------------------------------------------- plans (CPU)
def _table_plans():
    out = []
    for spec, mod in CASES:
        case = TC.make_case(spec, torch.float16, "cpu")
        for dtype in (torch.float16, torch.bfloat16):
            case.dtype = dtype
            for i, ks in enumerate(spec.ksplits):
                for flags in (TC.TC5, TC.TC5 | TC.PDL | (TC.PADDED if spec.padded else 0)):
                    plan = modulated_plan(TC.descriptor(case, ks, flags))
                    out.append((spec, mod, dtype, i, ks, plan, instantiation(spec, dtype, plan)))
    return out


@pytest.fixture(scope="module")
def table_plans(cabi_lib):
    return _table_plans()


def test_modulated_descriptor_plans_are_the_intended_ones(table_plans):
    for spec, _, dtype, i, ks, plan, key in table_plans:
        assert key == intended(spec, dtype, i), "%s %s ksplit %d: plan %s -> %s, intended %s" % (
            spec.name, TC.DTYPE_NAME[dtype], ks, TC.plan_str(plan), key, intended(spec, dtype, i))
        assert plan.ksplit == spec.expect[i][1]


def test_modulated_descriptor_plans_reach_every_mod_instantiation(table_plans):
    keys = {key for *_, key in table_plans if key is not None}
    assert len(MOD_INSTANTIATIONS) == 12
    assert sorted(keys) == MOD_INSTANTIATIONS, "missing: %s" % sorted(set(MOD_INSTANTIATIONS) - keys)


def test_modulated_descriptor_plans_cover_every_feature_wide_and_narrow(table_plans):
    seen = set()
    for spec, mod, _, _, _, plan, _ in table_plans:
        seen |= {(f, "wide" if plan.bn == 128 else "narrow") for f in mod_features(spec, mod)}
    required = {(f, "narrow") for f in ("per_sample_affine", "shared_affine", "residual", "upsampled_source", "channel_windows", "padded",
                                         "gamma_beta_windows")}
    required |= {(f, "wide") for f in ("shared_affine", "residual", "aux_only", "upsampled_source", "gamma_beta_windows", "slope1", "no_affine")}
    assert required <= seen, "not covered: %s" % sorted(required - seen)


def test_modulated_case_table_sizes_do_not_depend_on_the_h100_variant():
    for spec, _ in CASES:
        m_blocks = -(-spec.B * spec.N // 8)
        for e in spec.expect:
            if e[0] == 128:
                assert m_blocks * spec.Cout // 128 >= 132, spec.name
            else:
                assert m_blocks * spec.Cout // 64 <= 100, spec.name


def test_modulated_descriptors_that_stay_on_mma_sync_plan_it(cabi_lib):
    """No flag, a narrow Cin, a Cout that is not a multiple of 64, stride 2: the plan of a modulated descriptor says mma.sync (path 0) with
    that kernel's configuration and grid (restated in tests/mma_tile_conv_contract.py); the wgmma geometries with the flag plan wgmma
    exactly as the unmodulated descriptor does."""
    def plans(spec, flags):
        d = TC.descriptor(TC.make_case(spec, torch.float16, "cpu"), 0, flags)
        return modulated_plan(d), TC.plan_of(d)

    base = TC.Spec("base", B=1, H=62, W=62, srcs=((256, 0),), Cout=64, counts=(100,), preop="shared", seed=811)
    mod, plain = plans(base, TC.TC5)
    assert mod.path == 1 and (mod.bn, mod.ksplit, mod.deep_ring, mod.grid_x, mod.grid_y, mod.grid_z) == \
        (plain.bn, plain.ksplit, plain.deep_ring, plain.grid_x, plain.grid_y, plain.grid_z)
    for spec, flags in ((base, 0), (base, TC.PDL),
                        (dataclasses.replace(base, srcs=((96, 0),)), TC.TC5),
                        (dataclasses.replace(base, Cout=96), TC.TC5),
                        (dataclasses.replace(base, k=1, srcs=((40, 0),)), TC.TC5)):
        mod, _ = plans(spec, flags)
        want = MC.plan(spec.B * spec.N, spec.R, spec.R, spec.k, spec.k, spec.stride, spec.Cin, spec.Cout, 0)
        assert MC.plan_tuple(mod) == MC.expected_plan_tuple(want) and mod.path == 0 and mod.bn == 64, (spec.srcs, spec.Cout, flags)
    # stride 2 without a pre-op is a wgmma geometry for sige_tile_conv (pure-copy gather), not for the modulated launch
    s2 = TC.Spec("s2", B=1, H=34, W=30, stride=2, srcs=((64, 0),), Cout=128, counts=(40,), seed=812)
    mod, plain = plans(s2, TC.TC5)
    assert plain.path == 1 and mod.path == 0


def test_one_plan_query_for_modulated_descriptors(cabi_lib):
    import test_cabi_symbols as TS
    from sige_b200 import _cabi

    assert set(_cabi.PROTOTYPES) == TS._declared()
    assert _cabi.lib().sige_abi_version() == 3
    assert _cabi.lib().sige_tile_conv_plan(None, None) != 0 and b"null" in _cabi.lib().sige_last_error()


# ---------------------------------------------------------------------------------------------------------------- kernel (GPU)
def _device_plan_key(mc, ks, flags):
    return instantiation(mc.case.spec, mc.case.dtype, modulated_plan(TC.descriptor(mc.case, ks, flags)))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_wgmma_modulation_field_against_the_float64_contract(dtype):
    """Every case, at every split of the table, with and without PDL (and PADDED where the list is padded): the plan on this device is
    the intended MOD instantiation, every written element is within the contract's bound and every other element is unchanged."""
    dev = torch.device("cuda:0")
    worst = excess = 0.0
    n = 0
    for spec, mod in CASES:
        mc = TM._mod_case(spec, mod, dtype, dev)
        case = mc.case
        init = {k: v.clone() for k, v in case.buffers().items()}
        expects = TM.mod_reference(mc)
        for i, ks in enumerate(spec.ksplits):
            for flags in (TC.TC5, TC.TC5 | TC.PDL | (TC.PADDED if spec.padded else 0)):
                key, want = _device_plan_key(mc, ks, flags), intended(spec, dtype, i)
                label = "%s %s ksplit=%d flags=%d" % (spec.name, TC.DTYPE_NAME[dtype], ks, flags)
                assert key == want, "%s: plan %s, intended %s" % (label, key, want)
                for name, buf in case.buffers().items():
                    buf.copy_(init[name])
                TM._launch(mc, ks, flags)
                got = {k: v.clone() for k, v in case.buffers().items()}
                w_, e_ = TC.check(label, expects, got, init)
                worst, excess, n = max(worst, w_), max(excess, e_), n + 1
    print("wgmma modulated contract %s: %d launches, worst error/bound %.3f, accumulation headroom used %.3f" % (TC.DTYPE_NAME[dtype], n, worst, excess))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_zero_modulation_field_equals_the_plain_wgmma_launch(dtype):
    """gamma = beta = 0 and slope 1: bitwise the plain wgmma launch with the same scale / shift pre-op (both run the register-staged
    gather of the same plan): 3x3 and 1x1, BN 64 and 128, split and un-split, up-sampled sources."""
    dev = torch.device("cuda:0")
    n = 0
    for spec, _ in CASES:
        spec = spec if spec.preop else dataclasses.replace(spec, preop="shared")
        mc = TM._mod_case(spec, Mod(slope=1.0), dtype, dev)
        mc.gamma.zero_()
        mc.beta.zero_()
        case = mc.case
        init = {k: v.clone() for k, v in case.buffers().items()}
        for ks in spec.ksplits:
            outs = []
            for mod in (True, False):
                for name, buf in case.buffers().items():
                    buf.copy_(init[name])
                TM._launch(mc, ks, TC.TC5, mod=mod)
                outs.append({k: v.clone() for k, v in case.buffers().items()})
            assert _device_plan_key(mc, ks, TC.TC5) is not None
            for name in outs[0]:
                assert torch.equal(outs[0][name].view(torch.int16), outs[1][name].view(torch.int16)), (spec.name, ks, name)
                assert not torch.equal(outs[0][name], init[name])
            n += 1
    print("zero modulation %s: %d launches bitwise equal to the plain wgmma launch" % (TC.DTYPE_NAME[dtype], n))


# ---------------------------------------------------------------------------------------------------------------- fused step (GPU)
# The miniature's sparse blocks up_0 .. up_3 (ngf 32: 512 -> 256, 256 -> 128, 128 -> 64, 64 -> 32) each have three modulated launches,
# conv_0 (fin -> fmiddle, 3x3), conv_1 (fmiddle -> fout, 3x3) and conv_s (fin -> fout, 1x1).  Those of up_0, up_1 and up_2 have Cin and
# Cout multiples of 64 and run on wgmma; up_3's have Cout 32 (and conv_1 Cin 32) and stay on mma.sync.
MINI_WGMMA_MODULATED = 9


@pytest.mark.gpu
def test_spade_miniature_runs_its_wide_modulated_launches_on_wgmma():
    import test_spade_generator as TSG
    from sige.utils import dilate_mask, downsample_mask
    from sige_b200.roofline import plan_of

    net = TSG._generator("mini", "intree").to("cuda:0")
    TSG.consumers.run_gaugan(net, downsample_mask, dilate_mask, device="cuda:0", fused=lambda n: n.set_fused(True, dtype=torch.float16))
    step = net.fused_step
    mods = [f for f in step.fused if f.spec.modulation is not None]
    on_wgmma = [f for f in mods if plan_of(f).path == 1]
    assert len(mods) == 12
    assert len(on_wgmma) == MINI_WGMMA_MODULATED, [(f.name, f.spec.Cin, f.spec.Cout, f.spec.k) for f in on_wgmma]
    assert all(f.spec.Cin % 64 == 0 and f.spec.Cout % 64 == 0 for f in on_wgmma)
