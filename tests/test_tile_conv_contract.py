"""CPU checks of the tile-conv contract helpers (tests/tile_conv_contract.py), no GPU needed:

  * the float64 restatement of the sige_tile_conv descriptor agrees with the C oracle's gather -> conv -> scatter
    (and scatter_with_block_residual) composites on small fp32 cases;
  * the GPU sweep's case table reaches every wgmma kernel instantiation tc5_launch can pick, and every feature in its wide
    (BN = 128) and narrow (BN = 64) form.  The plans come from sige_tile_conv_plan, which without a device plans for an
    H100 80GB HBM3 (132 SMs).
"""
import numpy as np
import pytest
import torch

import tile_conv_contract as tcc

# small fp32 cases the oracle can compose (one tile list shared by the batch)
ORACLE_CASES = [
    tcc.Spec("shared_list", B=1, H=22, W=22, srcs=((64, 0),), Cout=64, counts=(20,), preop="shared", act=1, residual=(0, 0), seed=21),
    tcc.Spec("stride2", B=1, H=18, W=14, stride=2, srcs=((64, 0),), Cout=64, counts=(10,), residual=(0, 0), c_div_tile=True, seed=22),
    tcc.Spec("one_by_one", B=1, H=18, W=18, k=1, srcs=((64, 0),), Cout=72, counts=(15,), preop="shared", act=0, residual=(0, 0), seed=23),
    tcc.Spec("shortcut_flags", B=1, H=22, W=22, srcs=((64, 0),), Cout=64, counts=(20,), residual=(0, 0), shortcut=(64, 64), sc_flags=True,
             seed=24),
    tcc.Spec("upsampled", B=1, H=20, W=20, srcs=((64, 1),), Cout=64, counts=(18,), residual=(0, 0), seed=25),
    tcc.Spec("two_sources", B=1, H=22, W=18, srcs=((64, 0), (64, 1)), Cout=64, counts=(16,), seed=26),
    tcc.Spec("batch2_per_sample_affine", B=2, H=22, W=22, srcs=((64, 0),), Cout=64, counts=(20,), preop="per_sample", act=1,
             residual=(0, 0), seed=27),
]


def _nchw(t):
    return np.ascontiguousarray(t.permute(0, 3, 1, 2).float().numpy())


def _oracle_composite(oracle, case):
    s = case.spec
    x = np.concatenate([_nchw(t).repeat(1 << up, 2).repeat(1 << up, 3) for t, (_, up) in zip(case.srcs, s.srcs)], 1)
    idx = case.idx.numpy()
    sc = sh = None
    if s.preop:
        sc = case.scale.numpy().reshape(case.scale.shape[0], -1, 1, 1)
        sh = case.shift.numpy().reshape(case.shift.shape[0], -1, 1, 1)
    g = oracle.gather(x, s.R, s.R, idx, sc, sh, "swish" if s.act == 1 else "identity", False)
    w = case.w.numpy()
    b = None if case.bias is None else case.bias.numpy()
    tiles = oracle.conv2d_tiles(g, w, b, (s.stride, s.stride))
    y0 = _nchw(case.dst)
    res = None if case.residual is None else _nchw(case.residual)
    if not s.shortcut:
        return oracle.scatter(tiles, y0, s.off, s.off, s.stride, s.stride, idx, res)
    flagged = case.sc_flags.numpy() != 0 if case.sc_flags is not None else np.ones(idx.shape[0], bool)
    idx1 = np.ascontiguousarray(idx[flagged] + s.off)                 # the shortcut's own 4x4 tiles, output frame
    x2 = np.concatenate([_nchw(t) for t in case.src2], 1)
    sc_tiles = oracle.conv2d_tiles(oracle.gather(x2, 4, 4, idx1), case.w2.numpy(), case.bias2.numpy())
    return oracle.scatter_with_block_residual(tiles, y0, sc_tiles, res, s.off, s.off, s.stride, s.stride, idx, idx1)


@pytest.mark.parametrize("spec", ORACLE_CASES, ids=lambda s: s.name)
def test_reference_matches_oracle(oracle, spec):
    case = tcc.make_case(spec, torch.float32, "cpu")
    (dst,) = tcc.reference(case)
    want = _oracle_composite(oracle, case)
    got = dst.want.permute(0, 3, 1, 2).numpy()
    assert float(np.abs(got - want).max()) <= 1e-6 * float(np.abs(want).max())
    # the written set is exactly what the oracle changed (plus elements a write left equal, which random data makes unlikely)
    changed = want != _nchw(case.dst)
    assert np.array_equal(changed, dst.written.permute(0, 3, 1, 2).numpy())
    if spec.c_div_tile:     # the (-1, -1) tile writes outputs (0..1, 0..1): C division of the origin
        assert bool(dst.written[0, :2, :2].all())


def test_split_halo_fills_restatement():
    """Hand-worked points of the kernel's K partition: 256 -> 64 (12 ring steps of 3 taps) at ksplit 2 is [0, 6) and [6, 12),
    two chunks each; at ksplit 8 the slices are one or two steps of one chunk."""
    assert tcc.split_halo_fills(256, 0, 2) == 2
    assert tcc.split_halo_fills(256, 0, 8) == 1
    assert tcc.split_halo_fills(64, 0, 2) == 1            # 3 steps: [0, 1) and [1, 3), both in chunk 0
    assert tcc.split_halo_fills(64, 64, 4) == 1           # 3 main steps + 1 shortcut step, one per rank
    assert tcc.split_halo_fills(256, 256, 8) == 2         # 16 steps: [2, 4) spans chunks 0 and 1
    assert tcc.split_halo_fills(128, 0, 4) == 1           # 6 steps: [1, 3) and [4, 6) each stay in one chunk
    assert tcc.split_halo_fills(384, 0, 4) == 2           # 18 steps: [4, 9) spans chunks 1 and 2 (the segment boundary at 128)


def _table_plans():
    out = []
    for spec in tcc.CASES:
        case = tcc.make_case(spec, torch.float16, "cpu")
        for dtype in (torch.float16, torch.bfloat16):
            case.dtype = dtype
            for i, ks in enumerate(spec.ksplits):
                d = tcc.descriptor(case, ks, tcc.TC5)
                plan = tcc.plan_of(d)
                out.append((spec, dtype, i, ks, plan, tcc.instantiation(spec, dtype, plan)))
    return out


@pytest.fixture(scope="module")
def table_plans(cabi_lib):
    return _table_plans()


def test_case_plans_are_the_intended_ones(table_plans):
    for spec, dtype, i, ks, plan, key in table_plans:
        assert key == tcc.intended(spec, dtype, i), "%s %s ksplit %d: plan %s -> %s, intended %s" % (
            spec.name, tcc.DTYPE_NAME[dtype], ks, tcc.plan_str(plan), key, tcc.intended(spec, dtype, i))
        if key is not None:
            assert plan.ksplit == spec.expect[i][1]


def test_case_table_reaches_every_instantiation(table_plans):
    keys = {key for *_, key in table_plans if key is not None}
    assert len(tcc.ALL_INSTANTIATIONS) == 26
    assert sorted(keys) == tcc.ALL_INSTANTIATIONS, "missing: %s" % sorted(set(tcc.ALL_INSTANTIATIONS) - keys)


def test_case_table_covers_every_feature_wide_and_narrow(table_plans):
    seen = set()
    for spec, _, i, _, plan, key in table_plans:
        form = "mma.sync" if key is None else ("wide" if plan.bn == 128 else "narrow")
        seen |= {(f, form) for f in tcc.features(spec)}
    both = ["per_sample_affine", "shared_affine", "residual", "two_aux", "aux_only", "shortcut_flags", "shortcut_all_tiles",
            "shortcut_two_sources", "upsampled_source", "two_sources", "channel_windows", "per_image_lists", "padded"]
    required = {(f, form) for f in both for form in ("wide", "narrow")}
    required |= {("stride2", "narrow"), ("stride2", "mma.sync"), ("per_sample_affine", "narrow")}
    assert required <= seen, "not covered: %s" % sorted(required - seen)


def test_case_table_sizes_do_not_depend_on_the_h100_variant():
    """Wide cases keep BN = 128 down to 132 SMs' worth of wide CTAs; narrow ones stay at <= 100 narrow CTAs (below any
    H100's SM count), so the intended plan holds on every H100."""
    for spec in tcc.CASES:
        m_blocks = -(-spec.B * spec.N // (32 if spec.stride == 2 else 8))
        for e in spec.expect:
            if e is None:
                continue
            if e[0] == 128:
                assert m_blocks * spec.Cout // 128 >= 132, spec.name
            else:
                assert m_blocks * spec.Cout // 64 <= 100, spec.name


@pytest.mark.parametrize("spec", tcc.CASES, ids=lambda s: s.name)
def test_case_lists_are_well_formed(spec):
    """Distinct origins per image, tiles that overhang the top / left border (6x6 halo tiles start at -1), padding only at the
    tail, and shortcut flags of both values.  (reference() itself asserts that no output pixel is written twice.)"""
    case = tcc.make_case(spec, torch.float16, "cpu")
    idx = case.idx.numpy().reshape(spec.B if spec.per_image else 1, spec.N, 2)
    for b, n in enumerate(spec.counts):
        real = idx[b, :n]
        assert len({tuple(r) for r in real}) == n and (idx[b, n:] == tcc.TILE_NONE).all()
        assert real.min() < 0 or spec.stride == 2 or spec.k == 1
    if spec.shortcut and spec.sc_flags:
        f = case.sc_flags.numpy()
        assert f.min() == 0 and f.max() == 1
