"""CPU checks of tests/step_kernel_contracts.py: each float64 restatement against an independent computation (torch's softmax and
scaled_dot_product_attention, the plain SPADE formula, the in-tree C oracle of the tile ops), the case tables against the
launchers' predicates, and the C-ABI refusals that come before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import kernel_contracts as kc
import step_kernel_contracts as sk

F64 = torch.float64
P = 0x10000                     # not device memory: a launch would fault, so these calls must fail on their arguments


def _window(e: kc.Expect, t: torch.Tensor) -> torch.Tensor:
    return t[e.g.off:e.g.off + e.g.view.numel()].view(*e.g.view.shape)


def _outside_untouched(e: kc.Expect):
    assert not e.written[:e.g.off].any() and not e.written[e.g.off + e.g.view.numel():].any()
    assert torch.allclose(e.want[~e.written], e.g.flat.double()[~e.written], rtol=0, atol=0, equal_nan=True)


# ---------------------------------------------------------------------------------------------------------------- attention
def _sattn_cpu_specs():
    """One case per layout x mode where the table has one at a size the CPU takes in a moment, and the single-key cases."""
    picked, seen = [], set()
    for s in sk.SATTN_CASES:
        key = (s.layout, s.mode, s.dom)
        if key in seen or s.B * s.heads * s.Nq * s.Nk > 600000:
            continue
        seen.add(key)
        picked.append(s)
    return picked + [s for s in sk.SATTN_CASES if s.Nk == 1]


@pytest.mark.parametrize("spec", _sattn_cpu_specs(), ids=lambda s: s.name)
def test_sparse_attention_restatement_matches_softmax_and_sdpa(spec):
    """float64 operands: the restatement's values are softmax(scale q k^T) v and F.scaled_dot_product_attention to 1e-12; it
    writes exactly the D real columns of every (b, head, query); the padding columns after each head stay as they were."""
    case = sk.make_sattn(spec, F64, "cpu")
    (e,) = sk.sattn_reference(case)
    q, k, v = case.q, case.k, case.v
    sc = spec.s32
    want_sm = torch.softmax(sc * q @ k.transpose(2, 3), dim=-1) @ v
    want_sdpa = F.scaled_dot_product_attention(q.contiguous(), k.contiguous(), v.contiguous(), scale=sc)
    wv, wr =_window(e, e.want), _window(e, e.written)
    if case.out.layout == "bhnd":
        got, wr4 = wv, wr
    else:
        got, wr4 = wv[..., :spec.D].permute(0, 2, 1, 3), wr[..., :spec.D].permute(0, 2, 1, 3)
        assert not wr[..., spec.D:].any(), "the guard columns after each head are never written"
    assert bool(wr4.all())
    torch.testing.assert_close(got, want_sm, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(got, want_sdpa, rtol=1e-12, atol=1e-12)
    _outside_untouched(e)
    # the values are what the mode promises
    logits = sc * (q @ k.transpose(2, 3))
    if spec.mode == "flat":
        assert bool((logits == 0).all())
    elif spec.mode == "dominant":
        assert bool((logits.argmax(dim=-1) == spec.dom_key).all())
        top2 = logits.topk(2, dim=-1).values
        assert float((top2[..., 0] - top2[..., 1]).min()) > 9
    elif spec.mode == "rising":
        bm = F.pad(logits, (0, spec.blocks * sk.BNK - spec.Nk), value=-1e9).unflatten(-1, (spec.blocks, sk.BNK)).amax(-1)
        assert float((bm[..., 1:] - bm[..., :-1]).min()) > 4
    elif spec.mode == "falling":
        assert bool((logits.argmax(dim=-1) < sk.BNK).all())
    elif spec.mode == "large":
        assert 60 < float(logits.abs().max()) <= 80.5
    elif spec.mode == "constant_v":
        assert bool((v == v[:, :, :1]).all())
        assert torch.allclose(got, v[:, :, :1].expand_as(got), rtol=1e-12, atol=1e-12)


def test_sparse_attention_layouts_hold_the_same_values():
    """bnhd and kv_pair address the same [B, heads, N, D] values as bhnd, and the descriptor's strides are 0 on size-1 dims."""
    spec = next(s for s in sk.SATTN_CASES if s.name == "d40_q200_k77_kvpair_scale")
    cases = {lay: sk.make_sattn(spec, torch.float16, "cpu", layout=lay) for lay in sk.LAYOUTS}
    for lay in ("bnhd", "kv_pair"):
        for t in ("q", "k", "v"):
            assert torch.equal(getattr(cases[lay], t), getattr(cases["bhnd"], t)), (lay, t)
    c = cases["bnhd"]
    assert c.q.stride() == (spec.Nq * spec.heads * (spec.D + 8), spec.D + 8, spec.heads * (spec.D + 8), 1)
    assert cases["kv_pair"].v.data_ptr() - cases["kv_pair"].k.data_ptr() == spec.heads * spec.D * 2
    one = next(s for s in sk.SATTN_CASES if s.name == "d80_q1_k1_bnhd")
    d = sk.sattn_descriptor(sk.make_sattn(one, torch.float16, "cpu"))
    assert all(list(getattr(d, n)) == [0, 0, 0] for n in ("q_stride", "k_stride", "v_stride", "out_stride"))
    assert all(getattr(d, n)[i] % 8 == 0 for n in ("q_stride", "k_stride", "v_stride", "out_stride") for i in range(3))


def test_sparse_attention_bound_is_honest_and_tight():
    """The bound covers the output's rounding and the uncentred P rounding (u sum_j s_j |v_j|) and little else where the
    softmax is not peaked: within a small multiple of u (|want| + sum_j s_j |v_j|)."""
    for name in ("d40_q65_k130_constant_v", "d64_q63_k63_random_bhnd", "d80_q65_k1024_large"):
        spec = next(s for s in sk.SATTN_CASES if s.name == name)
        for dt in (torch.float16, torch.bfloat16):
            case = sk.make_sattn(spec, dt, "cpu")
            (e,) = sk.sattn_reference(case)
            u = kc.ROUNDOFF[dt]
            want, bound = _window(e, e.want), _window(e, e.bound)
            p = torch.softmax(spec.s32 * case.q.double() @ case.k.double().transpose(2, 3), -1)
            mag = p @ case.v.double().abs()
            ratio = bound / (u * (want.abs() + mag))
            assert float(ratio.min()) >= 1 and float(ratio.max()) < (8 if spec.mode != "large" else 40), (name, dt, float(ratio.max()))


def test_sparse_attention_case_table_covers_every_instantiation():
    cases = sk.SATTN_CASES
    for D in sk.HEAD_DIMS:
        mine = [s for s in cases if s.D == D]
        assert any(s.blocks == 1 for s in mine) and any(s.blocks > 1 for s in mine), D
        assert any(s.Nk % sk.BNK for s in mine if s.blocks > 1), "a multi-block case with a key tail at D = %d" % D
        assert any(s.Nq % sk.BM for s in mine), "a query tail at D = %d" % D
        assert {"bhnd", "bnhd", "kv_pair"} <= {s.layout for s in mine}
    assert [D for D in sk.HEAD_DIMS if sk.sattn_padded(D) != D] == [40], "D = 40 is the one padded head dim"
    assert sk.sattn_padded(80) // 16 == 5
    assert {1, 63, 64, 65, 200} <= {s.Nq for s in cases}
    assert {1, 63, 64, 65, 77, 130, 1024, 4096} <= {s.Nk for s in cases}
    assert set(sk.MODES) == {s.mode for s in cases}
    dom = [s for s in cases if s.mode == "dominant"]
    assert any(s.dom == "first" and s.blocks > 1 for s in dom)
    assert any(s.dom == "last" and s.Nk % sk.BNK and s.blocks > 1 for s in dom), "the dominant key in the last, partial block"
    assert any(s.scale is None and s.D ** -0.5 == 2.0 ** round(np.log2(s.D ** -0.5)) for s in cases)
    assert any(s.scale is not None and float(np.log2(s.scale)) % 1 for s in cases), "a scale that is not a power of two"
    assert any(s.B == 1 for s in cases) and any(s.heads == 1 for s in cases) and any(s.B * s.heads > 4 for s in cases)
    assert all(s.B * s.heads <= 2 for s in cases if s.Nk >= 4000), "B * heads stays small where Nk is large"


WIDE_SMS = kc.H100_SMS


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("spec", sk.WIDE_CASES, ids=lambda s: s.name)
def test_wide_kernel_emulation_stays_within_the_wide_bound(spec, dtype):
    """The wide kernel's arithmetic emulated in float32 (sk.wide_sattn_emulate: 32-key blocks, the cluster's key ranges, the
    merge) is within sk.wide_sattn_reference's bound everywhere, and its values are softmax(scale q k^T) v."""
    case = sk.make_sattn(spec, dtype, "cpu")
    (e,) = sk.wide_sattn_reference(case, WIDE_SMS, chunk=4)
    (old,) = sk.sattn_reference(case, chunk=4)
    got = sk.wide_sattn_emulate(case, WIDE_SMS)
    view = (lambda t: _window(e, t)) if spec.layout == "bhnd" else (lambda t: _window(e, t)[..., :spec.D].permute(0, 2, 1, 3))  # noqa: E731
    want, bound, old_bound = view(e.want), view(e.bound), view(old.bound)
    err = (got - want).abs()
    r, r_old = float((err / bound).max()), float((err / old_bound).max())
    print("[wide restatement] %s %s cs=%d: emulation |err| / bound %.3f, / the 64-key bound %.3f"
          % (spec.name, str(dtype)[6:], sk.wide_cluster(spec.Nq, spec.Nk, spec.B * spec.heads, WIDE_SMS),
             r, r_old))
    assert r <= 1.0, (spec.name, r)
    sm = torch.softmax(spec.s32 * case.q.double() @ case.k.double().transpose(2, 3), -1) @ case.v.double()
    torch.testing.assert_close(want, sm, rtol=1e-12, atol=1e-12)


def test_wide_bound_is_honest_and_tight():
    """As test_sparse_attention_bound_is_honest_and_tight, for the wide kernel's bound: at least the output's and P's rounding,
    and within a small multiple of u (|want| + sum_j s_j |v_j|) where the softmax is not peaked."""
    for name in ("q63_k65_bnhd", "q64_k4096_constant_v", "b2_q65_k130_bnhd", "b2h2_q64_k1000_cs8"):
        spec = next(s for s in sk.WIDE_CASES if s.name == name)
        for dt in (torch.float16, torch.bfloat16):
            case = sk.make_sattn(spec, dt, "cpu")
            (e,) = sk.wide_sattn_reference(case, WIDE_SMS, chunk=4)
            u = kc.ROUNDOFF[dt]
            want, bound = _window(e, e.want), _window(e, e.bound)
            if spec.layout != "bhnd":
                want, bound = want[..., :spec.D].permute(0, 2, 1, 3), bound[..., :spec.D].permute(0, 2, 1, 3)
            p = torch.softmax(spec.s32 * case.q.double() @ case.k.double().transpose(2, 3), -1)
            mag = p @ case.v.double().abs()
            ratio = bound / (u * (want.abs() + mag))
            assert float(ratio.min()) >= 1 and float(ratio.max()) < 8, (name, dt, float(ratio.max()))


def test_wide_case_table_covers_the_cluster_split():
    """At 132 SMs: cluster sizes 1, 2, 4 and 8, one of size 1 over several blocks; a range boundary inside the falling and the
    dominant patterns; B * heads > 1 with a split; a multi-block key range ending in a partial 32-key block."""
    cases = sk.WIDE_CASES
    cs = {s.name: sk.wide_cluster(s.Nq, s.Nk, s.B * s.heads, WIDE_SMS) for s in cases}
    assert {1, 2, 4, 8} <= set(cs.values())
    assert any(cs[s.name] == 1 and s.Nk > sk.WIDE_BNK for s in cases)
    for mode in ("falling", "dominant"):
        assert any(s.mode == mode and cs[s.name] > 1 for s in cases), mode
    assert any(s.B * s.heads > 1 and cs[s.name] > 1 for s in cases)
    assert any(s.Nk % sk.WIDE_BNK and s.Nk > sk.WIDE_BNK for s in cases)
    assert all(s.D == sk.WIDE_D for s in cases) and {"bhnd", "bnhd"} <= {s.layout for s in cases}
    # every range holds at least one block, and the ranges tile the blocks
    for s in cases:
        r = sk.wide_ranges(s.Nk, cs[s.name])
        assert r[0][0] == 0 and r[-1][1] == -(-s.Nk // sk.WIDE_BNK) and all(t1 > t0 for t0, t1 in r)
        assert all(a[1] == b[0] for a, b in zip(r, r[1:]))
    for s in cases:                  # a case named for its cluster size has that size
        named = [int(p[2:]) for p in s.name.split("_") if p.startswith("cs") and p[2:].isdigit()]
        assert named in ([], [cs[s.name]]), (s.name, cs[s.name])
    assert sk.wide_cluster(64, 4096, 1, 132) == 8 and sk.wide_cluster(64 * 132, 4096, 1, 132) == 1 and sk.wide_cluster(65, 65, 1, 132) == 2


def test_sparse_attention_refuses_a_scale_that_is_not_positive_and_finite(cabi_lib):
    """The header documents scale > 0; the entry point refuses anything else before it touches the device."""
    from sige_b200 import _cabi

    lib = _cabi.lib()
    spec = next(s for s in sk.SATTN_CASES if s.name == "d40_q65_k130_constant_v")
    d = _cabi.SparseAttention()
    d.q = d.k = d.v = d.out = P
    d.B, d.heads, d.Nq, d.Nk, d.D, d.dtype = spec.B, spec.heads, spec.Nq, spec.Nk, spec.D, _cabi.F16
    for bad in (0.0, -spec.s32, float("nan"), float("inf")):
        d.scale = bad
        assert lib.sige_sparse_attention(ctypes.byref(d), None) != 0
        assert b"must be positive and finite" in lib.sige_last_error(), bad


# ---------------------------------------------------------------------------------------------------------------- SPADE
@pytest.mark.parametrize("spec", [s for s in sk.SPADE_CASES if s.pixels < 10000], ids=lambda s: s.name)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=["f32", "f16", "bf16"])
def test_spade_restatement_matches_the_formula(spec, dtype):
    """leaky_relu(x * (1 + gamma) + beta, slope) in float64 on the stored operands, to the fp32 rounding of 1 + gamma; only the C
    channels of each pixel of out are written; identity cases are x itself."""
    case = sk.make_spade(spec, dtype, "cpu")
    (e,) = sk.spade_reference(case)
    x, g, b = case.x.double(), case.gamma.double(), case.beta.double()
    f = x * (1 + g) + b
    want = torch.where(f > 0, f, f * spec.slope)
    w, wr = _window(e, e.want), _window(e, e.written)
    C = case.C
    assert bool(wr[:, :C].all()) and not wr[:, C:].any()
    torch.testing.assert_close(w[:, :C], want, rtol=1e-6, atol=1e-7)
    _outside_untouched(e)
    if spec.identity:
        assert torch.equal(w[:, :C], x) and not bool(_window(e, e.bound).any())
    # the fp32 arithmetic restated: a value within the bound everywhere, the fmaf of the fp32 values
    if dtype == torch.float32:
        f32 = torch.addcmul(case.beta, case.x, 1 + case.gamma)
        alt = torch.where(f32 > 0, f32, f32 * np.float32(spec.slope))
        assert bool(((alt.double() - w[:, :C]).abs() <= _window(e, e.bound)[:, :C]).all())


def test_spade_case_table_covers_the_launch():
    cases = sk.SPADE_CASES
    for dt in (torch.float32, torch.float16):
        assert {sk.SPADE_VEC[dt], 64, 256} <= {s.channels(dt) for s in cases}
    assert {1.0, 0.2, 0.0} <= {s.slope for s in cases} and 1 in {s.pixels for s in cases}
    assert any(s.identity for s in cases)
    for dt in (torch.float32, torch.float16, torch.bfloat16):
        multi = [s for s in cases if sk.spade_iterations(s.pixels * s.channels(dt) // sk.SPADE_VEC[dt], kc.H100_SMS) > 1]
        assert multi, "a grid-stride loop that runs more than once at 132 SMs (%s)" % dt
    assert sk.spade_blocks(16 * 132 * 256 - 255, 132) == 16 * 132 - 1 + 1 and sk.spade_blocks(16 * 132 * 256, 132) == 16 * 132


def test_spade_refuses_misaligned_buffers_and_strides(cabi_lib):
    from sige_b200 import _cabi

    lib = _cabi.lib()
    for dt, vec in ((_cabi.F32, 4), (_cabi.F16, 8), (_cabi.BF16, 8)):
        ok = dict(xs=2 * vec, gs=2 * vec, bs=2 * vec, os=vec, C=vec)
        for k in ("xs", "gs", "bs", "os", "C"):
            a = dict(ok)
            a[k] += 2
            assert lib.sige_spade_modulate(P, a["xs"], P, a["gs"], P, a["bs"], P, a["os"], 5, a["C"], 0.2, dt, None) != 0
            assert b"multiples of %d elements" % vec in lib.sige_last_error(), (dt, k)
        for i in range(4):
            ptrs = [P] * 4
            ptrs[i] += 4 if dt == _cabi.F32 else 2
            assert lib.sige_spade_modulate(ptrs[0], ok["xs"], ptrs[1], ok["gs"], ptrs[2], ok["bs"], ptrs[3], ok["os"], 5, vec, 0.2, dt, None) != 0
            assert b"16-byte aligned" in lib.sige_last_error(), (dt, i)


# ---------------------------------------------------------------------------------------------------------------- tile ops
def _np(t):
    return None if t is None else t.detach().float().numpy()


def _oracle_out(case: sk.TileCase, oracle) -> torch.Tensor:
    """The oracle's result (NCHW fp32) for the case's fp32 inputs."""
    s = case.spec
    idx = case.idx["idx"].numpy()
    L = lambda n: _np(case.logical(n))                                                    # noqa: E731
    act = "swish" if s.act else "identity"
    if s.op == "gather":
        x = case.logical("x")
        if s.up:
            x = x.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
        return torch.from_numpy(oracle.gather(_np(x), 6, 6, idx, _np(case.bc.get("scale")), _np(case.bc.get("shift")), act, s.act_first))
    Ro, off = s.geometry
    if s.op == "scatter":
        y = _np(case.logical("out")) if s.inplace else L("y")
        return torch.from_numpy(oracle.scatter(L("x"), y, off, off, s.stride, s.stride, idx, _np(case.bc.get("residual"))))
    if s.op == "scatter_gather":
        m = oracle.get_scatter_map(s.H, s.W, 6, 6, 3, 3, 1, 1, 1, 1, idx)
        assert np.array_equal(m, case.idx["map"].numpy()), "the restated scatter map differs from the oracle's"
        return torch.from_numpy(oracle.scatter_gather(L("x"), L("y"), 6, 6, idx, m, _np(case.bc.get("scale")), _np(case.bc.get("shift")),
                                                      act, s.act_first))
    return torch.from_numpy(oracle.scatter_with_block_residual(L("x"), L("y"), L("x1"), L("y1"), off, off, s.stride, s.stride, idx,
                                                               case.idx["idx1"].numpy()))


@pytest.mark.parametrize("spec", sk.TILE_CASES, ids=lambda s: s.name)
def test_tile_op_restatement_matches_the_oracle(spec, oracle):
    """fp32 inputs: the restatement equals the C oracle bitwise on identity moves and to 1e-6 with affine / swish / residual
    arithmetic.  The oracle has no lower bound check on pasted positions, so the tiles pasted above or left of the image are
    left out here (test_tile_op_geometries_reach_the_edges keeps them in the GPU cases)."""
    case = sk.make_tile(spec, torch.float32, "cpu", oracle_safe=True)
    (e,) = sk.tile_reference(case)
    perm = (lambda t: t.permute(0, 3, 1, 2)) if spec.layout == "nhwc" else (lambda t: t)   # noqa: E731
    want, written = perm(_window(e, e.want)), perm(_window(e, e.written))
    ref = _oracle_out(case, oracle).double()
    if spec.op == "scatter" and spec.inplace:
        assert written.any() and not written.all()
        want, ref = want[written], ref[written]
    else:
        assert bool(written.all())
    if spec.identity:
        assert torch.equal(kc.bits(want.float()), kc.bits(ref.float())), spec.name
        assert not bool(e.bound.any())
    else:
        torch.testing.assert_close(want, ref, rtol=1e-6, atol=1e-6)
    _outside_untouched(e)


def test_tile_op_case_table_covers_every_path():
    cases = sk.TILE_CASES
    for op in sk.TILE_OPS:
        mine = [s for s in cases if s.op == op]
        for dt in (torch.float32,) + sk.F16_BF16:
            vec = 16 // sk._esize(dt)
            assert {sk.tile_path(s, dt) for s in mine} == {"nchw", "vec", "scalar"}, (op, dt)
            scal = [s for s in mine if sk.tile_path(s, dt) == "scalar"]
            assert any(s.C % vec for s in scal) and any(s.misalign and s.C % vec == 0 for s in scal), (op, dt)
    g = [s for s in cases if s.op == "gather"]
    assert any(s.up for s in g) and {sk.tile_path(s, torch.float16) for s in g if s.up} == {"nchw", "vec", "scalar"}
    for name in ("scale", "shift"):
        for adt in ("f32", "x"):
            assert {getattr(s, name) for s in g if s.aff_dt == adt} >= set(sk.BCAST_SHAPES), (name, adt)
    assert {(s.act, s.act_first) for s in g if s.scale or s.shift} == {(0, False), (1, False), (1, True)}
    assert any(s.act and not s.scale and not s.shift for s in g)
    sc = [s for s in cases if s.op == "scatter"]
    assert {s.residual for s in sc} >= set(sk.BCAST_SHAPES)
    assert any(s.inplace for s in sc) and any(not s.inplace for s in sc)
    assert {sk.tile_path(s, torch.float16) for s in sc if s.inplace} == {"nchw", "vec", "scalar"}
    assert any(s.stride == 2 for s in sc) and any(s.op == "scatter_gather" and s.act for s in cases)


def test_tile_op_misalignment_is_one_element_in_every_dtype():
    """A misaligned destination sits one whole element (4 bytes for f32, 2 for 16 bits) off 16-byte alignment, so f32 takes
    the scalar NHWC path too; the inputs stay aligned and hold the same values."""
    spec = next(s for s in sk.TILE_CASES if s.name == "s_nhwc_scalar_misaligned_copy")
    for dt in (torch.float32,) + sk.F16_BF16:
        case = sk.make_tile(spec, dt, "cpu")
        es = sk._esize(dt)
        assert case.out.view.data_ptr() % 16 == es and sk.tile_path(spec, dt) == "scalar", dt
        assert all(t.data_ptr() % 16 == 0 for t in case.t.values())


def test_f32_swish_bound_is_the_accurate_one():
    """The f32 tile ops evaluate swish as z / (1 + expf(-z)) with an IEEE division: a float32 evaluation of that formula is
    within SWISH_ACCURATE_REL of z sigmoid(z), which is tighter than the fast intrinsics' swish_rel everywhere."""
    z = torch.linspace(-30, 30, 200001, dtype=torch.float32)
    y32 = z / (1 + torch.exp(-z))
    y = z.double() * torch.sigmoid(z.double())
    assert bool(((y32.double() - y).abs() <= sk.SWISH_ACCURATE_REL * y.abs() + sk.HALF_SUBNORMAL[torch.float32]).all())
    assert bool((sk.swish_rel(z.double()) > 2 * sk.SWISH_ACCURATE_REL).all())
    _, err32 = sk.affine_act_bound(z.double(), None, None, sk.ACT_SWISH, False, torch.float32)
    _, err16 = sk.affine_act_bound(z.double(), None, None, sk.ACT_SWISH, False, torch.float16)
    assert torch.equal(err32, sk.SWISH_ACCURATE_REL * y.abs()) and bool((err16 > err32)[y != 0].all())


def test_tile_op_geometries_reach_the_edges():
    """Tiles stick out of the image on every side; stride-2 origins -1 and -2 land on rows 0 and -1 (C division truncates)."""
    assert sk._cdiv(-1, 2) == 0 and sk._cdiv(-2, 2) == -1 and sk._cdiv(-3, 2) == -1 and sk._cdiv(5, 2) == 2
    for s in sk.TILE_CASES:
        case = sk.make_tile(s, torch.float16, "cpu")
        o = case.idx["idx"].long()
        R = 6 if s.op in ("gather", "scatter_gather") else s.geometry[0]
        if s.op in ("gather", "scatter_gather"):
            assert bool((o < 0).any()) and bool(((o[:, 0] + R > s.H) | (o[:, 1] + R > s.W)).any()), s.name
        if s.stride == 2:
            assert {-1, -2} <= set(o.flatten().tolist()), s.name
