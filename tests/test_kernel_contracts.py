"""CPU checks of tests/kernel_contracts.py: each float64 restatement against an independent computation, the case tables against
the kernels' branch predicates, and the C-ABI refusals that come before any CUDA call."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import kernel_contracts as kc

F64 = torch.float64


def _window(e: kc.Expect, t: torch.Tensor) -> torch.Tensor:
    """The window of a flat expectation tensor, in the buffer's shape."""
    return t[e.g.off:e.g.off + e.g.view.numel()].view(*e.g.view.shape)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else kc.H100_SMS


# ---------------------------------------------------------------------------------------------------------------- separable
def _sep_dense(case: kc.SepCase, i: int) -> torch.Tensor:
    """Branch i on the whole destination of a buffer-source case: depthwise F.conv2d(groups=Cin) on the source padded by the
    output offset (out[p] reads x[p - off .. p - off + 2]), then a 1x1 F.conv2d; NCHW [B, Cout, dH, dW]."""
    s = case.spec
    x = case.src[..., s.pre:s.pre + s.Cin].permute(0, 3, 1, 2).double()
    xp = F.pad(x, (s.offW, 8, s.offH, 8))
    a = F.conv2d(xp, case.dw_w[i].double().view(s.Cin, 1, 3, 3), None if case.dw_b[i] is None else case.dw_b[i].double(), groups=s.Cin)
    a = a[:, :, :s.dh, :s.dw]
    return F.conv2d(a, case.pw_w[i].double().view(s.Cout, s.Cin, 1, 1), None if case.pw_b[i] is None else case.pw_b[i].double())


def _sep_rows(case: kc.SepCase, i: int) -> torch.Tensor:
    """Branch i on every row of a stack-source case, by F.conv2d: [B*N, Cout, 4, 4]."""
    s = case.spec
    x = case.src[..., s.pre:s.pre + s.Cin].permute(0, 3, 1, 2).double()
    a = F.conv2d(x, case.dw_w[i].double().view(s.Cin, 1, 3, 3), None if case.dw_b[i] is None else case.dw_b[i].double(), groups=s.Cin)
    return F.conv2d(a, case.pw_w[i].double().view(s.Cout, s.Cin, 1, 1), None if case.pw_b[i] is None else case.pw_b[i].double())


def _sep_written_by_loops(case: kc.SepCase, i: int) -> torch.Tensor:
    """bool mask of the destination window's pixels the launch writes, tile by tile in plain Python."""
    s = case.spec
    kind = s.dsts[i][0]
    rows = [(0, 0)] * s.N if case.idx is None else [tuple(r) for r in case.idx.tolist()]
    shape = (s.B * s.N, 4, 4) if kind == "stack" else (s.B, s.dh, s.dw)
    m = torch.zeros(shape, dtype=torch.bool)
    for b in range(s.B):
        for n, (h, w) in enumerate(rows):
            if h == kc.TILE_NONE:
                continue
            if kind == "stack":
                m[b * s.N + n] = True
                continue
            for oy in range(4):
                for ox in range(4):
                    hh, ww = h + s.offH + oy, w + s.offW + ox
                    if 0 <= hh < s.dh and 0 <= ww < s.dw:
                        m[b, hh, ww] = True
    return m


SEP_CPU = ["borders_lastwin_b3", "cin16_cout8", "cout72_partial_block", "stack_src_b2", "mixed_stack_buf", "mixed_buf_stack_stacksrc",
           "offH2_offW0_dst_extent", "no_biases", "stack_to_stack_no_list", "sm48_96_b3"]


@pytest.mark.parametrize("name", SEP_CPU)
def test_separable_restatement_matches_conv2d(name):
    """float64 case: the restatement's written set is the tiles' in-destination outputs (padding entries write nothing, to a
    stack as to a buffer), its values are F.conv2d(groups=Cin) -> 1x1 F.conv2d, and nothing else of any buffer changes."""
    spec = next(s for s in kc.SEP_CASES if s.name == name)
    case = kc.make_sep(spec, F64, "cpu")
    for i, e in enumerate(kc.sep_reference(case)):
        kind, extra, c0 = spec.dsts[i]
        written, want = _window(e, e.written), _window(e, e.want)
        m = _sep_written_by_loops(case, i)
        assert torch.equal(written[..., c0:c0 + spec.Cout], m[..., None].expand(*m.shape, spec.Cout)), "%s dst%d written set" % (name, i)
        assert not written[..., :c0].any() and not written[..., c0 + spec.Cout:].any()
        assert not e.written[:e.g.off].any() and not e.written[e.g.off + e.g.view.numel():].any()
        assert torch.equal(e.want[~e.written], case.dst[i].flat.double()[~e.written])
        if kind == "stack":
            ref = _sep_rows(case, i).permute(0, 2, 3, 1)                                # [B*N, 4, 4, Cout]
            if not spec.src_stack:
                continue                                                                # (buffer source to a stack: covered on the GPU)
        else:
            if spec.src_stack:
                # stack source to a buffer: paste each real row's 4x4 outputs at its origin + off
                rows = _sep_rows(case, i).permute(0, 2, 3, 1)
                ref = torch.zeros(spec.B, spec.dh, spec.dw, spec.Cout, dtype=F64)
                for t, (h, w) in enumerate(case.idx.tolist() * spec.B):
                    if h == kc.TILE_NONE:
                        continue
                    for oy in range(4):
                        for ox in range(4):
                            hh, ww = h + spec.offH + oy, w + spec.offW + ox
                            if 0 <= hh < spec.dh and 0 <= ww < spec.dw:
                                ref[t // spec.N, hh, ww] = rows[t, oy, ox]
            else:
                ref = _sep_dense(case, i).permute(0, 2, 3, 1)
        got = want[..., c0:c0 + spec.Cout][m]
        assert torch.allclose(got, ref[m], rtol=1e-12, atol=1e-12), "%s dst%d: %.3g" % (name, i, float((got - ref[m]).abs().max()))


def test_per_image_separable_restatement_is_each_image_on_its_own_list():
    """Per-image lists (row b*N + i a tile of image b): image b's part of the restatement is the shared-list restatement of a
    one-image case whose list is rows [b*N, (b+1)*N); an image whose list is all SIGE_TILE_NONE is left as it was."""
    import dataclasses

    spec = kc.SepSpec("pi_cpu", B=3, Cin=16, Cout=24, H=18, W=22, real=9, lead=9, tail=5, pre=16, per_image=True, seed=7)
    case = kc.make_sep(spec, F64, "cpu")
    rows = []
    for b, n in enumerate((9, 0, 4)):
        tiles = [t for t in kc.sep_tile_list(spec, np.random.default_rng(40 + b)) if t[0] != kc.TILE_NONE]
        rows += tiles[:n] + [(kc.TILE_NONE, kc.TILE_NONE)] * (spec.N - n)
    case.idx = torch.tensor(rows, dtype=torch.int32)
    s1 = dataclasses.replace(spec, B=1, per_image=False)
    for i, e in enumerate(kc.sep_reference(case)):
        want, written, bound = (_window(e, t) for t in (e.want, e.written, e.bound))
        for b in range(spec.B):
            flats = [g.view[b:b + 1].clone() for g in case.dst]
            c1 = kc.SepCase(s1, F64, case.src[b:b + 1], case.idx[b * spec.N:(b + 1) * spec.N], case.dw_w, case.dw_b, case.pw_w,
                            case.pw_b, [kc.Guarded(f.reshape(-1), f, 0, "nhwc") for f in flats])
            e1 = kc.sep_reference(c1)[i]
            w1, m1, b1 = (t.view(flats[i].shape)[0] for t in (e1.want, e1.written, e1.bound))
            assert torch.equal(written[b], m1) and torch.equal(bound[b], b1), (i, b)
            assert torch.equal(want[b][m1], w1[m1]), (i, b)
            assert bool(m1.any()) == (b != 1), "the image without tiles is not written"


def test_separable_restatement_matches_the_descriptor_simulator():
    """The restatement against SeparableSim (tests/test_separable_conv.py), the simulator the lowering tests run on, in fp32."""
    from test_separable_conv import _sim_executors

    SeparableSim, _ = _sim_executors()
    for name in ("borders_lastwin_b3", "sm64_48_b3", "no_biases"):
        spec = next(s for s in kc.SEP_CASES if s.name == name)
        case = kc.make_sep(spec, torch.float32, "cpu")
        expects = kc.sep_reference(case)
        branches, outs = [], []
        for i in range(len(spec.dsts)):
            out = torch.zeros(spec.B, spec.Cout, spec.dh, spec.dw)
            outs.append(out)
            dw = SimpleNamespace(weight=case.dw_w[i].view(spec.Cin, 1, 3, 3), bias=case.dw_b[i], scale=None, shift=None)
            branches.append((dw, case.pw_w[i].view(spec.Cout, spec.Cin, 1, 1), case.pw_b[i], SimpleNamespace(raw=out)))
        rec = SimpleNamespace(src=case.src.permute(0, 3, 1, 2), c0=spec.pre, Cin=spec.Cin, idx=case.idx, src_stack=spec.src_stack,
                              batch=spec.B, branches=branches, off=spec.offH)
        SeparableSim().prepare_separable(rec)(0)
        for e, out in zip(expects, outs):
            w = _window(e, e.written)[..., :spec.Cout]
            got = out.permute(0, 2, 3, 1)[w].double()
            want = _window(e, e.want)[..., :spec.Cout][w]
            assert float((got - want).abs().max()) <= 1e-5 * float(want.abs().max()), name
            assert bool((out.permute(0, 2, 3, 1)[~w] == 0).all()), "%s: the simulator writes where the restatement does not" % name


def test_separable_case_table_covers_the_launch_paths():
    cases = kc.SEP_CASES
    assert any(s.B > 1 for s in cases)
    assert {16, 256} <= {s.Cin for s in cases}
    assert {8, 1024} <= {s.Cout for s in cases}
    assert any(s.Cout > 64 and s.Cout % 64 for s in cases), "a partial last 64-channel block"
    assert any(s.Cout // 64 >= 16 for s in cases), "grid.y = 16"
    assert any(s.offH != s.offW and (s.dh, s.dw) != (s.H, s.W) for s in cases)
    assert any(not s.dw_bias and not s.pw_bias for s in cases)
    assert any(len({k for k, _, _ in s.dsts}) == 2 for s in cases), "mixed destination kinds"
    assert any(s.src_stack and s.no_list for s in cases) and any(s.src_stack and not s.no_list for s in cases)
    assert any(not s.src_stack and s.pre and not s.post for s in cases), "the last channel window of a wider pixel"
    rng = np.random.default_rng(0)

    def whole_cta_of_padding(s):
        rows = kc.sep_tile_list(s, rng)
        return any(all(rows[(t0 + j) % s.N][0] == kc.TILE_NONE for j in range(8)) for t0 in range(0, s.B * s.N, 8)
                   if (t0 % s.N) + 8 <= s.N)

    assert any(whole_cta_of_padding(s) and s.B > 1 for s in cases) and any(whole_cta_of_padding(s) and s.B == 1 for s in cases)
    for s in cases:
        assert s.Cin % 16 == 0 and 16 <= s.Cin <= 256 and s.Cout % 8 == 0 and 8 <= s.Cout <= 1024
        assert s.src_C % 8 == 0 and s.pre % 8 == 0 and all(c0 % 8 == 0 and (s.Cout + extra) % 8 == 0 for _, extra, c0 in s.dsts)
        if s.no_list:
            assert s.src_stack and all(k == "stack" for k, _, _ in s.dsts) and s.pad_run == s.tail == 0


def test_separable_table_has_every_sub_mobile_layer():
    """Every (Cin, Cout, source kind) the full-size sub-mobile lowering emits on the descriptor simulator is a case, at B = 1
    and B = 3, with the source window and pixel width the lowering passes."""
    from test_separable_conv import _lower_on_sim

    step, _, _ = _lower_on_sim("full")
    emitted = {(r.Cin, r.Cout, r.src_stack, int(r.src.shape[1]), r.c0) for r in step.low.separable}
    assert len(step.low.separable) == 14
    table = {(s.Cin, s.Cout, s.src_stack, s.src_C, s.pre) for s in kc.SEP_CASES}
    kinds = {(ci, co, st) for ci, co, st, _, _ in emitted}
    assert kinds <= {(s.Cin, s.Cout, s.src_stack) for s in kc.SEP_CASES if s.B == 1}
    assert kinds <= {(s.Cin, s.Cout, s.src_stack) for s in kc.SEP_CASES if s.B == 3}
    assert {(ci, co) for ci, co, _, _, _ in emitted} == {(ci, co) for ci, co, _, _ in kc.SUB_MOBILE_LAYERS}
    assert all(any(e[:2] == t[:2] and e[2:4] == t[2:4] for t in table) for e in emitted)


# ---------------------------------------------------------------------------------------------------------------- conv_in
@pytest.mark.parametrize("spec", kc.CONV_IN_CASES, ids=lambda s: s.name)
def test_conv_in_restatement_matches_conv2d(spec):
    case = kc.make_conv_in(spec, F64, "cpu")
    x = case.x.permute(0, 3, 1, 2)
    v = F.conv2d(x, case.w, case.bias, padding=1).permute(0, 2, 3, 1)
    m = torch.zeros(spec.B, spec.H, spec.W, dtype=torch.bool)
    if spec.tiles is None:
        m[:] = True
    else:
        per_image, _, R, _ = spec.tiles
        rows = case.idx.tolist()
        for b in range(spec.B):
            for (h, w) in (rows[b * case.n_tiles:(b + 1) * case.n_tiles] if per_image else rows):
                if h != kc.TILE_NONE:
                    m[b, max(h, 0):max(min(h + R, spec.H), 0), max(w, 0):max(min(w + R, spec.W), 0)] = True
        assert m.any() and not m.all()
    expects = kc.conv_in_reference(case)
    wants = [v] + [F.silu(v * (1 if case.scale[i] is None else case.scale[i].double()) + (0 if case.shift[i] is None else case.shift[i].double()))
                   if spec.aux[i][1] == 1 else v * (1 if case.scale[i] is None else case.scale[i].double()) + (0 if case.shift[i] is None else case.shift[i].double())
                   for i in range(len(spec.aux))]
    assert [e.name for e in expects] == ["out"] + ["aux%d" % i for i in range(len(spec.aux))]
    for e, want in zip(expects, wants):
        wr = _window(e, e.written)
        assert torch.equal(wr, m[..., None].expand_as(wr)), "%s %s written set" % (spec.name, e.name)
        assert not e.written[:e.g.off].any() and not e.written[e.g.off + e.g.view.numel():].any()
        assert torch.allclose(_window(e, e.want)[wr], want[wr], rtol=1e-12, atol=1e-12)


def test_conv_in_case_table_covers_the_launch_paths():
    dense = [s for s in kc.CONV_IN_CASES if s.tiles is None]
    tiles = [s for s in kc.CONV_IN_CASES if s.tiles is not None]
    assert {len(s.aux) for s in dense} == {0, 1, 2} and {len(s.aux) for s in tiles} == {0, 1, 2}
    assert {s.Cin for s in kc.CONV_IN_CASES} == {1, 2, 3, 4} and {8, 128, 256} <= {s.Cout for s in kc.CONV_IN_CASES}
    assert any(s.B == 2 for s in dense)
    assert {a[1] for s in kc.CONV_IN_CASES for a in s.aux} == {0, 1} and any(a[2] for s in kc.CONV_IN_CASES for a in s.aux)
    assert any(s.tiles[0] for s in tiles) and any(not s.tiles[0] for s in tiles)
    assert all(s.tiles[3] > 0 for s in tiles if s.tiles[0]), "per-image lists carry SIGE_TILE_NONE entries"
    assert all(s.W % 4 == 0 for s in dense) and any(s.W % 4 for s in tiles)
    # the shared-memory opt-in of weights above 48 KB (4 ((Cout / 8) 292 + Cout) bytes at Cin 4), on both sides and at its limit
    assert 4 * (1544 // 8 * 292 + 1544) == 231600 <= 227 * 1024 < 4 * (1552 // 8 * 292 + 1552)
    for paths in (dense, tiles):
        assert any(s.Cin == 4 and s.Cout == 1544 for s in paths) and any(s.Cin == 4 and s.Cout >= 328 for s in paths)
        assert any(s.Cin == 3 and s.Cout >= 432 and s.aux for s in paths)
    assert any(s.Cin == 4 and 256 < s.Cout < 328 for s in dense)
    assert any(s.Cin == 4 and s.Cout == 512 and s.tiles[0] for s in tiles), "the SD decoder's stem: per-image tiles, Cout 512"


# ---------------------------------------------------------------------------------------------------------------- GroupNorm fold
@pytest.mark.parametrize("spec", kc.GN_CASES, ids=lambda s: s.name)
def test_group_norm_restatement_matches_group_norm(spec):
    """scale / shift of the restatement fold F.group_norm; the same values rounded to fp32 (what the kernel stores) pass the
    check and the folded check, and an rstd 2^-9 (0.2 %) off fails the check wherever |mean| / std is small."""
    if spec.H * spec.W > 100000:
        pytest.skip("the statistics at this size are the same code path; the GPU test runs it")
    case = kc.make_gn(spec, torch.float16, "cpu", sms=_sms())
    expects, bounds = kc.gn_reference(case)
    sc, sh = (_window(e, e.want) for e in expects[:2])
    x = case.x.double()
    gn = F.group_norm(x.permute(0, 3, 1, 2), spec.G, None if case.gamma is None else case.gamma.double(),
                      None if case.beta is None else case.beta.double(), float(np.float32(spec.eps)))
    folded = x.permute(0, 3, 1, 2) * sc[:, :, None, None] + sh[:, :, None, None]
    assert float((folded - gn).abs().max()) <= 1e-9 * float(gn.abs().max())
    init = kc.snapshot(case.buffers())
    case.scale.view.copy_(sc.float())
    case.shift.view.copy_(sh.float())
    case.ws.view.zero_()                                                                # a workspace may hold anything
    got = {k: g.flat for k, g in case.buffers().items()}
    kc.check(spec.name, expects, got, init)
    assert kc.gn_folded_check(spec.name, case, bounds) <= 1.0
    if spec.mean / spec.std < 1:
        be = torch.zeros(spec.C, dtype=F64) if case.beta is None else case.beta.double()
        case.scale.view.copy_((sc * (1 + 2.0 ** -9)).float())
        case.shift.view.copy_((be - (be - sh) * (1 + 2.0 ** -9)).float())
        with pytest.raises(AssertionError):
            kc.check(spec.name, expects, got, init)


def test_group_norm_case_table_covers_the_launch_paths():
    cases = kc.GN_CASES
    assert {kc.gn_cpb(s.C, s.G) == 32 for s in cases} == {True, False}
    assert any(kc.gn_cpb(s.C, s.G) == s.C and s.C // s.G > 32 for s in cases), "groups wider than 32 channels"
    assert any(kc.gn_cpb(s.C, s.G) == s.C and s.C % 32 for s in cases), "C % 32 != 0"
    assert {256 % (s.C // 8) == 0 for s in cases} == {True, False}, "partial CTAs with and without idle threads"
    assert any(s.H * s.W < 64 for s in cases) and any((s.H, s.W) == (512, 512) for s in cases)
    assert {(s.H, s.W) for s in cases if s.mean / s.std >= 32} == {(256, 256), (512, 512)}
    assert any(not s.affine for s in cases) and any(s.B > 1 for s in cases)
    assert {(s.C, s.G) for s in cases} >= {(128, 32), (64, 1), (96, 3), (24, 8), (1024, 32)}


def test_group_norm_chain_length():
    """The chain the bound charges: a thread's pixels ceil(ceil(HW / nblk) / slots), plus the slots of its CTA."""
    assert kc.gn_nblk(512 * 512, 132) == 264 and kc.gn_nblk(40, 132) == 1 and kc.gn_nblk(64 * 100, 132) == 100
    assert kc.gn_slots(128) == 16 and kc.gn_slots(96) == 21 and kc.gn_slots(1024) == 2
    assert kc.gn_chain(512 * 512, 128, 132) == -(-993 // 16) + 16
    assert kc.gn_chain(40, 24, 132) == 40 // 85 + 1 + 85


# ---------------------------------------------------------------------------------------------------------------- conv_out
@pytest.mark.parametrize("spec", kc.CONV_OUT_CASES, ids=lambda s: s.name)
def test_conv_out_restatement_matches_conv2d(spec):
    case = kc.make_conv_out(spec, F64, "cpu")
    x = case.x.permute(0, 3, 1, 2)
    a = x
    if case.scale is not None:
        a = a * case.scale[:, :, None, None].double()
    if case.shift is not None:
        a = a + case.shift[:, :, None, None].double()
    if spec.act == 1:
        a = F.silu(a)
    want = F.conv2d(a, case.w, case.bias, padding=1)
    (e,) = kc.conv_out_reference(case)
    assert bool(_window(e, e.written).all()) and not e.written[:e.g.off].any() and not e.written[e.g.off + e.g.view.numel():].any()
    assert torch.allclose(_window(e, e.want), want, rtol=1e-12, atol=1e-12)


def test_conv_out_case_table_covers_the_launch_paths():
    cases = kc.CONV_OUT_CASES
    assert {kc.conv_out_per_element(s.C) for s in cases} == {True, False}
    assert {s.C for s in cases} == {16, 48, 96, 128, 160, 272}
    assert {1, 8} <= {s.Cout for s in cases} and all(1 <= s.Cout <= 8 for s in cases)
    assert any(s.H % 8 and s.W % 32 for s in cases)
    assert {s.pre for s in cases} == {"both", "scale", "shift", "none"} and {s.act for s in cases} == {0, 1}
    assert any(s.pre == "none" and s.act == 0 and kc.conv_out_per_element(s.C) for s in cases), "no pre-op on the per-element path"
    assert any(s.pre == "none" and s.act == 0 and not kc.conv_out_per_element(s.C) for s in cases)
    assert any(s.B > 1 and s.pre == "both" for s in cases)


# ---------------------------------------------------------------------------------------------------------------- attention
@pytest.mark.parametrize("spec", [s for s in kc.ATTN_CASES if s.N == 128 and s.C == 256 and s.B == 1], ids=lambda s: s.name)
def test_attention_restatement_matches_softmax(spec):
    case = kc.make_attn(spec, torch.bfloat16, "cpu")
    q, k, v = (t.double() for t in case.qkv.split(spec.C, dim=2))
    logits = q @ k.transpose(1, 2)
    want = torch.softmax(logits, dim=-1) @ v
    (e,) = kc.attn_reference(case)
    assert torch.allclose(_window(e, e.want), want, rtol=1e-12, atol=1e-12)
    assert bool(_window(e, e.written).all()) and e.g.off * 2 % 16 == 0 and e.g.view.data_ptr() % 16 == 0
    sl = logits.view(spec.B, spec.N, -1, kc.KPC).amax(dim=3)
    M = logits.amax(dim=2)
    if spec.mode == "flat":
        assert bool((logits == 0).all())
    elif spec.mode == "dominant":
        assert bool((logits.argmax(dim=2) == spec.r * kc.KPC + 17).all()) and float((M - logits.median(dim=2).values).min()) > 10
    elif spec.mode == "low_slice":
        gap = M - sl[:, :, spec.r]
        assert 27 < float(gap.min()) and float(gap.max()) < 33
    elif spec.mode == "large":
        assert 60 < float(logits.abs().max()) < 90
    # the bound is a small multiple of the output's own rounding where the softmax is not peaked
    bound = _window(e, e.bound)
    assert float((bound / (kc.ROUNDOFF[torch.bfloat16] * (want.abs() + (torch.softmax(logits, -1) @ v.abs())))).max()) < 8


def test_attention_case_table_covers_every_instantiation():
    cases = kc.ATTN_CASES
    assert {(s.N, s.C) for s in cases} == set(kc.ATTN_SHAPES)
    for (N, C) in kc.ATTN_SHAPES:
        for B in (1, 3):
            modes = {(s.mode, s.r) for s in cases if (s.N, s.C, s.B) == (N, C, B)}
            ks = N // kc.KPC
            assert {"random", "flat", "large"} <= {m for m, _ in modes}
            assert {r for m, r in modes if m == "dominant"} == set(range(ks))
            assert any(m == "low_slice" for m, _ in modes) == (ks > 1)


# ---------------------------------------------------------------------------------------------------------------- C-ABI refusals
def test_dense_glue_refuses_bad_arguments_before_any_cuda_call(cabi_lib):
    """The pointers here are not device memory: a launch would fault, so these calls must fail on their arguments."""
    from sige_b200 import _cabi

    lib = _cabi.lib()
    P = 0x10000
    for C, Cout in ((40, 3), (24, 3), (64, 9), (64, 0)):
        assert lib.sige_conv_out_nhwc(P, None, None, 1, P, None, P, _cabi.F16, 1, 16, 16, C, Cout, None) != 0
        assert b"C % 16 == 0 and Cout <= 8" in lib.sige_last_error()
    sms = _sms()
    B, H, W, C = 2, 64, 64, 128
    need = B * kc.gn_nblk(H * W, sms) * C * 2
    assert lib.sige_group_norm_fold_workspace(B, C) >= need
    assert lib.sige_group_norm_fold(P, _cabi.F16, B, H, W, C, 32, 1e-6, None, None, P, P, P, need - 1, None) != 0
    assert b"workspace too small" in lib.sige_last_error() and (b"need %d" % need) in lib.sige_last_error()
    for W_ in (6, 10, 13):
        assert lib.sige_conv_in_nhwc(P, P, None, P, _cabi.F16, 1, 8, W_, 3, 128, 0, None, None) != 0
        assert b"W % 4 == 0" in lib.sige_last_error()
