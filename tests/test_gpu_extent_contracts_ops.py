"""The tile ops, mask reduction, scatter map and dense glue kernels at the largest extents and counts their ABI accepts,
against the existing float64 restatements (tests/step_kernel_contracts.py, tests/kernel_contracts.py, sige_b200.masks).

  * Extents: images of 65535 rows by 16 columns and the transpose (65534 where a source is read up-sampled, 65532 where the
    dense stem needs W % 4 == 0), with tiles across row / column 32768 and against the last row / column
    (extent_contract.paste_targets).  Every launch is checked as the kernel contract tests check it: each written element
    within its bound, every other element of every written buffer (guard bands included) and every input bitwise unchanged,
    and a second launch bitwise identical.
  * Counts: get_scatter_map with N * Ro * So = 2^32 tile pixels, reduce_mask at the largest candidate grid it accepts
    (46340 x 46340 = 2^31 - 88048), and the tiled stem at 2^31 - 4096 outputs, whose grid-stride loop index used to wrap.
  * Offsets past 2^31: the D = 512 sparse attention reading keys / values and writing output rows as column slices of one
    [2^15 + 1, 2^16] buffer (clusters of 8 and of 1), and sige_cache_load into a destination of 2^31 + 2^20 elements.

Not measured: a reduce_mask call that lists more than 2^30 active tiles (its 64-bit list offsets) would need a 16 GiB list.
"""
from dataclasses import replace

import pytest
import torch

import extent_contract as ec
import kernel_contracts as kc
import step_kernel_contracts as sk
from kernel_contracts import _run_and_check
from tile_conv_contract import TILE_NONE

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MAX_PEAK = 10 * ec.GiB
NAME = {torch.float16: "f16", torch.bfloat16: "bf16", torch.float32: "f32"}
DTYPES3 = pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32], ids=["f16", "bf16", "f32"])
DTYPES2 = pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
TALL = pytest.mark.parametrize("tall", [True, False], ids=["tall", "wide"])


def _lib():
    from sige_b200 import _cabi

    return _cabi.lib()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _check_peak(label, peak):
    assert peak <= MAX_PEAK, "%s: %.1f GiB" % (label, peak / ec.GiB)
    ec.need(peak, DEV)


# ---------------------------------------------------------------------------------------------------------------- tile ops
SW = sk.ACT_SWISH
TILE_EDGE = [
    sk.TileSpec("g_nchw_up_per_sample_swish", "gather", "nchw", up=1, scale=(1, 1, 0, 0), shift=(1, 1, 0, 0), act=SW, seed=501),
    sk.TileSpec("g_nhwc_up_per_sample", "gather", "nhwc", up=1, scale=(1, 1, 0, 0), shift=(1, 1, 0, 0), seed=502),
    sk.TileSpec("g_nhwc_per_sample_swish_first", "gather", "nhwc", scale=(1, 1, 0, 0), shift=(1, 1, 0, 0), act=SW, act_first=True,
                seed=503),
    sk.TileSpec("s_nhwc_stride2_residual", "scatter", "nhwc", stride=2, residual=(1, 1, 1, 1), seed=504),
    sk.TileSpec("s_nchw_stride2_residual_inplace", "scatter", "nchw", stride=2, residual=(1, 1, 1, 1), inplace=True, seed=505),
    sk.TileSpec("sg_nhwc_per_sample_swish", "scatter_gather", "nhwc", scale=(1, 1, 0, 0), shift=(1, 1, 0, 0), act=SW, seed=506),
    sk.TileSpec("sg_nchw", "scatter_gather", "nchw", seed=507),
    sk.TileSpec("swbr_nhwc", "swbr", "nhwc", seed=508),
    sk.TileSpec("swbr_nchw_stride2", "swbr", "nchw", stride=2, seed=509),
]


def _device_map(case):
    s = case.spec
    m = torch.empty(s.H, s.W, 3, dtype=torch.int32, device=DEV)
    idx = case.idx["idx"]
    rc = _lib().sige_get_scatter_map(s.H, s.W, 6, 6, 3, 3, 1, 1, 1, 1, idx.data_ptr(), idx.shape[0], m.data_ptr(), _stream())
    torch.cuda.synchronize()
    assert rc == 0, _lib().sige_last_error()
    return m


@DTYPES3
@TALL
@pytest.mark.parametrize("base", TILE_EDGE, ids=lambda s: s.name)
def test_tile_op_at_the_extent_limit(base, tall, dtype):
    H, W = ec.edge_extent(tall, even=base.up == 1)
    spec = replace(base, name="%s_%s" % (base.name, "tall" if tall else "wide"), H=H, W=W)
    # the float64 restatement keeps about a dozen [B, C, H, W] float64 tensors
    _check_peak(spec.name, spec.B * spec.C * H * W * 8 * 16)
    case = sk.make_tile(spec, dtype, DEV, origins=ec.tile_op_origins(spec, tall))
    if spec.op == "scatter_gather":
        m = _device_map(case)
        assert torch.equal(m, case.idx["map"]), "%s: get_scatter_map differs from its restatement" % spec.name
        case.idx["map"] = m
    expects = sk.tile_reference(case)
    lib, keep = _lib(), []
    label = "%s %s (%d x %d, %d tiles)" % (spec.name, NAME[dtype], H, W, case.idx["idx"].shape[0])
    _run_and_check("tile_ops", label, case, expects, lambda flags: sk.tile_call(case, lib, keep))
    del case, expects
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------- reduce_mask
GEOMS = [((6, 6), (4, 4), (1, 1)), ((2, 2), (1, 1), (0, 0)), ((5, 5), (2, 2), (2, 2))]


def _edge_masks(tall):
    """[2, H, W] uint8: a few active pixels in the last row only, and in the last column only."""
    H, W = ec.edge_extent(tall)
    m = torch.zeros(2, H, W, dtype=torch.uint8, device=DEV)
    for w in (0, W // 2, W - 1):
        m[0, H - 1, w] = 1
    for h in (0, H // 2, H - 1):
        m[1, h, W - 1] = 1
    if tall:
        m[1, ec.MID, W - 1] = m[1, ec.MID - 1, W - 1] = 1
    else:
        m[0, H - 1, ec.MID] = m[0, H - 1, ec.MID - 1] = 1
    return m


@TALL
@pytest.mark.parametrize("geom", GEOMS, ids=lambda g: "b%d_s%d_p%d" % (g[0][0], g[1][0], g[2][0]))
def test_reduce_mask_at_the_extent_limit(geom, tall):
    from sige_b200 import masks as mk
    from sige_b200 import ops

    block, stride, pad = geom
    m = _edge_masks(tall)
    want = [mk._reduce_mask_host(m[e], block, stride, pad) for e in range(2)]
    assert all(w.shape[0] > 0 for w in want)
    for e in range(2):
        for _ in range(2):
            got = ops.reduce_mask_cuda(m[e], block, stride, pad)
            assert torch.equal(got, want[e]), "mask %d: reduce_mask differs from the host restatement" % e
    cap = max(w.shape[0] for w in want) + 3
    for _ in range(2):
        out, counts, status = ops.reduce_mask_batched_cuda(m, block, stride, pad, cap)
        torch.cuda.synchronize()
        assert int(status) == 0 and counts.tolist() == [w.shape[0] for w in want]
        for e in range(2):
            seg = out[e * cap:(e + 1) * cap]
            n = want[e].shape[0]
            assert torch.equal(seg[:n], want[e]), "mask %d: reduce_mask_batched differs from the host restatement" % e
            assert bool((seg[n:] == TILE_NONE).all())
    print("[extent contract] reduce_mask %s %s: %s tiles, bitwise equal to the host restatement"
          % ("tall" if tall else "wide", geom, [w.shape[0] for w in want]))


def test_reduce_mask_refuses_a_candidate_grid_of_2_to_the_32():
    """The capacity query's -1 is raised before the mask is materialised (the mask here is one expanded byte)."""
    from sige_b200 import _cabi, ops

    m = torch.zeros(1, 1, dtype=torch.uint8, device=DEV).expand(65535, 65535)
    with pytest.raises(_cabi.SigeError, match="too many candidate tiles"):
        ops.reduce_mask_cuda_launch(m, (1, 1), (1, 1), (0, 0))


def test_reduce_mask_at_the_largest_candidate_grid():
    """46339 x 46339 mask, 2 x 2 windows at stride 1: 46340^2 = 2^31 - 88048 candidates, the most a square grid may have.  A
    few active pixels, the last among them; the list (capacity 64) and count must equal the windows that hold them, in
    row-major order, and the rows past the count stay as they were."""
    H = W = 46339
    n_cand = (H + 1) * (W + 1)
    assert 2 ** 31 - 2 ** 17 < n_cand < 2 ** 31
    _check_peak("reduce_mask 46339^2", H * W + (1 << 20))
    lib = _lib()
    m = torch.zeros(H, W, dtype=torch.uint8, device=DEV)
    px = [(0, 0), (0, W - 1), (23170, 12345), (ec.MID, ec.MID), (H - 1, 0), (40000, W - 1), (H - 1, W - 1)]
    for h, w in px:
        m[h, w] = 1
    tiles = sorted({(i, j) for h, w in px for i in (h - 1, h) for j in (w - 1, w) if 0 <= i <= H and 0 <= j <= W})
    want = torch.tensor(tiles, dtype=torch.int32, device=DEV)
    cap = 64
    assert len(tiles) < cap
    out = torch.full((cap + 8, 2), -7, dtype=torch.int32, device=DEV)
    count = torch.zeros(1, dtype=torch.int32, device=DEV)
    for _ in range(2):
        assert lib.sige_reduce_mask(m.data_ptr(), H, W, 2, 2, 1, 1, 0, 0, out.data_ptr(), cap, count.data_ptr(), _stream()) == 0, \
            lib.sige_last_error()
        torch.cuda.synchronize()
        assert int(count) == len(tiles), "count %d, want %d" % (int(count), len(tiles))
        assert torch.equal(out[:len(tiles)], want) and bool((out[len(tiles):] == -7).all())
    seg = torch.full((cap, 2), -7, dtype=torch.int32, device=DEV)
    counts = torch.zeros(1, dtype=torch.int32, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    assert lib.sige_reduce_mask_batched(m.data_ptr(), 1, H, W, 2, 2, 1, 1, 0, 0, seg.data_ptr(), cap, counts.data_ptr(),
                                        status.data_ptr(), _stream()) == 0, lib.sige_last_error()
    torch.cuda.synchronize()
    assert int(counts) == len(tiles) and int(status) == 0
    assert torch.equal(seg[:len(tiles)], want) and bool((seg[len(tiles):] == TILE_NONE).all())
    print("[extent contract] reduce_mask %d x %d (%d candidates): %d tiles, bitwise equal" % (H, W, n_cand, len(tiles)))


# ---------------------------------------------------------------------------------------------------------------- scatter map
def test_get_scatter_map_past_2_to_the_32_tile_pixels():
    """2^28 tiles of 6 x 6 under a 3 x 3 kernel: N * Ro * So = 2^32 (0 in an int).  The list is SIGE_TILE_NONE but for a few
    tiles at indices above 2^27, whose map entries must name them."""
    N, H, W = 2 ** 28, 64, 64
    _check_peak("scatter map 2^28 tiles", N * 8 + (1 << 24))
    real = {2 ** 27 + 1: (-1, -1), 2 ** 27 + 12345: (29, 13), 2 ** 28 - 2: (59, 59), 2 ** 28 - 1: (61, 30)}
    idx = torch.full((N, 2), TILE_NONE, dtype=torch.int32, device=DEV)
    for n, o in real.items():
        idx[n] = torch.tensor(o, dtype=torch.int32)
    ids = torch.tensor(list(real), dtype=torch.int32)
    want = sk.scatter_map(H, W, torch.tensor(list(real.values()), dtype=torch.int32), 4, 4, 1, 1, 1, 1)
    want[..., 0] = torch.where(want[..., 0] >= 0, ids[want[..., 0].clamp(min=0).long()], want[..., 0])
    want = want.to(DEV)
    lib = _lib()
    first = None
    for _ in range(2):
        m = torch.zeros(H, W, 3, dtype=torch.int32, device=DEV)
        assert lib.sige_get_scatter_map(H, W, 6, 6, 3, 3, 1, 1, 1, 1, idx.data_ptr(), N, m.data_ptr(), _stream()) == 0, \
            lib.sige_last_error()
        torch.cuda.synchronize()
        assert bool((m != -1).any()), "the map is all -1: no tile was mapped"
        assert torch.equal(m, want), "%d map entries differ from the restatement" % int((m != want).any(-1).sum())
        assert first is None or torch.equal(m, first)
        first = m
    print("[extent contract] get_scatter_map: 2^28 tiles (2^32 tile pixels), %d mapped pixels equal" % int((want[..., 0] >= 0).sum()))


# ---------------------------------------------------------------------------------------------------------------- dense glue
def _edge_conv_in(tall, tiles):
    H, W = ec.edge_extent(tall)
    W = W - W % 4                                       # the dense stem needs W % 4 == 0
    name = "stem_%s_%s" % ("tiles" if tiles else "dense", "tall" if tall else "wide")
    spec = kc.ConvInSpec(name, B=1, H=H, W=W, Cin=3, Cout=16, aux=((True, 1, True),), seed=601 + 2 * tiles + tall)
    if not tiles:
        return spec, None
    org = ec.stem_tile_origins(H, W, 6, tall)
    return replace(spec, tiles=(False, (len(org),), 6, 0)), org


@DTYPES2
@TALL
@pytest.mark.parametrize("tiles", [False, True], ids=["dense", "tiles"])
def test_conv_in_at_the_extent_limit(tiles, tall, dtype):
    spec, org = _edge_conv_in(tall, tiles)
    _check_peak(spec.name, spec.H * spec.W * spec.Cout * 8 * 16)
    case = kc.make_conv_in(spec, dtype, DEV)
    if org is not None:
        case.idx = torch.tensor(org, dtype=torch.int32, device=DEV)
    expects = kc.conv_in_reference(case)
    lib = _lib()
    _run_and_check("conv_in", "%s %s (%d x %d)" % (spec.name, NAME[dtype], spec.H, spec.W), case, expects,
                   lambda flags: kc.conv_in_call(case, lib))


@DTYPES2
def test_conv_in_tiles_at_2_to_the_31_minus_4096_outputs(dtype):
    """Cin 1, Cout 512, 2^19 - 1 tiles of 8 x 8 on a 64 x 64 image: n_tiles * R * S * Cout / 8 = 2^31 - 4096, past the point
    (2^31 - 528 * 256 on 132 SMs) where an int grid-stride index would wrap.  Every tile but the last lies in the left half;
    the last alone covers the bottom-right corner, so its pixels show that the loop reached the end of the list."""
    n = 2 ** 19 - 1
    spec = kc.ConvInSpec("stem_tiles_2_31", B=1, H=64, W=64, Cin=1, Cout=512, tiles=(False, (1,), 8, 0), seed=611)
    assert n * 8 * 8 * 512 // 8 == 2 ** 31 - 4096
    case = kc.make_conv_in(spec, dtype, DEV)
    g = torch.Generator(device="cpu")
    g.manual_seed(611)
    org = torch.stack([torch.randint(-7, 64, (n,), generator=g), torch.randint(-7, 25, (n,), generator=g)], 1)
    org[-1] = torch.tensor([60, 60])
    case.idx, case.n_tiles = org.to(torch.int32).to(DEV), n
    expects = kc.conv_in_reference(case)
    assert bool(expects[0].written[case.out.off:case.out.off + case.out.view.numel()].view(64, 64, 512)[60:, 60:].all())
    lib = _lib()
    _run_and_check("conv_in", "%s %s (%d tiles)" % (spec.name, NAME[dtype], n), case, expects, lambda flags: kc.conv_in_call(case, lib))


@DTYPES2
@TALL
def test_group_norm_fold_at_the_extent_limit(tall, dtype):
    H, W = ec.edge_extent(tall)
    spec = kc.GNSpec("gn_%s" % ("tall" if tall else "wide"), B=2, H=H, W=W, C=32, G=8, seed=621 + tall)
    _check_peak(spec.name, spec.B * H * W * spec.C * 8 * 8)
    case = kc.make_gn(spec, dtype, DEV)
    expects, bounds = kc.gn_reference(case)
    lib = _lib()
    label = "%s %s (%d x %d)" % (spec.name, NAME[dtype], H, W)
    got = _run_and_check("gn_fold", label, case, expects, lambda flags: kc.gn_call(case, lib))
    for k, gb in case.buffers().items():
        gb.flat.copy_(got[k])
    r = kc.gn_folded_check(label, case, bounds)
    print("[extent contract] gn_fold %-40s x*scale + shift vs group_norm: worst |err| / bound %.3f" % (label, r))


@DTYPES2
@TALL
def test_conv_out_at_the_extent_limit(tall, dtype):
    H, W = ec.edge_extent(tall)
    spec = kc.ConvOutSpec("conv_out_%s" % ("tall" if tall else "wide"), B=2, H=H, W=W, C=32, Cout=3, seed=631 + tall)
    _check_peak(spec.name, spec.B * H * W * spec.C * 8 * 6)
    case = kc.make_conv_out(spec, dtype, DEV)
    expects = kc.conv_out_reference(case)
    lib = _lib()
    _run_and_check("conv_out", "%s %s (%d x %d)" % (spec.name, NAME[dtype], H, W), case, expects, lambda flags: kc.conv_out_call(case, lib))


# ---------------------------------------------------------------------------------------------------------------- write-back
def _code(dtype):
    from sige_b200 import _cabi

    return {torch.float16: _cabi.F16, torch.bfloat16: _cabi.BF16, torch.float32: _cabi.F32}[dtype]


def _wb_entry(src, dst, idx, B, C, H, W, dst_dtype, layout, off=1, stride=1, R=4):
    from sige_b200 import _cabi

    e = _cabi.WritebackEntry()
    e.src, e.dst, e.idx, e.N, e.B, e.C, e.H, e.W = src.data_ptr(), dst.data_ptr(), idx.data_ptr(), idx.shape[0], B, C, H, W
    e.src_dtype, e.dst_dtype, e.dst_layout = _code(src.dtype), _code(dst_dtype), layout
    e.offH = e.offW = off
    e.strideH = e.strideW = stride
    e.Ro = e.So = R
    return e


def _writeback(*entries):
    from sige_b200 import _cabi

    table = (_cabi.WritebackEntry * len(entries))(*entries)
    rc = _lib().sige_tile_writeback(table, len(entries), _stream())
    torch.cuda.synchronize()
    assert rc == 0, _lib().sige_last_error()


def _wb_want(src, org, off, stride, C, H, W, B, offsets, R=4):
    """(element offsets, values) of a write-back of `src` (NHWC [B, H, W, C]) through the tiles `org` (the same list for
    every image): the pasted pixels, every channel."""
    n, r, s, h, w = (t.to(src.device) for t in ec.tile_pixels(org, R, off, stride, H, W))
    pos, val = [], []
    for b in range(B):
        bb = torch.full_like(h, b)
        pos.append(offsets(C, H, W, bb, h, w))
        val.append(src[b, h, w, :])
    return torch.cat(pos), torch.cat(val)


@DTYPES2
@TALL
def test_tile_writeback_at_the_extent_limit(tall, dtype):
    """One call, two entries: 4 x 4 tiles into an fp32 NCHW cache (stride 1) and 2 x 2 tiles into an NHWC cache of the source
    dtype (stride 2)."""
    from sige_b200 import _cabi

    H, W = ec.edge_extent(tall)
    B, C = 2, 16
    n, short = (H, W) if tall else (W, H)
    org1 = ec.spread(ec.paste_targets(n, 4, 1, 1), 4, 4, 1, 1, 1, short, tall, "wb_s1")
    org2 = ec.spread(ec.paste_targets(n, 2, 0, 2), 2, 2, 0, 0, 2, short, tall, "wb_s2")
    src = torch.empty(B * H * W * C, dtype=dtype, device=DEV)
    ec.fill(src, 701)
    src = src.view(B, H, W, C)
    d1 = torch.empty(B * C * H * W, dtype=torch.float32, device=DEV)
    d2 = torch.empty(B * H * W * C, dtype=dtype, device=DEV)
    ec.fill(d1, 702)
    ec.fill(d2, 703)
    i1 = torch.tensor(org1, dtype=torch.int32, device=DEV)
    i2 = torch.tensor(org2, dtype=torch.int32, device=DEV)
    src0 = src.clone()
    p1, v1 = _wb_want(src, org1, 1, 1, C, H, W, B, ec.nchw_offsets)
    p2, v2 = _wb_want(src, org2, 0, 2, C, H, W, B, ec.nhwc_offsets, R=2)
    label = "writeback %s %s (%d x %d)" % ("tall" if tall else "wide", NAME[dtype], H, W)
    for _ in range(2):
        _writeback(_wb_entry(src, d1, i1, B, C, H, W, torch.float32, _cabi.NCHW),
                   _wb_entry(src, d2, i2, B, C, H, W, dtype, _cabi.NHWC, off=0, stride=2, R=2))
        ec.moved_check(label + " nchw f32", d1, 702, p1, v1.float())
        ec.moved_check(label + " nhwc", d2, 703, p2, v2)
    assert torch.equal(kc.bits(src), kc.bits(src0)), "%s: the source was modified" % label
    print("[extent contract] %-56s %d + %d elements, bitwise" % (label, p1.numel(), p2.numel()))


# ---------------------------------------------------------------------------------------------------------------- 2^31 elements
BIG = (2048, 1024, 1024)                 # C, H, W of a [1, C, H, W] tensor of 2^31 elements


@DTYPES2
def test_gather_nchw_reads_past_2_to_the_31_elements(dtype):
    """The source and the stack of a gather, one after the other in one buffer; the tiles reach the source's last element."""
    C, H, W = BIG
    n_x = C * H * W
    org = [(-5, -5), (0, W - 6), (511, 511), (H - 6, 0), (H - 6, W - 6), (H - 4, W - 3), (H - 1, W - 1)]
    N = len(org)
    es = torch.empty((), dtype=dtype).element_size()
    _check_peak("gather 2^31", (n_x + N * C * 36) * es + 2 * ec.CHUNK * 8)
    flat = torch.empty(n_x + N * C * 36, dtype=dtype, device=DEV)
    ec.fill(flat, 711)
    x, out = flat[:n_x].view(1, C, H, W), flat[n_x:]
    idx = torch.tensor(org, dtype=torch.int32, device=DEV)
    n, r, s, h, w = (t.to(DEV) for t in ec.tile_pixels(org, 6, 0, 1, H, W))
    want = torch.zeros(N, C, 6, 6, dtype=dtype, device=DEV)
    want[n, :, r, s] = x[0, :, h, w].t()
    pos = n_x + torch.arange(out.numel(), device=DEV)
    lib = _lib()
    label = "gather nchw %s (%d + %d elements)" % (NAME[dtype], n_x, out.numel())
    for _ in range(2):
        assert lib.sige_gather(x.data_ptr(), _code(dtype), 0, 1, C, H, W, 6, 6, idx.data_ptr(), N, None, None, 0, 0, out.data_ptr(),
                               _stream()) == 0, lib.sige_last_error()
        torch.cuda.synchronize()
        ec.moved_check(label, flat, 711, pos, want)
    print("[extent contract] %-56s bitwise" % label)


@DTYPES2
def test_scatter_nchw_writes_past_2_to_the_31_elements(dtype):
    """An in-place scatter into a [1, 2048, 1024, 1024] tensor whose stack follows it in the same buffer; tiles hang out of
    every border and the last writes the tensor's last element."""
    C, H, W = BIG
    n_y = C * H * W
    org = [(-2, -2), (510, 510), (H - 5, 0), (H - 4, W - 9), (H - 3, W - 4)]
    N = len(org)
    es = torch.empty((), dtype=dtype).element_size()
    _check_peak("scatter 2^31", (n_y + N * C * 16) * es + 2 * ec.CHUNK * 8)
    flat = torch.empty(n_y + N * C * 16, dtype=dtype, device=DEV)
    ec.fill(flat, 721)
    y, xs = flat[:n_y].view(1, C, H, W), flat[n_y:].view(N, C, 4, 4)
    idx = torch.tensor(org, dtype=torch.int32, device=DEV)
    n, r, s, h, w = (t.to(DEV) for t in ec.tile_pixels(org, 4, 1, 1, H, W))
    pos = ec.nchw_offsets(C, H, W, torch.zeros_like(h), h, w)
    assert int(pos.max()) == n_y - 1
    want = xs[n, :, r, s].clone()
    lib = _lib()
    label = "scatter nchw in place %s (%d + %d elements)" % (NAME[dtype], n_y, xs.numel())
    for _ in range(2):
        assert lib.sige_scatter(xs.data_ptr(), None, y.data_ptr(), _code(dtype), 0, 1, C, H, W, 4, 4, 1, 1, 1, 1, idx.data_ptr(), N, None,
                                _stream()) == 0, lib.sige_last_error()
        torch.cuda.synchronize()
        ec.moved_check(label, flat, 721, pos, want)
    print("[extent contract] %-56s bitwise" % label)


@DTYPES2
def test_tile_writeback_into_an_nchw_cache_past_2_to_the_31_elements(dtype):
    C, H, W = BIG
    n_d = C * H * W
    org = [(-2, -2), (510, 510), (H - 5, 0), (H - 4, W - 9), (H - 3, W - 4)]
    es = torch.empty((), dtype=dtype).element_size()
    _check_peak("writeback 2^31", 2 * n_d * es + 2 * ec.CHUNK * 8)
    from sige_b200 import _cabi

    src = torch.empty(n_d, dtype=dtype, device=DEV)
    ec.fill(src, 731)
    src = src.view(1, H, W, C)
    dst = torch.empty(n_d, dtype=dtype, device=DEV)
    ec.fill(dst, 732)
    idx = torch.tensor(org, dtype=torch.int32, device=DEV)
    pos, want = _wb_want(src, org, 1, 1, C, H, W, 1, ec.nchw_offsets)
    assert int(pos.max()) == n_d - 1
    label = "writeback nchw %s (%d elements)" % (NAME[dtype], n_d)
    for _ in range(2):
        _writeback(_wb_entry(src, dst, idx, 1, C, H, W, dtype, _cabi.NCHW))
        ec.moved_check(label, dst, 732, pos, want)
    print("[extent contract] %-56s bitwise" % label)


@DTYPES2
def test_conv_in_writes_past_2_to_the_31_elements(dtype):
    """The dense stem into a [1, 4097, 4096, 128] output (2^31 + 2^19 elements; its guard allows up to 2^32), one 16-byte
    guard band on either side.  The float64 restatement is evaluated 128 rows at a time."""
    import torch.nn.functional as F

    from sige_b200 import _cabi

    H, W, Cin, Cout = 4097, 4096, 3, 128
    n_out = H * W * Cout
    assert 2 ** 31 < n_out < 2 ** 32
    es = torch.empty((), dtype=dtype).element_size()
    _check_peak("conv_in 2^31", n_out * es + 128 * W * Cout * 8 * 8)
    g = torch.Generator(device=DEV)
    g.manual_seed(741)
    x = torch.randn(1, H, W, Cin, generator=g, device=DEV).to(dtype)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g, device=DEV) * (9 * Cin) ** -0.5).to(dtype)
    bias = (0.3 * torch.randn(Cout, generator=g, device=DEV)).to(dtype)
    guard = 16 // es
    flat = torch.empty(n_out + 2 * guard, dtype=dtype, device=DEV)
    ec.fill(flat, 742)
    out = flat[guard:guard + n_out]
    lib = _lib()
    u = kc.ROUNDOFF[dtype]
    x64 = x.double().permute(0, 3, 1, 2)
    w64, b64 = w.double(), bias.double().view(1, -1, 1, 1)
    label = "conv_in dense %s (%d x %d x %d)" % (NAME[dtype], H, W, Cout)
    first = None
    for launch in range(2):
        assert lib.sige_conv_in_nhwc(x.data_ptr(), w.data_ptr(), bias.data_ptr(), out.data_ptr(), _code(dtype), 1, H, W, Cin, Cout, 0,
                                     None, _stream()) == 0, lib.sige_last_error()
        torch.cuda.synchronize()
        assert torch.equal(kc.bits(flat[:guard]), kc.bits(ec._chunk(flat, 0, 742)[:guard])), "%s: the lead guard changed" % label
        tail = flat[-guard:]
        k = (flat.numel() - guard) // ec.CHUNK
        assert torch.equal(kc.bits(tail), kc.bits(ec._chunk(flat, k, 742)[(flat.numel() - guard) - k * ec.CHUNK:])), \
            "%s: the tail guard changed" % label
        o = out.view(H, W, Cout)
        if launch == 0:
            first = o.cpu()
            worst = 0.0
            for r0 in range(0, H, 128):
                r1 = min(r0 + 128, H)
                lo, hi = max(r0 - 1, 0), min(r1 + 1, H)
                xs = F.pad(x64[:, :, lo:hi], (0, 0, 1 if r0 == 0 else 0, 1 if r1 == H else 0))
                v = F.conv2d(xs, w64, padding=(0, 1)) + b64
                mag = F.conv2d(xs.abs(), w64.abs(), padding=(0, 1)) + b64.abs()
                v, mag = v[0].permute(1, 2, 0), mag[0].permute(1, 2, 0)
                bound = u * v.abs() + kc.ACC * mag + kc.ABS
                err = (o[r0:r1].double() - v).abs()
                ratio = torch.nan_to_num(torch.where(err == 0, torch.zeros_like(err), err / bound), nan=float("inf"))
                rmax = float(ratio.max())
                if rmax > 1:
                    hh, ww, cc = (int(z) for z in (ratio == ratio.max()).nonzero()[0])
                    raise AssertionError("%s: out at (h, w, c) = (%d, %d, %d): got %r, want %r, bound %.3g"
                                         % (label, r0 + hh, ww, cc, float(o[r0 + hh, ww, cc]), float(v[hh, ww, cc]), float(bound[hh, ww, cc])))
                worst = max(worst, rmax)
                del xs, v, mag, bound, err, ratio
        else:
            for r0 in range(0, H, 256):
                assert torch.equal(kc.bits(o[r0:r0 + 256].cpu()), kc.bits(first[r0:r0 + 256])), "%s: a second launch differs" % label
    print("[extent contract] %-56s worst |err| / bound %.3f" % (label, worst))


@DTYPES2
def test_spade_modulation_on_channel_slices_past_2_to_the_31_elements(dtype):
    """x, gamma, beta and out are 64-channel slices of one [2^22 + 1, 512] buffer: pixels x stride = 2^31 + 512, and the last
    pixel's slices lie past element 2^31.  Checked against step_kernel_contracts.spade_reference's formula, 2^18 pixels at a
    time."""
    import numpy as np

    P, S, C = 2 ** 22 + 1, 512, 64
    cx, cg, cb, co = 0, 128, 192, 320
    es = torch.empty((), dtype=dtype).element_size()
    _check_peak("spade 2^31", P * S * es + 4 * P * C * es + 2 * ec.CHUNK * 8 + (1 << 18) * C * 8 * 8)   # + input and result copies
    flat = torch.empty(P * S, dtype=dtype, device=DEV)
    ec.fill(flat, 751)
    buf = flat.view(P, S)
    x, gamma, beta, out = (buf[:, c:c + C] for c in (cx, cg, cb, co))
    slope = 0.2
    lib = _lib()
    u = kc.ROUNDOFF[dtype]
    label = "spade %s (%d pixels x %d stride)" % (NAME[dtype], P, S)
    inputs0 = [t.clone() for t in (x, gamma, beta)]
    first = None
    for launch in range(2):
        assert lib.sige_spade_modulate(x.data_ptr(), S, gamma.data_ptr(), S, beta.data_ptr(), S, out.data_ptr(), S, P, C, slope,
                                       _code(dtype), _stream()) == 0, lib.sige_last_error()
        torch.cuda.synchronize()
        ec.unchanged_outside(label, flat, 751, lambda i: (i % S >= co) & (i % S < co + C))
        assert all(torch.equal(kc.bits(a), kc.bits(b)) for a, b in zip((x, gamma, beta), inputs0)), "%s: an input changed" % label
        if launch == 0:
            first = out.clone()
            worst = 0.0
            for p0 in range(0, P, 1 << 18):
                sl = slice(p0, min(p0 + (1 << 18), P))
                f = x[sl].double() * (1 + gamma[sl].float()).double() + beta[sl].double()
                want = torch.where(f > 0, f, f * float(np.float32(slope)))
                bound = (u + 2 * kc.U32) * want.abs() + sk.HALF_SUBNORMAL[dtype] + 2.0 ** -149
                err = (out[sl].double() - want).abs()
                ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
                r = float(ratio.max())
                if r > 1:
                    p, c = (int(z) for z in (ratio == ratio.max()).nonzero()[0])
                    raise AssertionError("%s: pixel %d channel %d: got %r, want %r" % (label, p0 + p, c, float(out[p0 + p, c]), float(want[p, c])))
                worst = max(worst, r)
        else:
            assert torch.equal(kc.bits(out), kc.bits(first)), "%s: a second launch differs" % label
    print("[extent contract] %-56s worst |err| / bound %.3f" % (label, worst))


@DTYPES2
@pytest.mark.parametrize("form", ["simt_nchw", "depthwise_nhwc"])
def test_tile_conv_generic_reads_past_2_to_the_31_elements(form, dtype):
    """A stack of M x 64 x 6 x 6 > 2^31 elements (M = 932068) convolved 3 x 3 into 4 x 4 outputs: through the generic kernel
    (NCHW, 8 output channels) and the depthwise one (NHWC, groups = 64).  The output stack follows the input stack in one
    buffer.  Checked against generic_conv_contract's float64 conv and bound, 2^13 tiles at a time."""
    import generic_conv_contract as gc

    M, Cin, R = 932068, 64, 6
    Cout, groups, layout = (8, 1, "nchw") if form == "simt_nchw" else (64, 64, "nhwc")
    spec = gc.GenSpec("big_" + form, M, Cin, Cout, R, R, groups=groups, layout=layout, seed=761)
    n_x, n_out = M * Cin * R * R, M * Cout * spec.P
    assert n_x > 2 ** 31
    es = torch.empty((), dtype=dtype).element_size()
    _check_peak(spec.name, (n_x + 2 * n_out) * es + 2 * ec.CHUNK * 8 + (1 << 13) * Cin * 36 * 8 * 6)
    flat = torch.empty(n_x + n_out, dtype=dtype, device=DEV)
    ec.fill(flat, 761)
    phys = (lambda *s: (s[0], s[2], s[3], s[1])) if layout == "nhwc" else (lambda *s: s)     # noqa: E731
    x = flat[:n_x].view(*phys(M, Cin, R, R))
    out = flat[n_x:].view(*phys(M, Cout, spec.Ro, spec.So))
    logical = (lambda t: t.permute(0, 3, 1, 2)) if layout == "nhwc" else (lambda t: t)       # noqa: E731
    g = torch.Generator(device=DEV)
    g.manual_seed(761)
    w = (torch.randn(Cout, spec.cig, 3, 3, generator=g, device=DEV) * spec.K ** -0.5).to(dtype)
    b = (0.3 * torch.randn(Cout, generator=g, device=DEV)).to(dtype)
    lib = _lib()
    u = kc.ROUNDOFF[dtype]
    gm = gc.gamma(spec.K + 1)
    w64, b64 = w.double(), b.double()
    label = "generic %s %s (%d x %d x %d x %d stack)" % (form, NAME[dtype], M, Cin, R, R)
    first = None
    for launch in range(2):
        assert lib.sige_tile_conv_generic(x.data_ptr(), w.data_ptr(), b.data_ptr(), out.data_ptr(), _code(dtype), int(layout == "nhwc"), M,
                                          Cin, R, R, Cout, 3, 3, 1, 1, 1, 1, groups, _stream()) == 0, lib.sige_last_error()
        torch.cuda.synchronize()
        ec.unchanged_outside(label, flat, 761, lambda i: i >= n_x)
        if launch == 0:
            first = out.clone()
            worst = 0.0
            for m0 in range(0, M, 1 << 13):
                xs = logical(x[m0:m0 + (1 << 13)]).double()
                v = gc.conv64(xs, w64, b64, spec.stride, spec.dilation, groups, spec.Ro, spec.So)
                mag = gc.conv64(xs.abs(), w64.abs(), b64.abs(), spec.stride, spec.dilation, groups, spec.Ro, spec.So)
                bound = (1 + u) * (gm * mag + (spec.K + 1) * 2.0 ** -150 * (1 + gm)) + u * v.abs() + sk.HALF_SUBNORMAL[dtype]
                err = (logical(out[m0:m0 + (1 << 13)]).double() - v).abs()
                ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
                r = float(ratio.max())
                if r > 1:
                    i = [int(z) for z in (ratio == ratio.max()).nonzero()[0]]
                    raise AssertionError("%s: out at (m, c, r, s) = (%d, %d, %d, %d): got %r, want %r"
                                         % (label, m0 + i[0], i[1], i[2], i[3], float(logical(out)[m0 + i[0], i[1], i[2], i[3]]),
                                            float(v[tuple(i)])))
                worst = max(worst, r)
                del xs, v, mag, bound, err, ratio
        else:
            assert torch.equal(kc.bits(out), kc.bits(first)), "%s: a second launch differs" % label
    print("[extent contract] %-56s worst |err| / bound %.3f" % (label, worst))


@DTYPES2
def test_sparse_attention_keys_past_2_to_the_31_elements(dtype):
    """Keys and values are the first and last 64 columns of the rows of one [2^15 + 1, 2^16] buffer: k_sn * Nk = 2^31 + 2^16,
    and the last value ends on the buffer's last element.  Checked against step_kernel_contracts.sattn_reference."""
    Nk, kn, D, Nq = 2 ** 15 + 1, 2 ** 16, 64, 64
    es = torch.empty((), dtype=dtype).element_size()
    _check_peak("sparse attention 2^31", Nk * kn * es + 2 * ec.CHUNK * 8 + (1 << 28))
    flat = torch.empty(Nk * kn, dtype=dtype, device=DEV)
    ec.fill(flat, 771)
    rows = flat.view(Nk, kn)
    k, v = rows[:, :D][None, None], rows[:, kn - D:][None, None]
    g = torch.Generator(device=DEV)
    g.manual_seed(771)
    spec = sk.SAttnSpec("keys_past_2_31", 1, 1, Nq, Nk, D, seed=771)
    q = (torch.randn(1, 1, Nq, D, generator=g, device=DEV) * 2 / (spec.s32 * D ** 0.5)).to(dtype)
    out = kc.guarded((1, 1, Nq, D), dtype, DEV, g, "bhnd")
    case = sk.SAttnCase(spec, dtype, q, k, v, {"q": q}, out, out.view)
    expects = sk.sattn_reference(case)
    lib = _lib()
    label = "sparse_attention %s (k_sn %d x Nk %d)" % (NAME[dtype], kn, Nk)
    _run_and_check("sattn", label, case, expects, lambda flags: sk.sattn_call(case, lib))
    ec.unchanged_outside(label, flat, 771, lambda i: torch.zeros_like(i, dtype=torch.bool))


# ---------------------------------------------------------------------------------------------------------------- separable conv
def _sep_origins(n_long: int, n_short: int, tall: bool, off: int = 1):
    """Origins of the destination's regular 4 x 4 output grid (4 i - off): the first row (column) of tiles, the tiles across
    32768, and the last two (the last one hangs out), cycling over the short axis."""
    last = (n_long - 1) // 4
    ii = [0] + list(range(ec.MID // 4 - 2, ec.MID // 4 + 2)) + [last - 1, last]
    jj = list(range(-(-n_short // 4)))
    org = [(4 * i - off, 4 * jj[k % len(jj)] - off) for k, i in enumerate(ii)]
    return org if tall else [(w, h) for h, w in org]


@DTYPES2
@TALL
def test_separable_conv_at_the_extent_limit(tall, dtype):
    """Branch 0 into a channel window of a buffer, branch 1 into a stack, from a channel window of the source."""
    from ctypes import byref

    H, W = ec.edge_extent(tall)
    org = _sep_origins(*((H, W) if tall else (W, H)), tall)
    spec = kc.SepSpec("sep_%s" % ("tall" if tall else "wide"), B=1, Cin=16, Cout=24, H=H, W=W, real=len(org), lead=len(org), pre=16,
                      dsts=(("buf", 8, 8), ("stack", 0, 0)), seed=781 + tall)
    _check_peak(spec.name, H * W * (spec.Cout + 8) * 8 * 6)
    case = kc.make_sep(spec, dtype, DEV)
    case.idx = torch.tensor(org, dtype=torch.int32, device=DEV)
    expects = kc.sep_reference(case)
    d = kc.sep_descriptor(case)
    lib = _lib()

    def call(flags):
        d.flags = flags
        return lib.sige_separable_conv(byref(d), _stream())

    _run_and_check("separable", "%s %s (%d x %d)" % (spec.name, NAME[dtype], H, W), case, expects, call, (0, kc.PDL))


@DTYPES2
def test_separable_conv_destination_past_2_to_the_31_elements(dtype):
    """The last 64 channels of a [1, 1024, 1024, 2048] destination (2^31 elements), with a tile on its last pixel.  The values
    and bounds are those of the same launch into a stack (checked first), placed at the tiles' output pixels."""
    from ctypes import byref

    dH, dW, dC, Cout = 1024, 1024, 2048, 64
    org = [(-1, -1), (-1, dW - 5), (511, 507), (dH - 5, -1), (dH - 9, dW - 9), (dH - 5, dW - 5)]
    es = torch.empty((), dtype=dtype).element_size()
    _check_peak("separable 2^31", dH * dW * dC * es + 2 * ec.CHUNK * 8)
    spec = kc.SepSpec("sep_dst_2_31", B=1, Cin=16, Cout=Cout, H=dH, W=dW, real=len(org), lead=len(org), dsts=(("stack", 0, 0),), seed=791)
    case = kc.make_sep(spec, dtype, DEV)
    case.idx = torch.tensor(org, dtype=torch.int32, device=DEV)
    expects = kc.sep_reference(case)
    d = kc.sep_descriptor(case)
    lib = _lib()
    label = "separable %s into %d x %d x %d" % (NAME[dtype], dH, dW, dC)
    _run_and_check("separable", label + " (stack)", case, expects, lambda flags: lib.sige_separable_conv(byref(d), _stream()))
    g, e = case.dst[0], expects[0]
    want = e.want[g.off:g.off + g.view.numel()].view(g.view.shape)                     # [N, 4, 4, Cout]
    bound = e.bound[g.off:g.off + g.view.numel()].view(g.view.shape)
    big = torch.empty(dH * dW * dC, dtype=dtype, device=DEV)
    ec.fill(big, 792)
    br = d.branch[0]
    br.dst, br.dst_is_stack, br.dH, br.dW, br.dst_C, br.dst_c0 = big.data_ptr(), 0, dH, dW, dC, dC - Cout
    n, r, s, h, w = (t.to(DEV) for t in ec.tile_pixels(org, 4, 1, 1, dH, dW))
    pos = ((h * dW + w) * dC + dC - Cout)[:, None] + torch.arange(Cout, device=DEV)
    assert int(pos.max()) == big.numel() - 1
    first = None
    for _ in range(2):
        assert lib.sige_separable_conv(byref(d), _stream()) == 0, lib.sige_last_error()
        torch.cuda.synchronize()
        ec.unchanged_outside(label, big, 792, lambda i: torch.isin(i, pos))
        got = big[pos]
        err = (got.double() - want[n, r, s]).abs()
        ratio = torch.where(err == 0, torch.zeros_like(err), err / bound[n, r, s])
        assert float(ratio.max()) <= 1, "%s: %d elements over their bound" % (label, int((ratio > 1).sum()))
        assert first is None or torch.equal(kc.bits(got), kc.bits(first)), "%s: a second launch differs" % label
        first = got
    print("[extent contract] %-56s worst |err| / bound %.3f" % (label, float(ratio.max())))


# ---------------------------------------------------------------------------------------------------------------- D = 512 attention
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@DTYPES2
def test_wide_sparse_attention_keys_past_2_to_the_31_elements(dtype):
    """D = 512: keys and values are the first and last 512 columns of the rows of one [2^15 + 1, 2^16] buffer, so k_sn * Nk =
    2^31 + 2^16 and the last value ends on the buffer's last element; 64 queries split the 1025 key blocks over a cluster of 8.
    Checked against step_kernel_contracts.wide_sattn_reference (four queries at a time: [4, Nk, D] float64 is 0.5 GiB)."""
    Nk, kn, D, Nq = 2 ** 15 + 1, 2 ** 16, 512, 64
    es = torch.empty((), dtype=dtype).element_size()
    _check_peak("wide sparse attention keys 2^31", Nk * kn * es + 2 * ec.CHUNK * 8 + 2 * Nk * D * 8 + 4 * 4 * Nk * D * 8)
    flat = torch.empty(Nk * kn, dtype=dtype, device=DEV)
    ec.fill(flat, 781)
    rows = flat.view(Nk, kn)
    k, v = rows[:, :D][None, None], rows[:, kn - D:][None, None]
    g = torch.Generator(device=DEV)
    g.manual_seed(781)
    spec = sk.SAttnSpec("wide_keys_past_2_31", 1, 1, Nq, Nk, D, seed=781)
    assert sk.wide_cluster(Nq, Nk, 1, _sms()) == 8
    q = (torch.randn(1, 1, Nq, D, generator=g, device=DEV) * 2 / (spec.s32 * D ** 0.5)).to(dtype)
    out = kc.guarded((1, 1, Nq, D), dtype, DEV, g, "bhnd")
    case = sk.SAttnCase(spec, dtype, q, k, v, {"q": q}, out, out.view)
    expects = sk.wide_sattn_reference(case, _sms(), chunk=4)
    lib = _lib()
    label = "sparse_attention d512 %s (k_sn %d x Nk %d, cluster 8)" % (NAME[dtype], kn, Nk)
    _run_and_check("sattn", label, case, expects, lambda flags: sk.sattn_call(case, lib))
    ec.unchanged_outside(label, flat, 781, lambda i: torch.zeros_like(i, dtype=torch.bool))


@DTYPES2
def test_wide_sparse_attention_output_rows_past_2_to_the_31_elements(dtype):
    """D = 512: the output rows are the last 512 columns of the rows of one [2^15 + 1, 2^16] buffer, so o_sn * Nq = 2^31 + 2^16;
    64 keys and 513 query blocks give a cluster of 1.  The float64 restatement (wide_sattn_reference, 64 queries at a time: with 64
    keys [queries, Nk, D] is small) is written into a [Nq, D] stand-in; every element of the big buffer outside those columns
    stays bitwise as it was filled."""
    Nq, on, D, Nk = 2 ** 15 + 1, 2 ** 16, 512, 64
    es = torch.empty((), dtype=dtype).element_size()
    _check_peak("wide sparse attention output 2^31", Nq * on * es + 2 * ec.CHUNK * 8 + 6 * Nq * D * 8 + Nq * D * es)
    flat = torch.empty(Nq * on, dtype=dtype, device=DEV)
    ec.fill(flat, 782)
    o4 = flat.view(Nq, on)[:, on - D:][None, None]
    spec = sk.SAttnSpec("wide_out_past_2_31", 1, 1, Nq, Nk, D, seed=782)
    assert sk.wide_cluster(Nq, Nk, 1, _sms()) == 1
    qv, kv_, vv = sk.sattn_values(spec, DEV)
    q, k, v = (t.to(dtype).contiguous() for t in (qv, kv_, vv))
    del qv, kv_, vv
    g = torch.Generator(device=DEV)
    g.manual_seed(782)
    stand_in = kc.guarded((1, 1, Nq, D), dtype, DEV, g, "bhnd")
    case = sk.SAttnCase(spec, dtype, q, k, v, {"q": q, "k": k, "v": v}, stand_in, o4)
    (e,) = sk.wide_sattn_reference(case, _sms(), chunk=64)
    n = Nq * D
    want, bound = e.want[stand_in.off:stand_in.off + n].view(Nq, D), e.bound[stand_in.off:stand_in.off + n].view(Nq, D)
    del e
    inputs0 = [t.clone() for t in (q, k, v)]
    lib = _lib()
    label = "sparse_attention d512 %s (o_sn %d x Nq %d, cluster 1)" % (NAME[dtype], on, Nq)
    first, worst = None, 0.0
    for launch in range(2):
        assert sk.sattn_call(case, lib) == 0, lib.sige_last_error()
        torch.cuda.synchronize()
        ec.unchanged_outside(label, flat, 782, lambda i: i % on >= on - D)
        assert all(torch.equal(kc.bits(a), kc.bits(b)) for a, b in zip((q, k, v), inputs0)), "%s: an input changed" % label
        got = o4[0, 0]
        if launch == 0:
            first = got.clone()
            for r0 in range(0, Nq, 4096):
                err = (got[r0:r0 + 4096].double() - want[r0:r0 + 4096]).abs()
                ratio = torch.nan_to_num(torch.where(err == 0, torch.zeros_like(err), err / bound[r0:r0 + 4096]), nan=float("inf"))
                r = float(ratio.max())
                if r > 1:
                    i, c = (int(z) for z in (ratio == ratio.max()).nonzero()[0])
                    raise AssertionError("%s: query %d channel %d: got %r, want %r, bound %.3g"
                                         % (label, r0 + i, c, float(got[r0 + i, c]), float(want[r0 + i, c]), float(bound[r0 + i, c])))
                worst = max(worst, r)
        else:
            assert torch.equal(kc.bits(got), kc.bits(first)), "%s: a second launch differs" % label
    print("[extent contract] %-56s worst |err| / bound %.3f" % (label, worst))


# ---------------------------------------------------------------------------------------------------------------- cache load
@DTYPES2
@pytest.mark.parametrize("what", ["raw", "swish_view"])
def test_cache_load_destination_past_2_to_the_31_elements(what, dtype):
    """sige_cache_load of one image's f32 cache (C = 256, 2048 x 2049 pixels) into a channels-last destination of E = 2 images:
    2^31 + 2^20 elements, followed by a guard band of 2^16 in one buffer.  raw: the cache in `dtype`, bitwise, in both images;
    swish_view: swish(cache * scale + shift) within fused_step_contract.cached_view's bound.  Every other element of the buffer
    bitwise as it was filled; a second launch bitwise identical."""
    import fused_step_contract as fsc
    from sige_b200 import ops

    E, C, H, W, guard = 2, 256, 2048, 2049, 2 ** 16
    n = E * C * H * W
    assert n == 2 ** 31 + 2 ** 20
    es = torch.empty((), dtype=dtype).element_size()
    rows = 32                                                               # image rows per check chunk
    _check_peak("cache_load 2^31", (n + guard) * es + C * H * W * 4 + max(2 * ec.CHUNK * 8, 6 * rows * W * C * 8, 3 * (1 << 24) * 8))
    flat = torch.empty(n + guard, dtype=dtype, device=DEV)
    ec.fill(flat, 791)
    dst = flat[:n].view(E, H, W, C).permute(0, 3, 1, 2)                    # channels-last [E, C, H, W]
    g = torch.Generator(device=DEV)
    g.manual_seed(791)
    src = torch.randn(1, C, H, W, generator=g, device=DEV)
    sc = (1 + 0.3 * torch.randn(C, generator=g, device=DEV)).float()
    sh = (0.4 * torch.randn(C, generator=g, device=DEV)).float()
    entry = (src, dst, []) if what == "raw" else (src, None, [(dst, sc, sh, "swish")])
    run = ops.cache_load_launcher([entry], dtype)
    label = "cache_load %s %s (E 2 x %d elements)" % (what, NAME[dtype], C * H * W)

    def digest():                    # per chunk of the destination: a position-weighted sum of its bits (a second launch's check)
        out = []
        for k in range(0, n, 1 << 24):
            b = kc.bits(flat[k:min(k + (1 << 24), n)]).long()
            out.append(int((b * (torch.arange(b.numel(), device=DEV) % 65521 + 1)).sum()))
        return out

    worst = 0.0
    run(_stream())
    torch.cuda.synchronize()
    ec.unchanged_outside(label, flat, 791, lambda i: i < n)
    for e in range(E):
        for h0 in range(0, H, rows):
            c = src[:, :, h0:h0 + rows]
            got = dst[e:e + 1, :, h0:h0 + rows]
            if what == "raw":
                same = kc.bits(got.contiguous()) == kc.bits(c.to(dtype).contiguous())
                if not bool(same.all()):
                    _, ch, hh, ww = (int(z) for z in (~same).nonzero()[0])
                    raise AssertionError("%s: image %d (c, h, w) = (%d, %d, %d) is not the cache bit for bit" % (label, e, ch, h0 + hh, ww))
                continue
            want, bound = fsc.cached_view(c, sc, sh, "swish", dtype)
            ratio = torch.nan_to_num((got.double() - want).abs() / bound, nan=float("inf"))
            r = float(ratio.max())
            if r > 1:
                _, ch, hh, ww = (int(z) for z in (ratio == ratio.max()).nonzero()[0])
                raise AssertionError("%s: image %d (c, h, w) = (%d, %d, %d): got %r, want %r"
                                     % (label, e, ch, h0 + hh, ww, float(got[0, ch, hh, ww]), float(want[0, ch, hh, ww])))
            worst = max(worst, r)
            del want, bound, ratio
    first = digest()
    run(_stream())
    torch.cuda.synchronize()
    assert digest() == first, "%s: a second launch differs" % label
    ec.unchanged_outside(label, flat, 791, lambda i: i < n)
    print("[extent contract] %-56s worst |err| / bound %.3f" % (label, worst))
