"""The size limits of the C ABI, at the limit and one step inside it, on the host (no GPU, no launch).

  * The wgmma tile conv keeps 32-bit element offsets, so sige_tile_conv_plan must route a launch to mma.sync exactly when a
    source's pixels x pitch, or the destination's pixel count, reaches 2^31 — for every source form tc5_supported measures.
  * Each size guard refuses the first value past its limit with a message that names it.  One step inside, the descriptor is
    made to fail a check that comes AFTER the guard (a bad ksplit, n_aux or dtype), so the call is seen to pass the guard
    without anything being launched.  (sige_sparse_attention's B * heads and sige_tile_writeback's per-call tile count are the
    last checks before their launches: only the refusal side is tested here.)
  * The counts and products that used to be ints: the tiled stem's B * n_tiles, the GroupNorm fold's H * W and workspace
    size, reduce_mask's candidate grid (and the -1 of its capacity query) and get_scatter_map's tile pixels.  A restatement of
    the tiled stem's grid-stride loop in int32 shows the wrap the 64-bit index removes.

The pointers below are not device memory; only host checks may look at them.
"""
import ctypes

import pytest

from extent_contract import HOST_PTR as P
from extent_contract import host_tile_conv as _host_desc

WGMMA, MMA = 1, 0


def _plan(d):
    from sige_b200 import _cabi

    p = _cabi.TileConvPlan()
    assert _cabi.lib().sige_tile_conv_plan(ctypes.byref(d), ctypes.byref(p)) == 0, _cabi.last_error()
    return p.path


def _plain(H, W):
    d = _host_desc(cin=64, cout=64)
    d.H, d.W, d.dH, d.dW = H, W, 64, 64
    return d


def _window(H, W, pitch):
    d = _plain(H, W)
    d.src_pixel_stride = pitch
    return d


def _concat(H, W, c0, c1):
    d = _plain(H, W)
    d.n_src = 2
    d.src[0].C, d.src[1].ptr, d.src[1].C = c0, P, c1
    d.Cin = c0 + c1
    return d


def _stack_src(N):
    d = _host_desc(cin=64, cout=64, k=1, N=N)
    d.src_is_stack, d.H, d.W = 1, 4, 4
    return d


def _full_dst(B, dH, dW):
    d = _host_desc(cin=64, cout=64)
    d.B, d.dH, d.dW = B, dH, dW
    return d


def _stack_dst(N):
    d = _host_desc(cin=64, cout=64, k=1, N=N)
    d.dst_is_stack = 1
    return d


# (form, descriptor at the last product below 2^31 the form can take, descriptor at 2^31, the two products)
SWITCH = [
    ("plain", lambda: _plain(18631, 1801), lambda: _plain(32768, 1024), (18631 * 1801 * 64, 2 ** 31)),
    ("window", lambda: _window(3683, 4859, 120), lambda: _window(4096, 4096, 128), (3683 * 4859 * 120, 2 ** 31)),
    ("concat_first", lambda: _concat(4095, 4097, 128, 64), lambda: _concat(4096, 4096, 128, 64), (4095 * 4097 * 128, 2 ** 31)),
    ("concat_second", lambda: _concat(4095, 4097, 64, 128), lambda: _concat(4096, 4096, 64, 128), (4095 * 4097 * 128, 2 ** 31)),
    ("stack_src", lambda: _stack_src(2 ** 21 - 1), lambda: _stack_src(2 ** 21), ((2 ** 21 - 1) * 16 * 64, 2 ** 31)),
    ("full_dst", lambda: _full_dst(1, 1, 2 ** 31 - 1), lambda: _full_dst(2, 32768, 32768), (2 ** 31 - 1, 2 ** 31)),
    ("stack_dst", lambda: _stack_dst(2 ** 27 - 1), lambda: _stack_dst(2 ** 27), ((2 ** 27 - 1) * 16, 2 ** 31)),
]


@pytest.mark.parametrize("form,below,at,sizes", SWITCH, ids=[s[0] for s in SWITCH])
def test_wgmma_to_mma_switch_lands_on_2_to_the_31(cabi_lib, form, below, at, sizes):
    """`below` is the last product under 2^31 the form can take, within 2048 elements (the window's within 8)."""
    lo, hi = sizes
    assert lo < 2 ** 31 <= hi and 2 ** 31 - lo <= (8 if form == "window" else 2048), (form, lo)
    assert _plan(below()) == WGMMA, "%s: %d elements must stay on the wgmma kernel" % (form, lo)
    assert _plan(at()) == MMA, "%s: %d elements must go to mma.sync" % (form, hi)


# ---------------------------------------------------------------------------------------------------------------- size guards
def _err():
    from sige_b200 import _cabi

    return _cabi.last_error()


def _tile_conv(H, W, ksplit=0):
    from sige_b200 import _cabi

    d = _host_desc(cin=64, cout=64)
    d.H, d.W, d.ksplit = H, W, ksplit
    return _cabi.lib().sige_tile_conv(ctypes.byref(d), None)


@pytest.mark.parametrize("axis", ["H", "W"])
def test_tile_conv_extent_guard(cabi_lib, axis):
    hw = {"H": (65536, 64), "W": (64, 65536)}[axis]
    assert _tile_conv(*hw) != 0 and "extent too large" in _err()
    inside = tuple(v - 1 if v == 65536 else v for v in hw)
    assert _tile_conv(*inside, ksplit=9) != 0
    assert "ksplit out of range" in _err(), _err()


def _conv_in(H, n_aux):
    from sige_b200 import _cabi

    # total = B * H * (W / 4) * (Cout / 8) = H; refused once total * 4 reaches 2^31 - 1
    return _cabi.lib().sige_conv_in_nhwc(P, P, None, P, _cabi.F16, 1, H, 4, 3, 8, n_aux, None, None)


def test_conv_in_nhwc_size_guard(cabi_lib):
    assert _conv_in(2 ** 29, 0) != 0 and "sige_conv_in_nhwc: tensor too large" in _err()
    assert _conv_in(2 ** 29 - 1, 3) != 0 and "n_aux must be 0..2" in _err(), _err()


def _conv_in_tiles(B, H, W, n_tiles, n_aux):
    from sige_b200 import _cabi

    return _cabi.lib().sige_conv_in_nhwc_tiles(P, P, None, P, _cabi.F16, B, H, W, 3, 8, P, n_tiles, 1, 1, 0, n_aux, None, None)


def test_conv_in_nhwc_tiles_size_guards(cabi_lib):
    # tile outputs: n_tiles * R * S * (Cout / 8) < 2^31 - 1
    assert _conv_in_tiles(1, 8, 8, 2 ** 31 - 1, 0) != 0 and "sige_conv_in_nhwc_tiles: tensor too large" in _err()
    assert _conv_in_tiles(1, 8, 8, 2 ** 31 - 2, 3) != 0 and "n_aux must be 0..2" in _err(), _err()
    # the full tensor: B * H * W * Cout < (2^31 - 1) * 8
    assert _conv_in_tiles(1, 1, 2 ** 31 - 1, 1, 0) != 0 and "sige_conv_in_nhwc_tiles: tensor too large" in _err()
    assert _conv_in_tiles(1, 1, 2 ** 31 - 2, 1, 3) != 0 and "n_aux must be 0..2" in _err(), _err()


@pytest.mark.parametrize("dtype", ["F16", "BF16"])
@pytest.mark.parametrize("cin,cout", [(4, 1552), (2, 2984), (1, 5536)])
def test_conv_in_refuses_weights_beyond_shared_memory(cabi_lib, cin, cout, dtype):
    """The first stem per Cin whose staged weights, 4 ((Cout / 8) pitch(Cin) + Cout) bytes, pass 227 KB (Cin 4: 232,800 B) is
    refused by both entry points before any CUDA call; the accepting side (Cout 1544 at Cin 4) is a GPU contract case, since it
    calls cudaFuncSetAttribute."""
    from sige_b200 import _cabi

    lib, dt = _cabi.lib(), getattr(_cabi, dtype)
    assert lib.sige_conv_in_nhwc(P, P, None, P, dt, 1, 8, 8, cin, cout, 0, None, None) != 0
    assert "sige_conv_in_nhwc: weights do not fit in shared memory" in _err(), _err()
    assert lib.sige_conv_in_nhwc_tiles(P, P, None, P, dt, 1, 8, 8, cin, cout, P, 1, 6, 6, 0, 0, None, None) != 0
    assert "sige_conv_in_nhwc_tiles: weights do not fit in shared memory" in _err(), _err()


def _entry(N, B=1, src_dtype=None):
    from sige_b200 import _cabi

    e = _cabi.WritebackEntry()
    e.src, e.dst, e.idx, e.N, e.B, e.C, e.H, e.W = P, P, P, N, B, 64, 64, 64
    e.src_dtype = _cabi.F16 if src_dtype is None else src_dtype
    e.dst_dtype, e.dst_layout = _cabi.F16, _cabi.NHWC
    e.strideH = e.strideW = 1
    e.Ro = e.So = 4
    return e


def _writeback(*entries):
    from sige_b200 import _cabi

    table = (_cabi.WritebackEntry * len(entries))(*entries)
    return _cabi.lib().sige_tile_writeback(table, len(entries), None)


def test_tile_writeback_tile_count_guards(cabi_lib):
    from sige_b200 import _cabi

    # one entry: B * N < 2^31
    assert _writeback(_entry(2 ** 30, B=2)) != 0 and "entry 0: too many tiles" in _err()
    assert _writeback(_entry(2 ** 31 - 1), _entry(1, src_dtype=_cabi.F32)) != 0 and "entry 1: the source must be f16" in _err(), _err()
    # one call: the entries' tiles together < 2^31
    assert _writeback(_entry(2 ** 30), _entry(2 ** 30)) != 0 and "2147483648 tiles in one call" in _err()


def _attention(B, heads):
    from sige_b200 import _cabi

    a = _cabi.SparseAttention()
    a.q = a.k = a.v = a.out = P
    a.B, a.heads, a.Nq, a.Nk, a.D = B, heads, 1, 1, 32
    for s in (a.q_stride, a.k_stride, a.v_stride, a.out_stride):
        s[0], s[1], s[2] = 32, 32, 32
    a.scale, a.dtype = 1.0, _cabi.F16
    return _cabi.lib().sige_sparse_attention(ctypes.byref(a), None)


@pytest.mark.parametrize("B,heads", [(65536, 1), (256, 256), (1, 65536)])
def test_sparse_attention_grid_guard(cabi_lib, B, heads):
    assert _attention(B, heads) != 0 and "B * heads = 65536 exceeds the grid limit" in _err()


def _generic(Cin, Cout, groups, dtype=None):
    from sige_b200 import _cabi

    dt = _cabi.F16 if dtype is None else dtype
    return _cabi.lib().sige_tile_conv_generic(P, P, None, P, dt, _cabi.NHWC, 1, Cin, 3, 3, Cout, 3, 3, 1, 1, 1, 1, groups, None)


def test_tile_conv_generic_grid_guards(cabi_lib):
    # grid.z = groups <= 65535 (depthwise: groups == Cin == Cout)
    assert _generic(65536, 65536, 65536) != 0 and "sige_tile_conv_generic: grid too large" in _err()
    assert _generic(65535, 65535, 65535, dtype=99) != 0 and "unsupported dtype 99" in _err(), _err()
    # grid.y = ceil(Cout / groups / 64) <= 65535
    assert _generic(8, 65535 * 64 + 1, 1) != 0 and "sige_tile_conv_generic: grid too large" in _err()
    assert _generic(8, 65535 * 64, 1, dtype=99) != 0 and "unsupported dtype 99" in _err(), _err()


def _conv_in_tiles_aux(B, n_tiles, n_aux, R=1, S=1):
    from sige_b200 import _cabi

    return _cabi.lib().sige_conv_in_nhwc_tiles(P, P, None, P, _cabi.F16, B, 1, 1, 3, 8, P, n_tiles, R, S, 0, n_aux, None, None)


def test_conv_in_nhwc_tiles_batch_times_tiles_guard(cabi_lib):
    # B * n_tiles is a 64-bit product: 5 * 2^30 tiles (which wrapped to 2^30 in an int) are refused, not run for image 0 only
    assert _conv_in_tiles_aux(5, 2 ** 30, 0) != 0 and "sige_conv_in_nhwc_tiles: tensor too large" in _err()
    assert _conv_in_tiles_aux(2, 2 ** 30, 0) != 0 and "sige_conv_in_nhwc_tiles: tensor too large" in _err()
    assert _conv_in_tiles_aux(2, 2 ** 30 - 1, 3) != 0 and "n_aux must be 0..2" in _err(), _err()


# the near-limit tiled-stem case of tests/test_gpu_extent_contracts_ops.py: Cin 1, Cout 512, 8 x 8 tiles, 2^19 - 1 tiles
STEM_TILES, STEM_R, STEM_OV = 2 ** 19 - 1, 8, 512 // 8
H100_SMS = 132


def _stem_loop_next(total: int, grid: int, index_bits: int):
    """The value of conv_in_tiles_kernel's grid-stride loop index one step after each thread's last in-range index, with the
    index held in `index_bits` bits (two's complement), for every thread of a `grid` x 256 launch."""
    import numpy as np

    step = grid * 256
    tid = np.arange(step, dtype=np.int64)
    last = tid + (total - 1 - tid) // step * step
    nxt = last + step
    if index_bits == 32:
        nxt = ((nxt + 2 ** 31) % 2 ** 32) - 2 ** 31
    return nxt


def test_conv_in_tiles_loop_index_stays_in_range():
    """Restatement of the stem's grid-stride loop at the near-limit GPU case, on an H100's 132 SMs: with an int index the
    step past the last element wraps negative, the loop goes on, and the tile row `t` it reads is negative (an out-of-bounds
    read of idx); the long long index ends every thread's loop."""
    import numpy as np

    total = STEM_TILES * STEM_R * STEM_R * STEM_OV
    assert total == 2 ** 31 - 4096
    grid = min(-(-total // 256), 4 * H100_SMS)
    old = _stem_loop_next(total, grid, 32)
    again = old < total
    assert again.any() and (old[again] < 0).all()
    c_div = lambda a, d: np.sign(a) * (np.abs(a) // d)    # noqa: E731  (C's int division truncates)
    t = c_div(c_div(c_div(old[again], STEM_OV), STEM_R), STEM_R)
    assert (t < 0).all(), "the wrapped index must reach a negative tile row"
    new = _stem_loop_next(total, grid, 64)
    assert (new >= total).all() and new.max() < 2 ** 63
    assert not np.any(new < total)


def _gn(H, W, B=1, C=8, workspace=0, dtype=None):
    from sige_b200 import _cabi

    dt = _cabi.F16 if dtype is None else dtype
    return _cabi.lib().sige_group_norm_fold(P, dt, B, H, W, C, 1, 1e-5, None, None, P, P, P, workspace, None)


def _gn_blocks():
    from sige_b200 import _cabi

    return _cabi.lib().sige_group_norm_fold_workspace(1, 8) // 16      # B * nblk * C * 2 floats


def test_group_norm_fold_image_guard(cabi_lib):
    assert _gn(65536, 32768) != 0 and "sige_group_norm_fold: image too large (H * W = 2147483648" in _err()
    assert _gn(1, 2 ** 31 - 1) != 0 and "sige_group_norm_fold: workspace too small (0 floats" in _err(), _err()


def test_group_norm_fold_workspace_products(cabi_lib):
    from sige_b200 import _cabi, ops

    lib = _cabi.lib()
    nblk = _gn_blocks()
    per_image = nblk * 1024 * 2
    b_max = (2 ** 31 - 1) // per_image
    assert lib.sige_group_norm_fold_workspace(b_max, 1024) == b_max * per_image
    assert lib.sige_group_norm_fold_workspace(b_max + 1, 1024) == -1 and "exceed 2^31 - 1" in _err()
    with pytest.raises(_cabi.SigeError, match="sige_group_norm_fold_workspace"):
        ops.group_norm_fold_workspace(b_max + 1, 1024)
    # a batch whose int product wrapped to a small power of two, passed as the workspace size: refused as too small
    odd, twos = nblk, 0
    while odd % 2 == 0:
        odd, twos = odd // 2, twos + 1
    B = pow(odd, -1, 2 ** (21 - twos))
    wrapped = B * per_image % 2 ** 32
    assert wrapped == 2 ** (11 + twos) and B * per_image > 2 ** 32
    assert _gn(256, 256, B=B, C=1024, workspace=wrapped) != 0
    assert "workspace too small (%d floats, need %d)" % (wrapped, B * per_image) in _err(), _err()
    # the largest batch whose workspace fits: accepted, and refused by the dtype check that follows
    assert _gn(256, 256, B=b_max, C=1024, workspace=b_max * per_image, dtype=99) != 0
    assert "dtype must be f16/bf16" in _err(), _err()


# (H, W, strideH, pad) -> nI * nJ candidate tiles
CANDIDATES_PAST = [((46340, 46340, 1, 0), 46341 ** 2), ((65535, 32767, 1, 0), 2 ** 31), ((1, 2 ** 31 - 1, 2, 0), 2 ** 31),
                   ((65535, 65535, 1, 0), 2 ** 32)]
CANDIDATES_INSIDE = [((46339, 46339, 1, 0), 46340 ** 2), ((65535, 32766, 1, 0), 2 ** 31 - 2 ** 16),
                     ((1, 2 ** 31 - 2, 2, 0), 2 ** 31 - 1)]


@pytest.mark.parametrize("geom,n", CANDIDATES_PAST + CANDIDATES_INSIDE)
def test_reduce_mask_capacity_at_the_candidate_limit(cabi_lib, geom, n):
    from sige_b200 import _cabi

    H, W, sh, pad = geom
    cap = _cabi.lib().sige_reduce_mask_capacity(H, W, 1, 1, sh, 1, pad, pad)
    if n < 2 ** 31:
        assert cap == n
    else:
        assert cap == -1 and "sige_reduce_mask_capacity: too many candidate tiles (%d" % n in _err(), (cap, _err())


def _reduce_mask(H, W, sh, capacity, batched):
    from sige_b200 import _cabi

    lib = _cabi.lib()
    if batched:
        return lib.sige_reduce_mask_batched(P, 1, H, W, 1, 1, sh, 1, 0, 0, None, capacity, P, P, None)
    return lib.sige_reduce_mask(P, H, W, 1, 1, sh, 1, 0, 0, None, capacity, P, None)


@pytest.mark.parametrize("batched", [False, True], ids=["single", "batched"])
def test_reduce_mask_candidate_guard(cabi_lib, batched):
    name = "sige_reduce_mask_batched" if batched else "sige_reduce_mask"
    for (H, W, sh, _), n in CANDIDATES_PAST:
        assert _reduce_mask(H, W, sh, 1, batched) != 0
        assert "%s: too many candidate tiles (%d" % (name, n) in _err(), _err()
    for (H, W, sh, _), n in CANDIDATES_INSIDE:
        assert _reduce_mask(H, W, sh, 1, batched) != 0 and "idx_out is null" in _err(), _err()


def _scatter_map(N, R, S, k, idx=None):
    from sige_b200 import _cabi

    return _cabi.lib().sige_get_scatter_map(64, 64, R, S, k, k, 0, 0, 1, 1, idx, N, P, None)


def test_get_scatter_map_counts(cabi_lib):
    # N * Ro * So = 2^28 * 4 * 4 = 2^32 tile pixels (0 in an int): past every host check, up to the index list
    assert _scatter_map(2 ** 28, 6, 6, 3) != 0 and "sige_get_scatter_map: null index list" in _err(), _err()
    # the grid: ceil(N * Ro * So / 256) <= 2^31 - 1 blocks
    assert _scatter_map(2 ** 31 - 1, 16, 17, 1) != 0 and "sige_get_scatter_map: grid too large" in _err(), _err()
    assert _scatter_map(2 ** 31 - 1, 16, 16, 1) != 0 and "sige_get_scatter_map: null index list" in _err(), _err()
