"""Split-K narrow 3x3 wgmma launches in both halo layouts: one halo buffer + five weight stages, or two halo buffers + two
weight stages fed from L2 (chosen per launch from the K slices).  Each layout matches the oracle, and the two are
bitwise equal: they issue the same MMAs in the same order on every rank."""
import numpy as np
import pytest
import torch

from test_gpu_conv import TC5, _fused_desc, _round, T, rel_err

pytestmark = pytest.mark.gpu

# (main Cin, shortcut input channels or (), Cout, K split): the split 3x3 shape classes of a DDPM-256 step — up-path convs with a
# fused 1x1 shortcut whose last ranks hold only shortcut steps (e.g. 512 + 1024 at ksplit 8), and plain 3x3 layers
CASES = [(256, (512, 256), 256, 2), (256, (256, 256), 256, 2), (512, (512, 512), 512, 4), (512, (512, 256), 512, 4),
         (512, (512, 512), 512, 8), (256, (), 256, 2), (512, (), 512, 4), (512, (), 512, 8)]


def _set_halo(n):
    from sige_b200 import _cabi

    _cabi.check(_cabi.lib().sige_debug_set_split_halo_buffers(n), "sige_debug_set_split_halo_buffers")


def test_debug_setter_rejects_other_values():
    from sige_b200 import _cabi

    assert _cabi.lib().sige_debug_set_split_halo_buffers(3) != 0
    _set_halo(0)


@pytest.mark.parametrize("preop", [False, True], ids=["cp_async_gather", "register_gather"])
@pytest.mark.parametrize("case", CASES, ids=lambda c: "%d+%d-%d-ks%d" % (c[0], sum(c[1]), c[2], c[3]))
def test_split_halo_layouts_match_oracle_and_each_other(oracle, case, preop):
    from sige_b200 import ops

    Cm, Cx2, Co, ks = case
    dtype = torch.float16
    rng = np.random.default_rng(Cm + sum(Cx2) + ks)
    B, H, W = 1, 32, 32
    mask = np.zeros((H, W), bool)
    mask[5:19, 9:20] = True                      # a ragged number of tiles (not a multiple of 8 per CTA)
    mask[30, 2] = True
    idx0 = oracle.reduce_mask(mask, 6, 4, 1)
    assert idx0.shape[0] % 8 != 0
    t1 = _round(rng.standard_normal((B, Cm, H, W)).astype(np.float32), dtype)
    w2 = _round(rng.standard_normal((Co, Cm, 3, 3)).astype(np.float32) / np.sqrt(Cm * 9), dtype)
    b2 = rng.standard_normal((Co,)).astype(np.float32)
    y0 = _round(rng.standard_normal((B, Co, H, W)).astype(np.float32), dtype)
    sc = sh = None
    src = t1
    if preop:                                    # affine + SiLU in the gather: the register-staged path
        sc = (1 + 0.2 * rng.standard_normal((1, Cm, 1, 1))).astype(np.float32)
        sh = (0.2 * rng.standard_normal((1, Cm, 1, 1))).astype(np.float32)
        z = t1 * sc + sh
        src = z / (1 + np.exp(-z))
    main_tiles = oracle.conv2d_tiles(oracle.gather(src, 6, 6, idx0), w2, b2, (1, 1))
    out = T(y0, dtype, cl=True).clone(memory_format=torch.channels_last)
    kw = {}
    if preop:
        kw = dict(scale=T(sc).reshape(-1).contiguous(), shift=T(sh).reshape(-1).contiguous(), act=1)
    if Cx2:
        xs = [_round(rng.standard_normal((B, c, H, W)).astype(np.float32), dtype) for c in Cx2]
        xcat = np.concatenate(xs, 1)
        Cx = xcat.shape[1]
        wsc = _round(rng.standard_normal((Co, Cx, 1, 1)).astype(np.float32) / np.sqrt(Cx), dtype)
        bsc = rng.standard_normal((Co,)).astype(np.float32)
        y1 = _round(rng.standard_normal((B, Co, H, W)).astype(np.float32), dtype)
        idx1 = oracle.reduce_mask(mask, 4, 4, 0)
        sc_tiles = oracle.conv2d_tiles(oracle.gather(xcat, 4, 4, idx1), wsc, bsc, (1, 1))
        want = oracle.scatter_with_block_residual(main_tiles, y0, sc_tiles, y1, 1, 1, 1, 1, idx0, idx1)
        keys1 = {(int(a), int(b)) for a, b in idx1}
        flags = np.array([1 if (int(a) + 1, int(b) + 1) in keys1 else 0 for a, b in idx0], dtype=np.uint8)
        d = _fused_desc(ops, T(t1, dtype, cl=True), ops.pack_conv_weight(T(w2, dtype), dtype), T(b2), T(idx0), out, R=6, k=3, stride=1,
                        off=1, residual=T(y1, dtype, cl=True), **kw)
        txs = [T(v, dtype, cl=True) for v in xs]
        wscp, tb, tf = ops.pack_conv_weight(T(wsc, dtype), dtype), T(bsc), torch.from_numpy(flags).to("cuda:0")
        d.n_src2 = len(txs)
        for i, t in enumerate(txs):
            d.src2[i].ptr, d.src2[i].C, d.src2[i].up = t.data_ptr(), t.shape[1], 0
        d.Cin2, d.w2_packed, d.bias2, d.sc_flags = Cx, wscp.data_ptr(), tb.data_ptr(), tf.data_ptr()
        keep = (txs, wscp, tb, tf)
    else:
        want = oracle.scatter(main_tiles, y0, 1, 1, 1, 1, idx0, None)
        d = _fused_desc(ops, T(t1, dtype, cl=True), ops.pack_conv_weight(T(w2, dtype), dtype), T(b2), T(idx0), out, R=6, k=3, stride=1,
                        off=1, **kw)
        keep = ()
    d.flags, d.ksplit = TC5, ks
    got = {}
    try:
        for n in (1, 2, 0):
            _set_halo(n)
            out.copy_(T(y0, dtype, cl=True))
            ops.launch_tile_conv(d, torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
            got[n] = out.clone()
            e = rel_err(out, want)
            assert e <= 2e-3, "case %s preop %s, %d halo buffers: rel err %g" % (case, preop, n, e)
    finally:
        _set_halo(0)
    del keep
    assert torch.equal(got[1], got[2]), "the two halo layouts differ by %g" % float((got[1].float() - got[2].float()).abs().max())
    assert torch.equal(got[0], got[1])
