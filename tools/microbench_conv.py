"""Micro-benchmark of the fused tile-conv kernels (development aid, GPU only).

For a few representative DDPM layer shapes: time N back-to-back launches (warm L2) and N launches with an L2
flush before each (cold), for the mma.sync and the wgmma kernel and every split-K factor."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from sige_b200 import ops

DEV = "cuda:0"
dtype = torch.float16


def make(tiles_hw, H, Cin, Cout, k, all_tiles=False):
    x = torch.randn(1, Cin, H, H, device=DEV, dtype=dtype).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(Cout, Cin, k, k, device=DEV) / (Cin * k * k) ** 0.5).to(dtype)
    wp = ops.pack_conv_weight(w, dtype)
    bias = torch.randn(Cout, device=DEV)
    off = 1 if k == 3 else 0
    n = tiles_hw
    ii, jj = torch.meshgrid(torch.arange(0, 4 * n, 4), torch.arange(0, 4 * n, 4), indexing="ij")
    idx = (torch.stack([ii.reshape(-1), jj.reshape(-1)], 1) + (H // 2 // 4 * 4 - 2 * n if not all_tiles else 0) - off).to(torch.int32).to(DEV).contiguous()
    out = torch.zeros(1, Cout, H, H, device=DEV, dtype=dtype).contiguous(memory_format=torch.channels_last)
    sc = torch.rand(Cin, device=DEV) + 0.5
    sh = torch.randn(Cin, device=DEV) * 0.1
    d = ops.tile_conv_descriptor()
    d.dtype = ops._dt(x); d.n_src = 1
    d.src[0].ptr, d.src[0].C, d.src[0].up = x.data_ptr(), Cin, 0
    d.B, d.H, d.W = 1, H, H
    d.idx, d.N = idx.data_ptr(), idx.shape[0]
    d.R = d.S = 6 if k == 3 else 4
    d.scale, d.shift, d.affine_bstride, d.act = sc.data_ptr(), sh.data_ptr(), 0, 1
    d.w_packed, d.bias = wp.data_ptr(), bias.data_ptr()
    d.Cin, d.Cout, d.kH, d.kW, d.stride = Cin, Cout, k, k, 1
    d.dst, d.dst_is_stack = out.data_ptr(), 0
    d.dH, d.dW, d.dC, d.dst_c0 = H, H, Cout, 0
    d.offH = d.offW = off
    d.residual = None
    d._keep = (x, wp, bias, idx, out, sc, sh)
    return d


def timeit(d, reps, flush):
    st = torch.cuda.current_stream()
    s = st.cuda_stream
    for _ in range(3):
        ops.launch_tile_conv(d, s)
    torch.cuda.synchronize()
    if flush is None:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st)
        for _ in range(reps):
            ops.launch_tile_conv(d, s)
        b.record(st)
        b.synchronize()
        return 1e3 * a.elapsed_time(b) / reps
    tot = 0.0
    for i in range(reps):
        flush.fill_(i)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st)
        ops.launch_tile_conv(d, s)
        b.record(st)
        b.synchronize()
        tot += a.elapsed_time(b)
    return 1e3 * tot / reps


def time_graph(d, n=20, reps=10):
    """True device time per launch: n launches captured in one CUDA graph, replayed."""
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for _ in range(3):
            ops.launch_tile_conv(d, st.cuda_stream)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        s = torch.cuda.current_stream().cuda_stream
        for _ in range(n):
            ops.launch_tile_conv(d, s)
    g.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        g.replay()
    b.record()
    b.synchronize()
    return 1e3 * a.elapsed_time(b) / (reps * n)


def main():
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)
    shapes = [("64 tiles 128->128 3x3 @256", 8, 256, 128, 128, 3, False), ("16 tiles(all) 1024->512 3x3 @16", 4, 16, 1024, 512, 3, True),
              ("4 tiles(all) 512->512 3x3 @8", 2, 8, 512, 512, 3, True), ("64 tiles 256->128 1x1 @256", 8, 256, 256, 128, 1, False),
              ("1296 tiles 128->128 3x3 @256", 36, 256, 128, 128, 3, False)]
    for name, n, H, Cin, Cout, k, allt in shapes:
        d = make(n, H, Cin, Cout, k, allt)
        print("== %s" % name)
        for flags, kn in ((0, "mma.sync"), (2, "wgmma   "), (1, "mma+pdl "), (3, "tc5+pdl ")):
            row = []
            for ks in (1, 2, 4, 8, 0):
                d.flags, d.ksplit = flags, ks
                try:
                    row.append("ks%d: %5.1f/%5.1f" % (ks, time_graph(d), timeit(d, 10, flush)))
                except Exception as e:  # noqa: BLE001
                    row.append("ks%d: err %s" % (ks, str(e)[:40]))
            print("  %s  graph(warm)/cold us  " % kn + " | ".join(row))
    # empty-kernel launch floor for reference
    z = torch.zeros(1, device=DEV)
    st = torch.cuda.current_stream()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(st)
    for _ in range(200):
        z.add_(1)
    b.record(st)
    b.synchronize()
    print("tiny torch kernel back-to-back: %.2f us" % (1e3 * a.elapsed_time(b) / 200))


if __name__ == "__main__" and "--trace" not in sys.argv:
    main()


def trace(name, d, ks, flags=2):
    """Per-stage timeline (globaltimer, ns) of the wgmma kernel: median over CTAs, relative to the first CTA's start."""
    import ctypes
    from sige_b200 import _cabi
    lib = _cabi.lib()
    lib.sige_debug_set_trace.argtypes = [ctypes.c_void_p]
    buf = torch.zeros(4096 * 16, dtype=torch.int64, device=DEV)
    d.flags, d.ksplit = flags, ks
    s = torch.cuda.current_stream().cuda_stream
    for _ in range(3):
        ops.launch_tile_conv(d, s)
    torch.cuda.synchronize()
    lib.sige_debug_set_trace(buf.data_ptr())
    ops.launch_tile_conv(d, s)
    torch.cuda.synchronize()
    lib.sige_debug_set_trace(None)
    t = buf.view(-1, 16).cpu()
    t = t[t[:, 0] > 0]
    t0 = t[:, 0].min()
    rel = (t - t0).float()
    rel[t == 0] = float("nan")
    names = ["start", "setup", "idx", "ldg", "store", "mmaA", "mmaEnd", "accOut", "rowsIn", "reduce", "stored", "end"]
    med = [float(torch.nanmedian(rel[:, i])) for i in range(12)]
    mx = [float(rel[:, i][~torch.isnan(rel[:, i])].max()) if (~torch.isnan(rel[:, i])).any() else float("nan") for i in range(12)]
    print("  trace %s ks=%d ctas=%d | " % (name, ks, t.shape[0]) + " ".join("%s %.0f/%.0f" % (n, a, b) for n, a, b in zip(names, med, mx)))


if __name__ == "__main__" and "--trace" in sys.argv:
    for name, n, H, Cin, Cout, k, allt in [("64t 128->128 3x3", 8, 256, 128, 128, 3, False), ("16t 1024->512 3x3", 4, 16, 1024, 512, 3, True),
                                           ("64t 256->128 1x1", 8, 256, 256, 128, 1, False)]:
        d = make(n, H, Cin, Cout, k, allt)
        for ks in (1, 4, 8):
            trace(name, d, ks)
