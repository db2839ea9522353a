"""Stride-2 downsample (3x3 s2 on 5x5 tiles): wgmma kernel vs mma.sync kernel as a function of the tile count.
Device time per launch = 20 PDL-chained launches captured in one CUDA graph, replayed 10 times."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from sige_b200 import ops

DEV = "cuda:0"
dtype = torch.float16


def make(B, C, Co, H, ntiles):
    x = torch.randn(B, C, H, H, device=DEV, dtype=dtype).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(Co, C, 3, 3, device=DEV) / (C * 9) ** 0.5).to(dtype)
    wp = ops.pack_conv_weight(w, dtype)
    bias = torch.randn(Co, device=DEV)
    g = H // 4
    ii, jj = torch.meshgrid(torch.arange(0, 4 * g, 4), torch.arange(0, 4 * g, 4), indexing="ij")
    idx = torch.stack([ii.reshape(-1), jj.reshape(-1)], 1)[:ntiles].to(torch.int32).to(DEV).contiguous()
    out = torch.zeros(B, Co, H // 2, H // 2, device=DEV, dtype=dtype).contiguous(memory_format=torch.channels_last)
    d = ops.tile_conv_descriptor()
    d.dtype = ops._dt(x); d.n_src = 1
    d.src[0].ptr, d.src[0].C, d.src[0].up = x.data_ptr(), C, 0
    d.B, d.H, d.W = B, H, H
    d.idx, d.N = idx.data_ptr(), idx.shape[0]
    d.R = d.S = 5
    d.scale = d.shift = None
    d.affine_bstride, d.act = 0, 0
    d.w_packed, d.bias = wp.data_ptr(), bias.data_ptr()
    d.Cin, d.Cout, d.kH, d.kW, d.stride = C, Co, 3, 3, 2
    d.dst, d.dst_is_stack = out.data_ptr(), 0
    d.dH, d.dW, d.dC, d.dst_c0 = H // 2, H // 2, Co, 0
    d.offH = d.offW = 0
    d.residual = None
    d._keep = (x, wp, bias, idx, out)
    return d


def time_graph(d, n=20, reps=10):
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
    torch.cuda.synchronize()
    return 1e3 * a.elapsed_time(b) / (n * reps)


for (B, C, H, tiles) in [(1, 128, 256, [16, 32, 64, 128, 256, 512, 1024, 4096]), (1, 128, 128, [16, 64, 256, 1024]), (1, 256, 64, [16, 64, 256]),
                         (1, 256, 32, [64]), (2, 256, 32, [64]), (4, 256, 32, [64]), (8, 256, 32, [64]),
                         (1, 512, 16, [16]), (2, 512, 16, [16]), (4, 512, 16, [16]), (8, 512, 16, [16])]:
    for n in tiles:
        d = make(B, C, C, H, n)
        res = []
        for flags in (1, 3):          # PDL | (TC5)
            d.flags, d.ksplit = flags, 0
            res.append(time_graph(d))
        print("B %d C %d H %d tiles/img %d (NT %d): mma %.2f us  tc5 %.2f us  -> %s" % (B, C, H, n, B * n, res[0], res[1], "tc5" if res[1] < res[0] else "mma"), flush=True)
