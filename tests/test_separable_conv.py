"""sige_separable_conv: the separable 3x3 convolutions of GAN Compression's sub-mobile SPADE (reference
gaugan/models/mobile_modules.py:65-119) as one launch per SPADE layer.  CPU: the C-ABI's argument checks and shape predicate.
GPU: the kernel against F.conv2d(groups=C) -> affine -> 1x1 in fp32 on the same 16-bit inputs."""
import ctypes
import os

import pytest
import torch
from torch.nn import functional as F

from conftest import REPO

TILE_NONE = -30000


# ---------------------------------------------------------------------------------------------------------------- C-ABI (CPU)
def _desc(cin=48, cout=96, n=8):
    from sige_b200 import _cabi

    d = _cabi.SeparableConv()
    d.dtype, d.src, d.src_is_stack, d.src_C, d.src_c0 = _cabi.F16, 0x10000, 0, 3 * cin, cin
    d.B, d.H, d.W, d.idx, d.N, d.Cin, d.Cout = 1, 64, 128, 0x20000, n, cin, cout
    d.offH = d.offW = 1
    d.nbranch = 2
    for i in range(2):
        b = d.branch[i]
        b.dw_weight, b.pw_weight, b.dst = 0x30000, 0x40000, 0x50000 + 0x1000 * i
        b.dst_is_stack, b.dH, b.dW, b.dst_C, b.dst_c0 = 0, 64, 128, cout, 0
    return d


def test_separable_conv_entry_points_check_arguments_without_a_device(cabi_lib):
    """Bad descriptors return non-zero with a message before any CUDA call (the pointers here are not device memory: a launch
    would fault); N == 0 is a no-op."""
    from sige_b200 import _cabi

    lib = _cabi.lib()
    assert lib.sige_separable_conv(None, None) != 0 and b"null descriptor" in lib.sige_last_error()
    d = _desc(cin=40)
    assert lib.sige_separable_conv(ctypes.byref(d), None) != 0 and b"Cin = 40" in lib.sige_last_error()
    d = _desc()
    d.src_c0 = 2 * 48 + 8          # window [104, 152) of a 144-channel pixel
    assert lib.sige_separable_conv(ctypes.byref(d), None) != 0 and b"channel window" in lib.sige_last_error()
    d = _desc()
    d.branch[1].dst_c0 = 8         # [8, 104) of a 96-channel destination
    assert lib.sige_separable_conv(ctypes.byref(d), None) != 0 and b"destination channel window" in lib.sige_last_error()
    d = _desc()
    d.branch[1].dst = 0x50008      # not 16-byte aligned
    assert lib.sige_separable_conv(ctypes.byref(d), None) != 0 and b"aligned" in lib.sige_last_error()
    d = _desc()
    d.nbranch = 3
    assert lib.sige_separable_conv(ctypes.byref(d), None) != 0 and b"nbranch" in lib.sige_last_error()
    d = _desc()
    d.dtype = _cabi.F32
    assert lib.sige_separable_conv(ctypes.byref(d), None) != 0
    d = _desc(n=0)
    d.src = d.idx = 0
    assert lib.sige_separable_conv(ctypes.byref(d), None) == 0
    d = _desc()
    d.idx = 0
    assert lib.sige_separable_conv(ctypes.byref(d), None) != 0 and b"tile list" in lib.sige_last_error()


def test_separable_conv_predicate_is_host_logic(cabi_lib):
    from sige_b200 import _cabi

    lib = _cabi.lib()
    for cin in (16, 32, 48, 64, 96, 256):
        for cout in (8, 32, 48, 96, 256, 768, 1024):
            assert lib.sige_separable_conv_supported(cin, cout, 3, _cabi.F16) == 1
            assert lib.sige_separable_conv_supported(cin, cout, 3, _cabi.BF16) == 1
    assert lib.sige_separable_conv_supported(48, 96, 3, _cabi.F32) == 0
    assert lib.sige_separable_conv_supported(40, 96, 3, _cabi.F16) == 0
    assert lib.sige_separable_conv_supported(272, 96, 3, _cabi.F16) == 0
    assert lib.sige_separable_conv_supported(48, 100, 3, _cabi.F16) == 0
    assert lib.sige_separable_conv_supported(48, 1032, 3, _cabi.F16) == 0
    assert lib.sige_separable_conv_supported(48, 96, 1, _cabi.F16) == 0


# ---------------------------------------------------------------------------------------------------------------- kernel (GPU)
def _tiles_of(x32, idx):
    """6x6 halo tiles of an fp32 NCHW image at the given origins, zero outside the image."""
    P = 8
    xp = F.pad(x32, (P, P, P, P))
    return torch.stack([xp[0, :, h + P:h + P + 6, w + P:w + P + 6] for h, w in idx.tolist()])


def _reference(tiles32, dw_w, dw_b, scale, shift, pw_w16, pw_b):
    """fp32: depthwise 3x3 -> x*scale + shift -> 1x1 (the 16-bit pointwise weights the kernel reads), [n, Cout, 4, 4]."""
    c = tiles32.shape[1]
    y = F.conv2d(tiles32, dw_w, dw_b, groups=c)
    y = y * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1)
    return F.conv2d(y, pw_w16.float().view(pw_w16.shape[0], c, 1, 1), pw_b)


def _branch(cin, cout, dtype, gen, dev):
    dw_w = torch.randn(cin, 1, 3, 3, generator=gen).to(dev) * 0.3
    dw_b = torch.randn(cin, generator=gen).to(dev) * 0.1
    scale = torch.rand(cin, generator=gen).to(dev) + 0.5
    shift = torch.randn(cin, generator=gen).to(dev) * 0.2
    pw_w = (torch.randn(cout, cin, generator=gen).to(dev) / cin ** 0.5).to(dtype)
    pw_b = torch.randn(cout, generator=gen).to(dev) * 0.1
    return dw_w, dw_b, scale, shift, pw_w, pw_b


# a SPADE layer's (hidden, oc) pairs of the sub-mobile generator and the extremes of the kernel's range
SHAPES = [(16, 32), (32, 48), (48, 96), (64, 256), (96, 768), (96, 32), (16, 768), (48, 256)]


@pytest.mark.gpu
@pytest.mark.parametrize("cin,cout", SHAPES)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("source", ["buffer", "stack"])
@pytest.mark.parametrize("nbranch", [1, 2])
def test_separable_conv_matches_fp32_torch(cin, cout, dtype, source, nbranch):
    from sige_b200 import ops

    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(cin * 1000 + cout)
    H, W = 22, 30
    # origins of 6x6 halo tiles (offset 1): negative at the top-left, ragged at the right and bottom edges; 11 real tiles plus two
    # SIGE_TILE_NONE paddings = 13 (not a multiple of the CTA's 8)
    real = [(-1, -1), (-1, 3), (3, -1), (7, 11), (11, 23), (15, 27), (19, 3), (19, 27), (-1, 27), (11, 11), (3, 19)]
    idx = torch.tensor(real[:6] + [(TILE_NONE, TILE_NONE)] + real[6:] + [(TILE_NONE, TILE_NONE)], dtype=torch.int32, device=dev)
    # the source is a channel window of a wider pixel (torch.split of mlp_shared's output)
    big = torch.randn(1, 3 * cin, H, W, generator=gen).to(dev).to(dtype).contiguous(memory_format=torch.channels_last)
    x_full = big[:, cin:2 * cin]
    x32 = x_full.float()
    tiles32 = torch.zeros(idx.shape[0], cin, 6, 6, device=dev)
    real_rows = [i for i, (h, _) in enumerate(idx.tolist()) if h != TILE_NONE]
    tiles32[real_rows] = _tiles_of(x32, idx[real_rows])
    if source == "stack":
        stack_big = torch.randn(idx.shape[0], 3 * cin, 6, 6, generator=gen).to(dev).to(dtype).contiguous(memory_format=torch.channels_last)
        stack_big[:, cin:2 * cin] = tiles32.to(dtype)
        stack_big[[i for i in range(idx.shape[0]) if i not in real_rows], cin:2 * cin] = 7.0     # rows of padding tiles: never written
        x = stack_big[:, cin:2 * cin]
    else:
        x = x_full
    branches, refs, outs, sentinels = [], [], [], []
    for b in range(nbranch):
        dw_w, dw_b, scale, shift, pw_w, pw_b = _branch(cin, cout, dtype, gen, dev)
        # branch 0 writes a whole buffer, branch 1 a channel window [cout, 2 cout) of a wider one
        width = cout if b == 0 else 2 * cout
        dst_full = torch.randn(1, width, H, W, generator=gen).to(dev).to(dtype).contiguous(memory_format=torch.channels_last)
        dst = dst_full[:, (0 if b == 0 else cout):(cout if b == 0 else 2 * cout)]
        sentinels.append(dst_full.clone())
        outs.append((dst_full, dst))
        w_f, b_f = ops.separable_fold(dw_w, dw_b, scale, shift)
        branches.append((w_f, b_f, pw_w, pw_b, dst))
        refs.append(_reference(tiles32, dw_w, dw_b, scale, shift, pw_w, pw_b))
    ops.separable_conv(x, branches, idx, src_stack=(source == "stack"), offset=1)
    torch.cuda.synchronize()
    tol = 4e-3 if dtype == torch.float16 else 1.6e-2        # bf16: two units in the last place at the largest magnitude
    for b in range(nbranch):
        dst_full, dst = outs[b]
        written = torch.zeros(1, 1, H, W, dtype=torch.bool, device=dev)
        expect = sentinels[b].float().clone()
        c0 = 0 if b == 0 else cout
        for i in real_rows:
            h, w = idx[i].tolist()
            for oy in range(4):
                for ox in range(4):
                    hh, ww = h + 1 + oy, w + 1 + ox
                    if 0 <= hh < H and 0 <= ww < W:
                        written[0, 0, hh, ww] = True
                        expect[0, c0:c0 + cout, hh, ww] = refs[b][i, :, oy, ox]
        got = dst_full.float()
        untouched = ~written.expand_as(got).clone()
        untouched[:, c0 + cout:] = True
        untouched[:, :c0] = True
        assert torch.equal(dst_full[untouched], sentinels[b][untouched]), "pixels outside the active tiles changed"
        scale_ = refs[b][real_rows].abs().max().item()
        err = (got - expect).abs().max().item()
        assert err <= tol * scale_, "branch %d: max error %.3g of max|ref| %.3g" % (b, err / scale_, scale_)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_separable_conv_stack_to_stack(dtype):
    """Stack source and stack destination (no tile list): rows b*N + i in, 4x4 outputs of the same row out."""
    from sige_b200 import ops

    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(5)
    cin, cout, n = 48, 96, 21
    x = torch.randn(n, cin, 6, 6, generator=gen).to(dev).to(dtype).contiguous(memory_format=torch.channels_last)
    dw_w, dw_b, scale, shift, pw_w, pw_b = _branch(cin, cout, dtype, gen, dev)
    out = torch.empty(n, cout, 4, 4, dtype=dtype, device=dev, memory_format=torch.channels_last)
    w_f, b_f = ops.separable_fold(dw_w, dw_b, scale, shift)
    ops.separable_conv(x, [(w_f, b_f, pw_w, pw_b, out)], None, src_stack=True, dst_stack=True)
    ref = _reference(x.float(), dw_w, dw_b, scale, shift, pw_w, pw_b)
    tol = 4e-3 if dtype == torch.float16 else 1.6e-2
    assert (out.float() - ref).abs().max().item() <= tol * ref.abs().max().item()


# ---------------------------------------------------------------------------------------------------------------- lowering (CPU)
def _sim_executors():
    """(SeparableSim, SimExecutor): the descriptor simulator with and without the CPU restatement of sige_separable_conv."""
    import sys

    sys.path.insert(0, os.path.join(REPO, "tests"))
    from sim_executor import SimExecutor

    class SeparableSim(SimExecutor):
        def separable_supported(self, cin, cout):
            """sige_separable_conv_supported(): Cin a multiple of 16 in [16, 256], Cout a multiple of 8 in [8, 1024]."""
            return cin % 16 == 0 and 16 <= cin <= 256 and cout % 8 == 0 and 8 <= cout <= 1024

        def prepare_separable(self, rec):
            """sige_separable_conv: per branch depthwise 3x3 -> x*scale + shift -> 1x1 on the 6x6 halo tiles, 4x4 outputs pasted in
            place at (origin + off); SIGE_TILE_NONE tiles read zeros and write nothing."""
            def run(_stream):
                self.launches += 1
                src = rec.src[:, rec.c0:rec.c0 + rec.Cin].float()
                idx = rec.idx.tolist()
                n = len(idx)
                if rec.src_stack:
                    X = src
                    assert X.shape[0] == rec.batch * n
                else:
                    P = 8
                    padded = F.pad(src, (P, P, P, P))
                    X = torch.stack([padded[bi, :, iy + P:iy + P + 6, ix + P:ix + P + 6] if iy > TILE_NONE else torch.zeros_like(padded[0, :, :6, :6])
                                     for bi in range(rec.batch) for (iy, ix) in idx])
                for dw, pw_w, pw_b, dst in rec.branches:
                    y = F.conv2d(X, dw.weight.float(), None if dw.bias is None else dw.bias.float(), groups=X.shape[1])
                    if dw.scale is not None:
                        y = y * dw.scale.view(1, -1, 1, 1)
                    if dw.shift is not None:
                        y = y + dw.shift.view(1, -1, 1, 1)
                    y = F.conv2d(y, pw_w.float(), None if pw_b is None else pw_b.float())
                    out = dst.raw
                    H, W = out.shape[2], out.shape[3]
                    for m in range(y.shape[0]):
                        iy, ix = idx[m % n]
                        if iy == TILE_NONE:
                            continue
                        oy, ox = iy + rec.off, ix + rec.off
                        y0, x0, y1, x1 = max(oy, 0), max(ox, 0), min(oy + 4, H), min(ox + 4, W)
                        if y1 > y0 and x1 > x0:
                            out[m // n, :, y0:y1, x0:x1] = y[m, :, y0 - oy:y1 - oy, x0 - ox:x1 - ox].to(out.dtype)

            return run

    return SeparableSim, SimExecutor


def _lower_on_sim(size="mini", net=None):
    """(fused step with the separable launches, fused step as before them, operator-module output) of the sub-mobile generator
    on the descriptor simulator.  The plain SimExecutor has no separable predicate: it lowers the way the step did before."""
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import dilate_mask, downsample_mask
    from sige_b200.fused import FusedStep
    from sige_b200.workloads import gaugan_gc as G

    SeparableSim, Before = _sim_executors()
    net = net if net is not None else G.build_gaugan_gc(size)
    with reference_cpu_runtime():
        _, via_modules = G.run_gaugan_gc(net, downsample_mask, dilate_mask, size=size, fused=lambda n: n.set_fused(False))
        args = (G.gaugan_gc_inputs(size)[1],)
        with torch.no_grad():
            step = FusedStep(net, *args, executor=SeparableSim())
            before = FusedStep(net, *args, executor=Before())
    return step, before, via_modules


def _separable_eager(step):
    """Modules of the separable convs (mlp_gamma / mlp_beta) whose recorded sige.conv calls still run eagerly."""
    from sige_b200.fused import RealStack

    names = {id(m): n for n, m in step.model.named_modules()}
    return [names[id(n.module)] for n in step.tape.nodes if n.name == "sige.conv" and (".mlp_gamma." in names[id(n.module)] or ".mlp_beta." in names[id(n.module)])
            and isinstance(step.low.env.get(id(n.outs[0])), RealStack)]


def _counts(step):
    from collections import Counter

    e = Counter(step.eager_nodes)
    return e["sige.conv"], e["sige.scatter_gather"], e["to_nhwc"], len(step.eager_nodes)


def test_sub_mobile_miniature_lowers_each_spade_layer_to_one_separable_launch():
    """In-tree sub-mobile generator, miniature (ngf 32, config 16_16_16_16_16_16_16_16, 64 x 128, 4 sparse blocks = 12 sparse SPADE
    layers): every SPADE layer's gamma and beta are ONE nbranch = 2 launch, no separable conv is left eager, and the result equals
    the operator modules' to fp32 rounding."""
    step, before, ref = _lower_on_sim("mini")
    assert [len(r.branches) for r in step.low.separable] == [2] * 12
    assert len(before.low.separable) == 0
    assert _separable_eager(step) == [] and len(_separable_eager(before)) == 4 * len(step.low.separable)
    assert _counts(before) == (56, 21, 70, 308)            # today's path (the figures the change started from)
    conv, sg, nhwc, eager = _counts(step)
    assert conv == 56 - 48 and sg == 21 - 16 and nhwc < 70 and eager < 308
    scale = ref.abs().max().item()
    assert (step.output - ref).abs().max().item() <= 2e-5 * scale
    assert (before.output - ref).abs().max().item() <= 2e-5 * scale


def test_sub_mobile_full_size_lowering():
    """Full size (ngf 64, config 32_32_32_48_32_24_24_32, 512 x 1024, 5 sparse blocks): 14 sparse SPADE layers -> 14 separable launches;
    of the 56 recorded sige.conv calls the 12 that remain eager are the 36-channel mlp_shared and the 24/32-channel main convs."""
    step, before, ref = _lower_on_sim("full")
    assert [len(r.branches) for r in step.low.separable] == [2] * 14
    assert _separable_eager(step) == [] and len(_separable_eager(before)) == 4 * len(step.low.separable)
    assert _counts(before) == (56, 27, 78, 320)
    conv, sg, nhwc, eager = _counts(step)
    assert conv == 12 and sg == 27 - 20 and nhwc < 78 and eager < 320
    assert (step.output - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()


# ---------------------------------------------------------------------------------------------------------------- fused step (GPU)
def _golden_or_none():
    path = os.path.join(REPO, "tests", "golden", "gaugan_gc_mini_golden.npz")
    if not os.path.isfile(path):
        return None
    from conftest import golden

    return golden("gaugan_gc_mini_golden.npz")


@pytest.mark.gpu
def test_sub_mobile_miniature_on_gpu_modules_fp32_and_fused_fp16():
    """In-tree sub-mobile generator (no reference needed): the fp32 operator modules and the fused fp16 step with its separable
    launches, against the reference's output (the golden made by running the reference's own file) and each other; graph replay
    is bitwise idempotent."""
    import numpy as np

    from sige.utils import dilate_mask, downsample_mask
    from sige_b200.workloads import gaugan_gc as G

    saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        net = G.build_gaugan_gc("mini").to("cuda:0")
        full0, via_modules = G.run_gaugan_gc(net, downsample_mask, dilate_mask, device="cuda:0", fused=lambda n: n.set_fused(False))
        _, fused = G.run_gaugan_gc(net, downsample_mask, dilate_mask, device="cuda:0", fused=lambda n: n.set_fused(True, dtype=torch.float16))
        step = net.fused_step
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved
    assert step is not None and [len(r.branches) for r in step.low.separable] == [2] * 12
    assert [k for k, _ in step.steps].count("separable") == 12
    ref = via_modules.float().cpu().numpy()
    G_ = _golden_or_none()
    if G_ is not None:
        assert np.abs(full0.cpu().numpy() - G_["full0"]).max() <= 2e-5 * np.abs(G_["full0"]).max()
        assert np.abs(ref - G_["sparse1"]).max() <= 2e-5 * np.abs(G_["sparse1"]).max(), "fp32 operator modules vs the reference"
        ref = G_["sparse1"]
    e = np.abs(fused.float().cpu().numpy() - ref).max() / np.abs(ref).max()
    print("sub-mobile mini: fused fp16 vs %s %.3g" % ("golden" if G_ is not None else "fp32 operator modules", e))
    assert e <= 1e-2
    a = step.replay().clone()
    b = step.replay().clone()
    assert torch.equal(a, b), "graph replay must be idempotent"


def _two_separable_model(cin=64, cout=96):
    """Smallest model whose whole sparse step is separable launches: gamma and beta of a 6x6 Gather of the input, scattered
    through the same tile set (the sub-mobile SPADE's pattern with the input itself as the shared activation)."""
    from sige.nn import Gather, Scatter, SIGEModel
    from sige_b200.workloads.ddpm import init_deterministic
    from sige_b200.workloads.gaugan_gc import SIGESeparableConv2d

    class TwoSeparable(SIGEModel):
        def __init__(self):
            super().__init__()
            self.mlp_gamma = SIGESeparableConv2d(cin, cout, 3, padding=1, support_sparse=True)
            self.mlp_beta = SIGESeparableConv2d(cin, cout, 3, padding=1, support_sparse=True)
            self.gather = Gather(self.mlp_gamma.conv[0], 6)
            self.scatter_gamma = Scatter(self.gather)
            self.scatter_beta = Scatter(self.gather)

        def forward(self, x):
            t = self.gather(x)
            g, b = self.mlp_gamma(t), self.mlp_beta(t)
            return self.scatter_gamma(g) * 0.5 + self.scatter_beta(b)

    return init_deterministic(TwoSeparable(), seed=3).eval()


@pytest.mark.gpu
def test_next_edit_reuses_the_compiled_separable_step():
    """The separable launches read the same fixed-capacity tile lists as the tile convs: a second edit that fits is installed by
    `rebind` and by `set_masks_async` without re-tracing, and equals a fresh compile bitwise."""
    from sige.utils import downsample_mask

    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(1)
    net = _two_separable_model().to(dev).half()
    x0 = torch.randn(1, 64, 32, 48, generator=gen).to(dev).half()
    edit = torch.randn(1, 64, 32, 48, generator=gen).to(dev).half()

    def edited(mask):
        return x0 + edit * mask.to(dev).half()

    mask_a = torch.zeros(32, 48, dtype=torch.bool)
    mask_a[4:14, 6:20] = True
    mask_b = torch.zeros(32, 48, dtype=torch.bool)
    mask_b[18:27, 30:41] = True            # a smaller edit elsewhere: fits the capacity of edit A
    with torch.no_grad():
        net.set_mode("full")
        net(x0)
        net.set_mode("sparse")
        net.set_fused(True, headroom=0.5)
        net.set_masks(downsample_mask(mask_a.to(dev), min_res=(4, 4), dilation=1))
        out_a = net(edited(mask_a))
        step = net.fused_step
        assert [k for k, _ in step.steps].count("separable") == 1 and not any(n.startswith("sige.") for n in step.eager_nodes)
        assert len(step.low.separable[0].branches) == 2
        pyr_b = downsample_mask(mask_b.to(dev), min_res=(4, 4), dilation=1)
        net.set_masks(pyr_b)
        out_b = net(edited(mask_b))
        assert net.fused_step is step, "rebind: the second edit re-uses the compiled step"
        assert net.set_masks_async(downsample_mask(mask_a.to(dev), min_res=(4, 4), dilation=1)) is True
        out_a_async = net(edited(mask_a))
        assert net.fused_step is step and net.masks_async_ok()
        net.set_fused(True, headroom=0.5)               # fresh compiles
        net.set_masks(pyr_b)
        fresh_b = net(edited(mask_b))
        assert net.fused_step is not step
        net.set_masks(downsample_mask(mask_a.to(dev), min_res=(4, 4), dilation=1))
        fresh_a = net(edited(mask_a))
        net.set_fused(False)
        net.set_masks(pyr_b)
        want_b = net(edited(mask_b))
    assert torch.equal(out_b, fresh_b) and torch.equal(out_a_async, fresh_a) and torch.equal(out_a, fresh_a)
    assert float((out_b.float() - want_b.float()).abs().max() / want_b.float().abs().max()) <= 1e-2


# ---------------------------------------------------------------------------------------------------------------- reference file (CPU)
def _consumers():
    import sys

    sys.path.insert(0, os.path.join(REPO, "baseline"))
    import consumers

    return consumers


needs_ref = pytest.mark.skipif(not _consumers().available(), reason="baseline/_ref absent (python baseline/build_ref.py)")


def _reference_generator(size="mini"):
    import importlib

    from sige_b200.workloads import gaugan_gc as G

    c = _consumers()
    c._paths()
    cls = importlib.import_module(c._gaugan_package() + ".sub_mobile_spade_generators.sige_fused_sub_mobile_spade_generator").SIGEFusedSubMobileSPADEGenerator
    return G.build_gaugan_gc(size, cls=cls)


@needs_ref
def test_reference_sub_mobile_file_lowers_to_separable_launches_and_matches_its_golden():
    """The reference's own sub-mobile generator file, unmodified, on this repository's sige: traced and lowered on the simulator,
    every sparse SPADE layer's gamma and beta are one nbranch = 2 launch and the output is the reference's (golden) to 2e-5."""
    import numpy as np

    from conftest import golden

    net = _reference_generator("mini")
    assert type(net).__module__.endswith("sige_fused_sub_mobile_spade_generator")
    step, before, ref = _lower_on_sim("mini", net=net)
    G_ = golden("gaugan_gc_mini_golden.npz")
    assert [len(r.branches) for r in step.low.separable] == [2] * 12
    assert _separable_eager(step) == []
    assert _counts(before)[1] - _counts(step)[1] == 16          # gamma / beta ScatterGathers of the 8 SPADE layers off the shortcut path
    scale = np.abs(G_["sparse1"]).max()
    assert np.abs(ref.numpy() - G_["sparse1"]).max() <= 1e-6 * scale
    assert np.abs(step.output.numpy() - G_["sparse1"]).max() <= 2e-5 * scale


@needs_ref
def test_in_tree_sub_mobile_generator_is_the_reference_file():
    """sige_b200/workloads/gaugan_gc.py restates the reference's file: same state-dict keys, same dense and sparse outputs bit for bit
    on the CPU runtime."""
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import dilate_mask, downsample_mask
    from sige_b200.workloads import gaugan_gc as G

    ref_net, ours = _reference_generator("mini"), G.build_gaugan_gc("mini")
    assert list(ref_net.state_dict()) == list(ours.state_dict())
    with reference_cpu_runtime():
        a = G.run_gaugan_gc(ref_net, downsample_mask, dilate_mask, fused=lambda n: n.set_fused(False))
        b = G.run_gaugan_gc(ours, downsample_mask, dilate_mask, fused=lambda n: n.set_fused(False))
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
