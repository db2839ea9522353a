"""A batch of independent label edits through one fused GauGAN step on the GPU.

Kernels: the modulated tile conv (wgmma and mma.sync MOD instantiations), the windowed (strided) tile conv and sige_separable_conv
with per-image tile lists and SIGE_CONV_PER_IMAGE_OPERANDS, f16 and bf16, lists with SIGE_TILE_NONE padding and one edit without
tiles: each within the float64 contract's per-element bound, every element outside the edits' tiles bitwise untouched, and
SIGE_CONV_PADDED (padding CTAs exit at once) bitwise the same result as without it.
Steps: both in-tree generators at mini size, fp16, E = 3 — each edit within the fp16 GauGAN tolerance of its own single-edit step,
graph replay bitwise the eager launch list, the next batch in place through `set_masks` and through `set_masks_async` (no host
synchronisation, bitwise the synchronous install), an overflowing batch flagged on the device and recompiled by `set_masks`."""
import ctypes
import dataclasses
import os
import sys

import numpy as np
import pytest
import torch

from conftest import REPO

sys.path.insert(0, os.path.join(REPO, "tests"))

import kernel_contracts as kc  # noqa: E402
import test_modulated_tile_conv as TM  # noqa: E402
import tile_conv_contract as TC  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
PER = 128          # SIGE_CONV_PER_IMAGE_OPERANDS


def _no_tiles(case, e):
    """Edit `e` of a per-image case loses its tiles: its whole list becomes SIGE_TILE_NONE padding."""
    n = case.spec.N
    case.idx[e * n:(e + 1) * n] = TC.TILE_NONE


def _flag_sets(spec):
    """(kernel, flags without PADDED) per kernel the descriptor can take: the wgmma kernel where its geometry allows, and mma.sync."""
    wgmma = spec.stride == 1 and spec.Cin % 64 == 0 and spec.Cout % 64 == 0 and (spec.k, spec.R) in ((3, 6), (1, 4))
    return ([("wgmma", TC.TC5 | PER)] if wgmma else []) + [("mma.sync", PER)]


def _check_kernels(label, case, expects, launch):
    """Every kernel and split: within the contract, padding-CTA early exit bitwise equal to the full grid, PDL bitwise equal."""
    init = {k: v.clone() for k, v in case.buffers().items()}
    n = 0
    for kernel, flags in _flag_sets(case.spec):
        for ks in TM._ksplits(case.spec):
            outs = []
            for extra in (0, TC.PADDED, TC.PADDED | TC.PDL):
                for name, buf in case.buffers().items():
                    buf.copy_(init[name])
                d = launch(ks, flags | extra)
                plan = TC.plan_of(d)
                assert (plan.path == 1) == (kernel == "wgmma"), (label, kernel)
                torch.cuda.synchronize()
                got = {k: v.clone() for k, v in case.buffers().items()}
                TC.check("%s %s ksplit=%d flags=%d" % (label, kernel, ks, flags | extra), expects, got, init)
                outs.append(got)
                n += 1
            for got in outs[1:]:
                assert all(torch.equal(got[k].view(torch.int16), outs[0][k].view(torch.int16)) for k in got), (label, kernel, ks)
    return n


# ---------------------------------------------------------------------------------------------------------------- modulated
MOD_CASES = [
    # (spec, Mod, edit without tiles): per-image lists of B = 3 edits, N a whole number of CTAs for SIGE_CONV_PADDED
    (TC.Spec("pi_mod64_k3", B=3, H=30, W=38, srcs=((64, 0),), Cout=64, counts=(37, 4, 12), per_image=True, pad_to=40, padded=True,
             preop="per_sample", seed=901), TM.Mod(), 1),
    (TC.Spec("pi_mod128_k3_up", B=3, H=32, W=40, srcs=((128, 1),), Cout=128, counts=(9, 30, 22), per_image=True, pad_to=32, padded=True,
             preop="shared", residual=(8, 8), seed=902), TM.Mod(16, 8, 8, 0), 0),
    (TC.Spec("pi_mod256_k1", B=3, H=28, W=36, k=1, srcs=((256, 0),), Cout=128, counts=(20, 41, 4), per_image=True, pad_to=48, padded=True,
             seed=903), TM.Mod(0, 0, 24, 16, 1.0), 2),
    (TC.Spec("pi_mod40_up", B=3, H=32, W=40, srcs=((40, 1),), Cout=48, counts=(21, 4, 15), per_image=True, pad_to=24, padded=True,
             preop="per_sample", seed=904), TM.Mod(), 1),
    (TC.Spec("pi_mod96_k1", B=3, H=30, W=38, k=1, srcs=((96, 0),), Cout=144, counts=(33, 12, 4), per_image=True, pad_to=40, padded=True,
             preop="shared", aux=((8, 0, False, 0),), seed=905), TM.Mod(96, 96, 0, 0, 1.0), 2),
]


@DTYPES
@pytest.mark.parametrize("spec,mod,empty", MOD_CASES, ids=lambda c: getattr(c, "name", ""))
def test_per_image_modulated_launch_meets_the_float64_contract(spec, mod, empty, dtype):
    mc = TM._mod_case(spec, mod, dtype, DEV)
    _no_tiles(mc.case, empty)
    expects = TM.mod_reference(mc)
    stream = torch.cuda.current_stream().cuda_stream
    from sige_b200 import _cabi

    def launch(ks, flags):
        d = TC.descriptor(mc.case, ksplit=ks, flags=flags)
        d.modulation = ctypes.pointer(TM.modulation(mc))
        _cabi.check(_cabi.lib().sige_tile_conv(ctypes.byref(d), stream), "sige_tile_conv")
        return d

    n = _check_kernels("%s %s" % (spec.name, TC.DTYPE_NAME[dtype]), mc.case, expects, launch)
    print("per-image modulated %s %s: %d launches within the contract" % (spec.name, TC.DTYPE_NAME[dtype], n))


# ---------------------------------------------------------------------------------------------------------------- strided
WIN_CASES = [
    # (spec, (pitch, c0) of the window the source becomes, edit without tiles)
    (TC.Spec("pi_win128_k3", B=3, H=34, W=38, srcs=((128, 0),), Cout=128, counts=(40, 4, 17), per_image=True, pad_to=48, padded=True,
             seed=911), (384, 128), 1),
    (TC.Spec("pi_win64_k1", B=3, H=30, W=34, k=1, srcs=((64, 0),), Cout=64, counts=(30, 12, 4), per_image=True, pad_to=32, padded=True,
             preop="per_sample", act=1, seed=912), (192, 64), 2),
    (TC.Spec("pi_win40", B=3, H=30, W=38, srcs=((40, 0),), Cout=64, counts=(4, 26, 19), per_image=True, pad_to=32, padded=True,
             residual=(0, 0), seed=913), (120, 80), 0),
]


@DTYPES
@pytest.mark.parametrize("spec,win,empty", WIN_CASES, ids=lambda c: getattr(c, "name", ""))
def test_per_image_window_launch_meets_the_float64_contract(spec, win, empty, dtype):
    """The source is channels [c0, c0 + Cin) of a wider buffer of E images, NaN in every other channel."""
    import test_spade_generator as TSG
    from sige_b200 import _cabi

    pitch, c0 = win
    case, wide = TSG._strided_case(spec, pitch, c0, dtype, DEV)
    _no_tiles(case, empty)
    expects = TC.reference(case)
    stream = torch.cuda.current_stream().cuda_stream

    def launch(ks, flags):
        d = TC.descriptor(case, ksplit=ks, flags=flags)
        d.src[0].ptr, d.src_pixel_stride = wide[..., c0:].data_ptr(), pitch
        _cabi.check(_cabi.lib().sige_tile_conv(ctypes.byref(d), stream), "sige_tile_conv")
        return d

    n = _check_kernels("%s %s" % (spec.name, TC.DTYPE_NAME[dtype]), case, expects, launch)
    print("per-image window %s %s: %d launches within the contract" % (spec.name, TC.DTYPE_NAME[dtype], n))


def test_flag_clear_keeps_the_parent_results():
    """Without SIGE_CONV_PER_IMAGE_OPERANDS a modulated or windowed launch of one edit is the launch it always was: setting the flag
    on a per-image list of one image changes no bit (B = 1: the per-image and the shared layout are the same list)."""
    import test_spade_generator as TSG
    from sige_b200 import _cabi

    stream = torch.cuda.current_stream().cuda_stream
    spec = TC.Spec("one_edit", B=1, H=30, W=38, srcs=((128, 0),), Cout=128, counts=(37,), pad_to=40, padded=True, preop="shared", seed=921)
    mc = TM._mod_case(spec, TM.Mod(), torch.float16, DEV)
    case, wide = TSG._strided_case(dataclasses.replace(spec, preop=None), 384, 128, torch.float16, DEV)
    for c, what in ((mc.case, "mod"), (case, "win")):
        init = c.dst.clone()
        outs = []
        for per_image, flags in ((0, TC.TC5 | TC.PADDED), (1, TC.TC5 | TC.PADDED | PER), (0, TC.PADDED), (1, TC.PADDED | PER)):
            c.dst.copy_(init)
            d = TC.descriptor(c, flags=flags)
            d.idx_per_image = per_image
            if what == "mod":
                d.modulation = ctypes.pointer(TM.modulation(mc))
            else:
                d.src[0].ptr, d.src_pixel_stride = wide[..., 128:].data_ptr(), 384
            _cabi.check(_cabi.lib().sige_tile_conv(ctypes.byref(d), stream), "sige_tile_conv")
            torch.cuda.synchronize()
            outs.append(c.dst.clone().view(torch.int16))
        assert torch.equal(outs[0], outs[1]) and torch.equal(outs[2], outs[3]), what
        assert not torch.equal(outs[0], init.view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------- separable
SEP_CASES = [
    # B = 3 edits, N rows per edit (real tiles at the front, SIGE_TILE_NONE behind), one edit without tiles
    (kc.SepSpec("pi_sep48_96", B=3, Cin=48, Cout=96, H=22, W=30, real=20, lead=20, tail=12, pre=96, per_image=True, seed=931), (20, 7, 0)),
    (kc.SepSpec("pi_sep64_256_one_branch", B=3, Cin=64, Cout=256, H=20, W=24, real=14, lead=14, tail=2, post=64,
                dsts=(("buf", 64, 64),), per_image=True, seed=932), (0, 14, 5)),
    (kc.SepSpec("pi_sep16_40", B=3, Cin=16, Cout=40, H=18, W=26, real=15, lead=15, tail=9, per_image=True, seed=933), (15, 0, 9)),
]


def _per_image_sep(spec, counts, dtype):
    """A separable case whose tile list holds one list of N rows per image: image b's first counts[b] tiles of its own draw."""
    case = kc.make_sep(spec, dtype, DEV)
    rows = []
    for b, n in enumerate(counts):
        tiles = [t for t in kc.sep_tile_list(spec, np.random.default_rng(spec.seed + 17 * b)) if t[0] != kc.TILE_NONE]
        rows += tiles[:n] + [(kc.TILE_NONE, kc.TILE_NONE)] * (spec.N - n)
    case.idx = torch.tensor(rows, dtype=torch.int32, device=DEV)
    return case


@DTYPES
@pytest.mark.parametrize("spec,counts", SEP_CASES, ids=lambda c: getattr(c, "name", ""))
def test_per_image_separable_launch_meets_the_float64_contract(spec, counts, dtype):
    from sige_b200 import _cabi

    case = _per_image_sep(spec, counts, dtype)
    expects = kc.sep_reference(case)
    d = kc.sep_descriptor(case)
    lib = _cabi.lib()

    def call(flags):
        d.flags = flags
        return lib.sige_separable_conv(ctypes.byref(d), torch.cuda.current_stream().cuda_stream)

    kc._run_and_check("separable", "%s %s" % (spec.name, TC.DTYPE_NAME[dtype]), case, expects, call, (PER, PER | kc.PDL))


# ---------------------------------------------------------------------------------------------------------------- steps
def _net(which):
    if which == "gc":
        from sige_b200.workloads import gaugan_gc as G

        return G.build_gaugan_gc("mini").to(DEV)
    from sige_b200.workloads import gaugan_spade as GS

    return GS.build_gaugan_spade("mini").to(DEV)


def _pyr(m):
    from sige.utils import dilate_mask, downsample_mask

    return downsample_mask(dilate_mask(m, 1), min_res=(4, 8), dilation=0)


def _batch(masks):
    from sige_b200.masks import stack_mask_pyramids

    return stack_mask_pyramids([_pyr(m) for m in masks])


@pytest.mark.parametrize("which", ["gc", "spade"])
def test_batched_generator_step_and_the_next_batch_in_place(which):
    from sige_b200.workloads import gaugan_gc as G

    saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        net = _net(which)
        s0, s1s, masks = (t.to(DEV) for t in G.gaugan_gc_edits("mini", 5))
        A, B = [0, 1, 2], [1, 3, 4]
        with torch.no_grad():
            net.set_mode("full")
            net(s0)
            net.set_mode("sparse")
            singles = []
            for e in A:
                net.set_fused(True, dtype=torch.float16)
                net.set_masks(_pyr(masks[e]))
                singles.append(net(s1s[e:e + 1]).clone())
            net.set_fused(True, dtype=torch.float16, headroom=0.5)
            net.set_masks(_batch(masks[A]))
            out_a = net(s1s[A]).clone()
            step = net.fused_step
            low = step.low
            assert not any(n.startswith(("sige.", "gather(")) for n in step.eager_nodes), step.eager_nodes
            mods = [f for f in step.fused if f.spec.modulation is not None]
            assert mods and all(f.spec.tile_img is not None and f.desc.flags & PER for f in mods)
            assert all(r.tile_img is not None for r in low.separable) and (len(low.separable) > 0) == (which == "gc")
            assert "batch" in low.sparse_update_reason
            replay = step.replay().clone()
            eager = step.run_eager().clone()
            assert torch.equal(replay, eager), "graph replay == the eager launch list"

            pyr_a, pyr_b, x_b = _batch(masks[A]), _batch(masks[B]), s1s[B]
            net.set_masks(pyr_b)
            out_b = net(s1s[B]).clone()
            assert net.fused_step is step, "batch B fits: installed in place by set_masks"
            net.set_masks(pyr_a)
            assert torch.equal(net(s1s[A]), out_a) and net.fused_step is step
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
            try:
                assert net.set_masks_async(pyr_b) is True
                out_b_async = net(x_b).clone()
            finally:
                torch.cuda.set_sync_debug_mode("default")
            assert net.fused_step is step and net.masks_async_ok()
            assert torch.equal(out_b_async, out_b), "device-installed lists == host-installed lists"

            big = masks[B].clone()
            big[1, :, : big.shape[2] // 2] = True             # half the image: more tiles than the capacity allows
            assert net.set_masks_async(_batch(big)) is True
            assert not net.masks_async_ok()
            net.set_masks(_batch(big))
            out_c = net(s1s[B])
            assert net.fused_step is not step and net.masks_async_ok()
            assert bool(torch.isfinite(out_c).all())
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved
    for i, want in enumerate(singles):
        e = ((out_a[i:i + 1].float() - want.float()).abs().max() / want.float().abs().max()).item()
        print("%s mini, edit %d of a batch of 3 vs its own fp16 step: %.3g of the output scale" % (which, A[i], e))
        assert e <= 1e-2
