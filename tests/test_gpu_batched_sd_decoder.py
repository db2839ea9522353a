"""A batch of independent edits of one latent through one fused Stable Diffusion VAE decoder step on the GPU.

Kernels: sige_tile_conv with per-image tile lists and a tile stack on one side (SIGEAttnBlock's q conv writes a stack, proj_out reads
one), on the wgmma and mma.sync kernels, f16 and bf16, lists with SIGE_TILE_NONE padding and one edit without tiles: each within the
float64 contract's per-element bound, every element outside the tiles bitwise untouched, padding stack rows keep their NaN sentinel
bitwise, SIGE_CONV_PADDED bitwise the same as without it.  sige_sparse_attention at D = 512 and B = E, each edit's padded queries.
Step: the mini decoder, E = 3, fp16 and bf16 — edit 0 against the golden, each edit against its own single-edit step, graph replay
bitwise the eager launch list, the whole-state walk with its poisoned replay, the next batch through `set_masks` and through
`set_masks_async` bitwise equal, and an overflowing batch flagged on the device.  The worst error / bound ratios are printed."""
import os
import sys

import pytest
import torch

from conftest import REPO, golden

sys.path.insert(0, os.path.join(REPO, "tests"))

import kernel_contracts as kc  # noqa: E402
import mma_tile_conv_contract as mc  # noqa: E402
import step_kernel_contracts as sk  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
TC5 = 2

# (spec): per-image lists of B = 3 edits, one of them without tiles, N a whole number of CTAs so that SIGE_CONV_PADDED exits early
STACK_CASES = [
    mc.Spec("pis_q_k1_dst_stack", B=3, H=16, W=16, srcs=((512, 0),), Cout=512, counts=(11, 0, 5), R=4, k=(1, 1), dst_stack=True,
            per_image=True, pad_to=16, padded=True, preop="shared", seed=1201),
    mc.Spec("pis_proj_k1_src_stack", B=3, H=16, W=16, srcs=((512, 0),), Cout=512, counts=(6, 14, 0), R=4, k=(1, 1), src_stack=True,
            per_image=True, pad_to=16, padded=True, residual=(0, 0), aux=((0, 0, True, 1),), seed=1202),
    mc.Spec("pis_k3_dst_stack", B=3, H=24, W=20, srcs=((128, 0),), Cout=128, counts=(0, 9, 17), R=6, dst_stack=True, per_image=True,
            pad_to=24, padded=True, preop="per_sample", act=1, seed=1203),
    mc.Spec("pis_k3_src_stack", B=3, H=24, W=20, srcs=((128, 0),), Cout=64, counts=(13, 0, 4), R=6, src_stack=True, per_image=True,
            pad_to=16, padded=True, residual=(0, 0), seed=1204),
]


def _pad_rows(case):
    return (case.idx[:, 0] <= mc.TILE_NONE).to(DEV)


def _launch(d):
    from sige_b200 import ops

    ops.launch_tile_conv(d, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


@DTYPES
@pytest.mark.parametrize("spec", STACK_CASES, ids=lambda s: s.name)
def test_per_image_stack_launch_meets_the_float64_contract(spec, dtype):
    case = mc.make_case(spec, dtype, DEV)
    pad = _pad_rows(case)
    if spec.dst_stack:           # the padding rows of a stack destination are never written: a NaN sentinel must survive bitwise
        case.dst.view[pad] = float("nan")
    expects = mc.reference(case)
    if spec.dst_stack:
        for e in expects:
            n = e.g.view.numel()
            for t in (e.written, e.bound, e.rounding):
                t[e.g.off:e.g.off + n].view(e.g.view.shape)[pad] = 0
            e.want[e.g.off:e.g.off + n].view(e.g.view.shape)[pad] = e.g.view[pad].double()
    else:                        # a stack source's padding rows are read and discarded
        case.srcs[0][pad] = float("nan")
    init = kc.snapshot(case.buffers())
    inputs = case.inputs()
    inputs0 = {k: v.clone() for k, v in inputs.items()}
    worst = []
    for kernel, base in (("wgmma", TC5), ("mma.sync", 0)):
        outs = []
        for flags in (base, base | mc.PADDED, base | mc.PADDED | mc.PDL):
            d = mc.descriptor(case, 0, flags)
            assert mc.plan_of(d).path == (1 if kernel == "wgmma" else 0), (spec.name, kernel)
            kc.restore(case.buffers(), init)
            _launch(d)
            out = kc.snapshot(case.buffers())
            label = "%s %s %s flags %d" % (spec.name, mc.DTYPE_NAME[dtype], kernel, flags)
            worst.append((label, kc.check(label, expects, out, init, inputs, inputs0)))
            if spec.dst_stack:
                got = out["dst"][case.dst.off:case.dst.off + case.dst.view.numel()].view(case.dst.view.shape)
                assert bool(torch.isnan(got[pad]).all()), label
            outs.append(out)
        for out in outs[1:]:
            assert all(torch.equal(kc.bits(out[k]), kc.bits(outs[0][k])) for k in out), "%s %s: SIGE_CONV_PADDED / PDL changed bits" % (spec.name, kernel)
    for label, (r, x) in worst:
        print("[per-image stack tile conv] %-60s worst |err| / bound %.3f, beyond rounding %.3f" % (label, r, x))


# ---------------------------------------------------------------------------------------------------------------- attention
BATCH_ATTENTION = [
    # B = E edits, one head, cap * 16 queries per edit (real tiles then padding rows), every key of the edit's latent
    sk.SAttnSpec("b3_q256_k256", 3, 1, 256, 256, 512, seed=1211),
    sk.SAttnSpec("b3_q384_k4096", 3, 1, 384, 4096, 512, seed=1212),
    sk.SAttnSpec("b4_q128_k4096_bnhd", 4, 1, 128, 4096, 512, layout="bnhd", seed=1213),
]


@DTYPES
@pytest.mark.parametrize("spec", BATCH_ATTENTION, ids=lambda s: s.name)
def test_batched_d512_attention_meets_the_float64_contract(spec, dtype):
    from kernel_contracts import _run_and_check
    from sige_b200 import _cabi

    lib = _cabi.lib()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    case = sk.make_sattn(spec, dtype, DEV)
    expects = sk.wide_sattn_reference(case, sms, chunk=4)
    d = sk.sattn_descriptor(case)
    label = "%s %s" % (spec.name, mc.DTYPE_NAME[dtype])
    _run_and_check("sparse_att_d512", label, case, expects, lambda flags: sk.sattn_call(case, lib, d))


# ---------------------------------------------------------------------------------------------------------------- the step
def _setup():
    from sige_b200.workloads import sd_decoder as SD

    net = SD.build_sd_decoder("mini").to(DEV)
    z0, z1s, masks = (t.to(DEV) for t in SD.sd_decoder_edits("mini", 5))
    with torch.no_grad():
        net.set_mode("full")
        net(z0)
        net.set_mode("sparse")
    return net, z1s, masks


def _pyr(mask):
    from sige.utils import downsample_mask

    return downsample_mask(mask, min_res=(4, 4), dilation=0)


def _batch(masks):
    from sige_b200.masks import stack_mask_pyramids

    return stack_mask_pyramids([_pyr(m) for m in masks])


@DTYPES
def test_batched_decoder_step_and_the_next_batch_in_place(dtype):
    net, z1s, masks = _setup()
    A, B = [0, 1, 2], [1, 3, 4]
    G = golden("sd_decoder_mini_golden.npz")
    with torch.no_grad():
        singles = []
        for e in A:
            net.set_fused(True, dtype=dtype)
            net.set_masks(_pyr(masks[e]))
            singles.append(net(z1s[e:e + 1]).clone())
        net.set_fused(True, dtype=dtype, headroom=0.5)
        net.set_masks(_batch(masks[A]))
        out_a = net(z1s[A]).clone()
        step = net.fused_step
        kinds = [k for k, _ in step.steps]
        assert kinds.count("sparse_attention") == 1 and step.eager_nodes == [], step.eager_nodes
        assert all(f.spec.tile_img is not None and f.desc.idx_per_image == 1 for f in step.fused)
        stacks = [f for f in step.fused if f.desc.src_is_stack or f.desc.dst_is_stack]
        assert len(stacks) == 2 and all(f.desc.B == 3 for f in stacks)
        replay = step.replay().clone()
        eager = step.run_eager().clone()
        assert torch.equal(replay, eager), "graph replay == the eager launch list"

        pyr_a, pyr_b, x_b = _batch(masks[A]), _batch(masks[B]), z1s[B]      # (these synchronise: made before the check below)
        net.set_masks(pyr_b)
        out_b = net(z1s[B]).clone()
        assert net.fused_step is step, "batch B fits: installed in place by set_masks"
        net.set_masks(pyr_a)
        assert torch.equal(net(z1s[A]), out_a) and net.fused_step is step
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
        out_c = net(z1s[B])
        assert net.fused_step is not step and net.masks_async_ok()
        assert bool(torch.isfinite(out_c).all())
    tol = 1e-2 if dtype == torch.float16 else 2e-2          # (bf16's unit roundoff is 8x fp16's)
    ref = torch.from_numpy(G["sparse1"]).to(DEV)
    err0 = float((out_a[0:1].float() - ref).abs().max() / ref.abs().max())
    print("sd decoder mini %s, edit 0 of a batch of 3 vs the golden: %.3g" % (mc.DTYPE_NAME[dtype], err0))
    assert err0 <= tol
    for i, want in enumerate(singles):
        e = float((out_a[i:i + 1].float() - want.float()).abs().max() / want.float().abs().max())
        print("sd decoder mini %s, edit %d of a batch of 3 vs its own step: %.3g of the output scale" % (mc.DTYPE_NAME[dtype], A[i], e))
        assert e <= tol


@DTYPES
def test_batched_decoder_step_meets_its_records_with_poisoned_replay(dtype):
    import test_gpu_fused_step_contract as GF

    net, z1s, masks = _setup()
    with torch.no_grad():
        net.set_masks(_batch(masks[:3]))
    step = GF._step(net, z1s[:3], step_dtype=dtype, headroom=0.5)
    res = GF._walk_and_replay(step, "sd_decoder mini batch of 3 %s" % mc.DTYPE_NAME[dtype], model=net)
    assert res["kinds"]["sparse_attention"].launches == 1
