"""The Stable Diffusion VAE encoder's fused step on the H100 (sige_b200/workloads/sd_encoder.py; "mini": a 512-channel mid block, so
the D = 512 sparse-attention launch runs, after a stride-2 tile conv and the 3 -> 128 stem on its tiles): fp16 against the golden
the reference's own SIGEEncoder produced, graph replay against stream launches, the next edit — on the bottom and right borders —
installed in place (set_masks, set_masks_async) against a fresh compile, a batch of three edits against their own single-edit steps
and the next batch in place, and the whole-state walk with its poisoned replay on mini f16 / bf16 and on the full encoder.
Kernel: sige_conv_out_nhwc on more channels than one halo fill holds beside the weights (the encoder's 512 -> 8 conv_out), against
the float64 contract."""
import os
import sys

import pytest
import torch

from conftest import REPO, golden

sys.path.insert(0, os.path.join(REPO, "tests"))

import kernel_contracts as kc  # noqa: E402
from tile_conv_contract import DTYPE_NAME  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])


# (spec): halo fills of cc channels, cc the largest multiple of 16 dividing C that fits beside the 8 x 9C weights in 227 KB
WIDE_CONV_OUT = [
    kc.ConvOutSpec("c512_cout8", B=2, H=16, W=40, C=512, Cout=8, seed=1301),                       # the encoder's tail: 4 fills of 128
    kc.ConvOutSpec("c512_swish_shift_only", B=1, H=10, W=20, C=512, Cout=5, pre="shift", seed=1302),
    kc.ConvOutSpec("c384_cout3", B=2, H=11, W=35, C=384, Cout=3, seed=1303),                       # 2 fills of 192, per-element staging
    kc.ConvOutSpec("c1024_cout4_no_preop", B=1, H=9, W=33, C=1024, Cout=4, act=0, pre="none", seed=1304),   # 16 fills of 64
]


@DTYPES
@pytest.mark.parametrize("spec", WIDE_CONV_OUT, ids=lambda s: s.name)
def test_conv_out_wider_than_one_halo_fill_meets_the_float64_contract(spec, dtype):
    from sige_b200 import _cabi

    case = kc.make_conv_out(spec, dtype, DEV)
    expects = kc.conv_out_reference(case)
    kc._run_and_check("conv_out", "%s %s" % (spec.name, DTYPE_NAME[dtype]), case, expects, lambda flags: kc.conv_out_call(case, _cabi.lib()))


def _pyr(mask):
    from sige.utils import downsample_mask

    return downsample_mask(mask, min_res=(4, 4), dilation=0)


def _batch(masks):
    from sige_b200.masks import stack_mask_pyramids

    return stack_mask_pyramids([_pyr(m) for m in masks])


def _setup(size="mini"):
    """(net, x1, x2, pyramids): the encoder after its dense pass on x0; the first edit (x1, mask) and, at mini, the border edit of
    tests/test_sd_encoder.py (x2, mask2)."""
    import test_sd_encoder as TSE
    from sige_b200.workloads import sd_encoder as SE

    net = SE.build_sd_encoder(size).to(DEV)
    x0, x1, mask = SE.sd_encoder_inputs(size)
    x2, mask2 = TSE._border_edit(x0, mask) if size == "mini" else (x1, mask)
    with torch.no_grad():
        net.set_mode("full")
        net(x0.to(DEV))
        net.set_mode("sparse")
    return net, x1.to(DEV), x2.to(DEV), [_pyr(m.to(DEV)) for m in (mask, mask2)]


def test_fused_step_matches_the_reference_golden_and_graph_replay_is_bitwise():
    import test_sd_encoder as TSE
    from sige_b200.fused import FusedStep

    net, x1, _, pyrs = _setup()
    G = golden("sd_encoder_mini_golden.npz")
    with torch.no_grad():
        net.set_masks(pyrs[0])
        net.set_fused(True, dtype=torch.float16)
        out = net(x1).float()
        step = net.fused_step
        stream = FusedStep(net, x1, use_graph=False, dtype=torch.float16).output.clone()
        again = net(x1).clone()
    levels, kinds, strided, stems = TSE._launch_mix(step, net)
    ref = torch.from_numpy(G["sparse1"]).to(DEV)
    err = float((out - ref).abs().max() / ref.abs().max())
    print("sd encoder mini, fused fp16: %.3g of the golden's largest magnitude; %d tile convs (%d stride-2), %s, stem on %d tiles, "
          "eager %s" % (err, len(step.fused), len(strided), dict(kinds), len(stems[0].tiles) if stems else 0, step.eager_nodes))
    assert len(strided) == levels and kinds["conv_in"] == 1 and len(stems) == 1
    assert kinds["sparse_attention"] == 1 and kinds["tail"] == 1 and step.eager_nodes == []
    assert err <= 1e-2
    assert step.graph is not None and torch.equal(again.float(), out) and torch.equal(stream, again)


def test_next_edit_on_the_borders_installs_in_place_like_a_fresh_compile():
    net, x1, x2, pyrs = _setup()
    with torch.no_grad():
        net.set_fused(True, dtype=torch.float16)
        net.set_masks(pyrs[1])
        fresh = net(x2).clone()
        fresh_caps = sorted(sl.cap for sl in net.fused_step.low.slots.values())
        net.set_fused(True, dtype=torch.float16)
        net.set_masks(pyrs[0])
        net(x1)
        step = net.fused_step
        net.set_masks(pyrs[1])
        out_sync = net(x2).clone()
        assert net.fused_step is step, "the border edit fits: installed in place"
        net.set_masks(pyrs[0])
        net(x1)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            assert net.set_masks_async(pyrs[1]) is True
            out_async = net(x2).clone()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert net.fused_step is step and net.masks_async_ok()
        caps = sorted(sl.cap for sl in step.low.slots.values())
        net.set_fused(False)
        eager = net(x2)
    assert torch.equal(out_async, out_sync), "device-installed lists == host-installed lists"
    d = float((out_sync.float() - fresh.float()).abs().max() / fresh.float().abs().max())
    e = float((out_sync.float() - eager).abs().max() / eager.abs().max())
    print("border edit in place vs fresh compile: %.3g, vs the eager fp32 modules: %.3g (tile-list capacities %s, fresh %s)"
          % (d, e, caps, fresh_caps))
    assert e <= 1e-2
    if caps == fresh_caps:          # the same launch plans: the same bits
        assert torch.equal(out_sync, fresh)
    else:                           # other capacities may pick other split-K / cluster plans: fp16 reassociation only
        assert d <= 3e-3


def test_batched_encoder_step_matches_its_singles_and_takes_the_next_batch_in_place():
    from sige_b200.workloads import sd_encoder as SE

    net = SE.build_sd_encoder("mini").to(DEV)
    x0, x1s, masks = (t.to(DEV) for t in SE.sd_encoder_edits("mini", 5))
    A, B = [0, 1, 2], [1, 3, 4]
    with torch.no_grad():
        net.set_mode("full")
        net(x0)
        net.set_mode("sparse")
        singles = []
        for e in A:
            net.set_fused(True, dtype=torch.float16)
            net.set_masks(_pyr(masks[e]))
            singles.append(net(x1s[e:e + 1]).clone())
        net.set_fused(True, dtype=torch.float16, headroom=0.5)
        net.set_masks(_batch(masks[A]))
        out_a = net(x1s[A]).clone()
        step = net.fused_step
        assert step.eager_nodes == [] and all(f.spec.tile_img is not None for f in step.fused)
        replay = step.replay().clone()
        assert torch.equal(replay, step.run_eager()), "graph replay == the eager launch list"

        pyr_a, pyr_b, x_b = _batch(masks[A]), _batch(masks[B]), x1s[B]      # (these synchronise: made before the check below)
        net.set_masks(pyr_b)
        out_b = net(x_b).clone()
        assert net.fused_step is step, "batch B fits: installed in place by set_masks"
        net.set_masks(pyr_a)
        assert torch.equal(net(x1s[A]), out_a) and net.fused_step is step
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            assert net.set_masks_async(pyr_b) is True
            out_b_async = net(x_b).clone()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert net.fused_step is step and net.masks_async_ok()
        net.set_fused(True, dtype=torch.float16, headroom=0.5)
        net.set_masks(pyr_b)
        fresh_b = net(x_b).clone()
    assert torch.equal(out_b_async, out_b), "device-installed lists == host-installed lists"
    db = float((out_b.float() - fresh_b.float()).abs().max() / fresh_b.float().abs().max())
    print("sd encoder mini, batch B in place vs a fresh compile: %.3g" % db)
    assert db <= 3e-3
    for i, want in enumerate(singles):
        e = float((out_a[i:i + 1].float() - want.float()).abs().max() / want.float().abs().max())
        print("sd encoder mini f16, edit %d of a batch of 3 vs its own step: %.3g of the output scale" % (A[i], e))
        assert e <= 1e-2


def _launches(step, res, net):
    import test_sd_encoder as TSE

    levels, _, strided, stems = TSE._launch_mix(step, net)
    assert res["kinds"]["sparse_attention"].launches == 1 and res["kinds"]["conv_in"].launches == 1 and res["poisoned"] > 0
    assert len(strided) == levels and len(stems) == 1


@DTYPES
def test_encoder_step_meets_its_records_with_poisoned_replay_before_and_after_a_rebind(dtype):
    import test_gpu_fused_step_contract as GF

    net, x1, x2, pyrs = _setup()
    with torch.no_grad():
        net.set_masks(pyrs[0])
    step = GF._step(net, x1, step_dtype=dtype)
    _launches(step, GF._walk_and_replay(step, "sd_encoder mini %s" % dtype, model=net), net)
    net.set_masks(pyrs[1])
    with torch.no_grad():
        assert step.rebind()
    step.static_inputs[0].copy_(x2)
    _launches(step, GF._walk_and_replay(step, "sd_encoder mini %s after rebind (border edit)" % dtype, model=net), net)


def test_full_encoder_step_meets_its_records_with_poisoned_replay():
    import test_gpu_fused_step_contract as GF

    net, x1, _, pyrs = _setup("full")
    with torch.no_grad():
        net.set_masks(pyrs[0])
    torch.cuda.reset_peak_memory_stats()
    step = GF._step(net, x1, step_dtype=torch.float16)
    res = GF._walk_and_replay(step, "sd_encoder full fp16", model=net)
    print("[fused step contract] sd_encoder full: %d tile convs, peak %.2f GB" % (len(step.fused), torch.cuda.max_memory_allocated() / 2 ** 30))
    _launches(step, res, net)
    assert sum(1 for f in step.fused if f.spec.stride == 2) == 3
