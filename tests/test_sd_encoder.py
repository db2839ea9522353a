"""The Stable Diffusion VAE encoder (sige_b200/workloads/sd_encoder.py) in miniature, on the CPU: the in-tree restatement and the
reference's own SIGEEncoder file against the golden the reference produced (tests/golden/make_golden_sd_encoder.py), and its fused
step on the descriptor simulator — one stride-2 tile conv per downsample level, the 3 -> 128 stem restricted to the tiles its
readers gather, the mid block's 512-channel attention core as ONE sparse-attention launch and the GroupNorm-fold + conv_out tail,
with no eager node; a second mask on the bottom and right borders installed in place; a batch of three edits against their own
single-edit steps and the next batch installed in place; every launch against its record and no PDL hazard, before and after a
rebind.  The simulators here take the product executor's limits for the tail, whose 512 input channels do not fit in shared memory
as one halo fill."""
import os
import sys
from collections import Counter

import numpy as np
import pytest
import torch

from conftest import REPO, golden

sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "tests", "golden"))

import fused_step_contract as fsc  # noqa: E402
import pdl_hazards as ph  # noqa: E402
from test_batched_sd_decoder import BatchSim  # noqa: E402
from test_sd_decoder import TileListSim  # noqa: E402

from sige_b200.fused import CudaExecutor  # noqa: E402

E = 3
GOLDEN = "sd_encoder_mini_golden.npz"


class ProductTailSim(TileListSim):
    """TileListSim with the product executor's rule for which GroupNorm-fold + conv_out tails one launch takes."""

    tail_supported = CudaExecutor.tail_supported


class ProductTailBatchSim(BatchSim):
    tail_supported = CudaExecutor.tail_supported


def _rel(a, ref):
    return float(np.abs(np.asarray(a, dtype=np.float64) - ref).max() / np.abs(ref).max())


def _pyramid(mask):
    from sige.utils import downsample_mask

    return downsample_mask(mask, min_res=(4, 4), dilation=0)


def _border_edit(x0, mask):
    """A second edit of the mini image on its bottom and right borders, with fewer tiles than the first: (x2, mask2)."""
    mask2 = torch.zeros_like(mask)
    mask2[25:32, 24:32] = True
    rng = np.random.default_rng(11)
    new = torch.from_numpy(rng.uniform(-1.0, 1.0, size=tuple(x0.shape)).astype(np.float32))
    return torch.where(mask2, new, x0), mask2


def _launch_mix(step, net):
    levels = sum(1 for d in net.down if hasattr(d, "downsample"))
    kinds = Counter(k for k, _ in step.steps)
    strided = [f.name for f in step.fused if f.spec.stride == 2]
    stems = [r for r in step.low.conv_ins if r.tiles is not None]
    return levels, kinds, strided, stems


def test_the_product_executor_takes_tails_wider_than_one_halo_fill():
    """sige_conv_out_nhwc fills its halo in chunks of channels when all of them do not fit beside the weights: the encoder's
    512 -> 8 conv_out (and up to 1024 channels) is one tail launch, not an eager GroupNorm, SiLU and conv2d."""
    ex = CudaExecutor.__new__(CudaExecutor)
    assert all(ex.tail_supported(c, cout) for c, cout in ((128, 3), (272, 3), (384, 3), (512, 8), (1024, 8)))
    assert not any(ex.tail_supported(c, cout) for c, cout in ((512, 9), (520, 8), (1040, 8)))


def test_in_tree_encoder_matches_the_reference_golden():
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import downsample_mask
    from sige_b200.workloads import sd_encoder as SE

    net = SE.build_sd_encoder("mini")
    G = golden(GOLDEN)
    with reference_cpu_runtime():
        full0, sparse1 = SE.run_sd_encoder(net, downsample_mask, fused=lambda n: n.set_fused(False))
    assert tuple(sparse1.shape) == (1, SE.OUT_CH, 16, 16)
    assert _rel(full0.numpy(), G["full0"]) <= 1e-6
    assert _rel(sparse1.numpy(), G["sparse1"]) <= 1e-6


def test_reference_encoder_file_matches_the_golden_and_shares_the_state_dict():
    sys.path.insert(0, os.path.join(REPO, "baseline"))
    import consumers

    if not consumers.available():
        pytest.skip("baseline/_ref absent (python baseline/build_ref.py)")
    from make_golden_sd_encoder import build_reference_encoder
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import downsample_mask
    from sige_b200.workloads import sd_encoder as SE

    net = build_reference_encoder("mini")          # the reference's class on this repository's sige.nn
    ours = SE.build_sd_encoder("mini").state_dict()
    theirs = net.state_dict()
    assert list(theirs) == list(ours) and all(torch.equal(theirs[k], ours[k]) for k in ours)
    G = golden(GOLDEN)
    with reference_cpu_runtime():
        full0, sparse1 = SE.run_sd_encoder(net, downsample_mask, fused=lambda n: n.set_fused(False))
    assert _rel(full0.numpy(), G["full0"]) <= 1e-6
    assert _rel(sparse1.numpy(), G["sparse1"]) <= 1e-6


def _steps(executor):
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import downsample_mask
    from sige_b200.fused import FusedStep
    from sige_b200.workloads import sd_encoder as SE

    net = SE.build_sd_encoder("mini")
    with reference_cpu_runtime():
        SE.run_sd_encoder(net, downsample_mask, fused=lambda n: n.set_fused(False))
        x1 = SE.sd_encoder_inputs("mini")[1]
        with torch.no_grad():
            step = FusedStep(net, x1, executor=executor)
    return SE, net, step


def test_fused_step_lowers_every_layer_and_matches_the_golden():
    G = golden(GOLDEN)
    _, net, step = _steps(ProductTailSim())
    levels, kinds, strided, stems = _launch_mix(step, net)
    print("sd encoder mini on the simulator: %d tile convs (%d stride-2), %s, stem on %d tiles of %d x %d, eager %s, %.3g"
          % (len(step.fused), len(strided), dict(kinds), len(stems[0].tiles), stems[0].tile_size, stems[0].tile_size,
             step.eager_nodes, _rel(step.output.numpy(), G["sparse1"])))
    assert levels == 1 and len(strided) == levels and all(n.endswith("downsample.scatter") for n in strided), strided
    assert kinds["conv"] == len(step.fused) and kinds["conv_in"] == 1 and len(stems) == 1 and len(step.low.conv_ins) == 1
    assert kinds["sparse_attention"] == 1 and kinds["tail"] == 1
    assert step.eager_nodes == [] and step.refresh_reason is None
    assert _rel(step.output.numpy(), G["sparse1"]) <= 2e-5


def test_a_second_mask_on_the_borders_rebinds_in_place_like_a_fresh_compile():
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige_b200.fused import FusedStep

    SE, net, step = _steps(ProductTailSim())
    x0, _, mask = SE.sd_encoder_inputs("mini")
    x2, mask2 = _border_edit(x0, mask)
    with reference_cpu_runtime(), torch.no_grad():
        net.set_masks(_pyramid(mask2))
        assert step.rebind(), "the border edit fits the first edit's lists"
        out = step(x2).clone()
        fresh = FusedStep(net, x2, executor=ProductTailSim())
        net.set_fused(False)
        eager = net(x2)
    assert torch.equal(out, fresh.output)
    assert _rel(out.numpy(), eager.numpy()) <= 2e-5
    (stem,) = step.low.conv_ins
    assert stem.tiles is not None and torch.equal(stem.tiles, fresh.low.conv_ins[0].tiles)


def test_batch_of_encoder_edits_runs_as_one_step_and_takes_the_next_batch_in_place():
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige_b200.fused import FusedStep
    from sige_b200.masks import stack_mask_pyramids
    from sige_b200.workloads import sd_encoder as SE

    net = SE.build_sd_encoder("mini")
    x0, x1s, masks = SE.sd_encoder_edits("mini", E + 2)
    assert any(bool(m[:, -1].any()) for m in masks[E:])                    # the next batch holds the bottom-right corner edit
    with reference_cpu_runtime(), torch.no_grad():
        net.set_mode("full")
        net(x0)
        net.set_mode("sparse")
        singles = []
        for e in range(E):
            net.set_masks(_pyramid(masks[e]))
            singles.append(FusedStep(net, x1s[e:e + 1], executor=ProductTailSim()))
        net.set_masks(stack_mask_pyramids([_pyramid(m) for m in masks[:E]]))
        step = FusedStep(net, x1s[:E], executor=ProductTailBatchSim(), headroom=0.5)
    levels, kinds, strided, _ = _launch_mix(step, net)
    assert kinds == Counter(k for k, _ in singles[0].steps) and len(strided) == levels and step.eager_nodes == []
    assert all(f.spec.tile_img is not None and f.spec.slot.E == E for f in step.fused)
    out = step.output.clone()
    for e, one in enumerate(singles):
        assert _rel(out[e:e + 1].numpy(), one.output.numpy()) <= 2e-5, e
    assert _rel(out[0:1].numpy(), golden(GOLDEN)["sparse1"]) <= 2e-5

    order = [1, 3, 4]
    with reference_cpu_runtime(), torch.no_grad():
        net.set_masks(stack_mask_pyramids([_pyramid(masks[e]) for e in order]))
        assert step.rebind(), "a batch that fits is installed in place"
        out_b = step(x1s[order]).clone()
        fresh_b = FusedStep(net, x1s[order], executor=ProductTailBatchSim(), headroom=0.5).output
    assert torch.equal(out_b, fresh_b)


def test_encoder_program_meets_its_records_and_has_no_pdl_hazard_before_and_after_a_rebind(cabi_lib):
    from oracle.cpu_runtime import reference_cpu_runtime

    SE, net, step = _steps(fsc.recording(ph.planned(ProductTailSim))())
    res = fsc.walk(step, model=net)
    print(fsc.summary("sd_encoder mini", res))
    fsc.checked_all(step, res)
    assert res["kinds"]["sparse_attention"].launches == 1 and res["kinds"]["conv_in"].launches == 1
    ph.verify(step, "sd_encoder mini", net)
    x0, _, mask = SE.sd_encoder_inputs("mini")
    x2, mask2 = _border_edit(x0, mask)
    with reference_cpu_runtime(), torch.no_grad():
        net.set_masks(_pyramid(mask2))
        assert step.rebind()
    step.static_inputs[0].copy_(x2)
    fsc.checked_all(step, fsc.walk(step, model=net))
    ph.verify(step, "sd_encoder mini after rebind", net)
