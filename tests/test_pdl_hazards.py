"""Programmatic dependent launch on every compiled program of tests/test_fused_step_contract.py, without a GPU: no launch reads,
before its griddepcontrol.wait, a 128-byte line that a launch still possibly running beside it writes (tests/pdl_hazards.py).
The wgmma / mma.sync choice of each tile conv comes from the host plan, as on the GPU, so the lowering's early marks are the
ones the GPU runs.  Three broken lowerings or models must be rejected by name."""
import os
import re
import sys
import warnings

import pytest
import torch

from conftest import REPO

sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "baseline"))

import fused_step_contract as fsc  # noqa: E402
import pdl_hazards as ph  # noqa: E402
import test_fused_step_contract as TF  # noqa: E402


def _planned(base=None):
    from sim_executor import SimExecutor

    return fsc.recording(ph.planned(base or SimExecutor))


@pytest.fixture(autouse=True)
def _lib(cabi_lib):
    return cabi_lib


@pytest.mark.parametrize("opts", [{}, {"producer_preop": False}, {"fuse_shortcut": False, "sparse_stem": False}, {"tc5": False},
                                  {"fused_attention": False}])
def test_ddpm_small_step_has_no_pdl_hazard(opts):
    model, x1, t = TF._prepared()
    step = TF._step(model, x1, t, executor=_planned()(), **opts)
    st = ph.verify(step, "ddpm_small %s" % opts, model)["main then main"]
    assert st.pdl > 0 and (st.early > 0) == opts.get("tc5", True)


def test_batch_of_three_edits_has_no_pdl_hazard():
    from sige.utils import downsample_mask
    from sige_b200.masks import stack_mask_pyramids
    from sige_b200.workloads.ddpm import DDPMConfig, synthetic_inputs

    model, _, t = TF._prepared()
    edits = []
    for e, (ratio, shift) in enumerate([(0.05, (0, 0)), (0.02, (-14, 9)), (0.09, (11, -13))]):
        x0, x1, mask, _ = synthetic_inputs(DDPMConfig.small(), ratio, seed=0, edit_seed=e)
        edits.append((x0 + torch.roll(x1 - x0, shift, (2, 3)), torch.roll(mask, shift, (0, 1))))
    model.set_masks(stack_mask_pyramids([downsample_mask(m, min_res=8) for _, m in edits]))
    step = TF._step(model, torch.cat([x for x, _ in edits], 0), t, executor=_planned(TF._batched_class())())      # (per-edit lists, as on the GPU)
    assert any(f.spec.tile_img is not None for f in step.fused)
    ph.verify(step, "ddpm_small batch of 3", model)


def test_rebound_step_has_no_pdl_hazard():
    model, x1, t = TF._prepared()
    step = TF._step(model, x1, t, executor=fsc.recording(ph.planned(type(_load_base())))(), headroom=0.6)
    ph.verify(step, "ddpm_small headroom 0.6", model)
    TF._second_edit(model)
    with torch.no_grad():
        assert step.rebind()
    res = ph.verify(step, "ddpm_small after rebind", model)
    assert "loads then main" in res


def test_sparse_update_epilogue_has_no_pdl_hazard():
    model, step = TF._sparse_update_step(_planned(TF._writeback_class()))
    res = ph.verify(step, "ddpm_small with sparse_update", model)
    assert "main then sparse_update" in res
    assert not any(e.pdl for e in ph.entries(step, step.low.epilogue, "sparse_update"))


def test_gaugan_minis_have_no_pdl_hazard():
    step = TF._gaugan_gc_step(_planned(TF._modulated_sim()))
    assert {e.kernel for e in ph.entries(step)} >= {"separable", "mma.sync", "wgmma", "spade", "eager"}
    ph.verify(step, "gaugan_gc mini")
    step = TF._gaugan_spade_step(_planned(TF._strided_sim()))
    ph.verify(step, "gaugan_spade mini")


@pytest.mark.parametrize("which", ["gc", "spade"])
def test_batched_gaugan_step_has_no_pdl_hazard_nor_the_next_batch(which):
    import test_batched_gaugan as TBG
    from oracle.cpu_runtime import reference_cpu_runtime

    net, step, s1s, masks = TF._batched_gaugan(which, _planned(TF._batched_class()))
    ph.verify(step, "gaugan_%s mini batch of %d" % (which, TBG.E), net)
    with reference_cpu_runtime(), torch.no_grad():
        net.set_masks(TBG._batch_masks(masks[[1, 3, 4]]))
        assert step.rebind()
    ph.verify(step, "gaugan_%s mini next batch" % which, net)


def test_sd_decoder_step_has_no_pdl_hazard_before_and_after_a_rebind():
    import test_sd_decoder as TSD

    _, net, step = TF._sd_step(_planned(TSD.TileListSim))
    ph.verify(step, "sd_decoder mini", net)
    TF._sd_rebind(net, step)
    ph.verify(step, "sd_decoder mini after rebind", net)


def test_cache_load_programs_have_no_pdl_hazard():
    import consumers
    import test_spade_generator as TS
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige_b200.workloads import gaugan_spade as GS

    model, x1, t = TF._prepared()
    step = TF._step(model, x1, t, executor=fsc.recording(ph.planned(type(_load_base())))())
    assert [e.kernel for e in ph.load_entries(step)][:1] == ["cache_load"]
    ph.verify(step, "ddpm_small with cache loads", model)
    net = GS.build_gaugan_spade("mini")
    s0, s1, mask = consumers.gaugan_inputs("mini")
    with reference_cpu_runtime(), torch.no_grad():
        net.set_mode("full")
        net(s0)
        net.set_masks(TS._pyramid(mask))
        net.set_mode("sparse")
        step = TF._step(net, s1, executor=fsc.recording(ph.planned(type(_load_base(TF._spade_base()))))())
    ph.verify(step, "gaugan_spade mini with cache loads", net)


def _load_base(base=None):
    import test_cache_refresh as TCR

    return TCR._sim(base)


# ---------------------------------------------------------------------------------------------------------------------
# broken lowerings and a broken model entry: each must be rejected with the launch it breaks
# ---------------------------------------------------------------------------------------------------------------------
def _narrow_ddpm():
    """A DDPM U-Net of base width 32: the block that widens 32 -> 64 channels runs its conv1 (and its shortcut) on the mma.sync
    kernel, which releases its dependents before it waits, and its conv2 on the wgmma kernel."""
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import downsample_mask
    from sige_b200.workloads.ddpm import DDPMConfig, SIGEDDPMUNet, init_deterministic, synthetic_inputs

    cfg = DDPMConfig(image_size=64, ch=32, ch_mult=(1, 2, 2), num_res_blocks=1, attn_resolutions=(16,), sparse_resolution_threshold=32)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model = init_deterministic(SIGEDDPMUNet(cfg), seed=0).eval()
    x0, x1, mask, t = synthetic_inputs(cfg, 0.05, seed=0)
    with torch.no_grad():
        model.set_mode("full")
        model(x0, t)
        model.set_masks(downsample_mask(mask, min_res=8))
        model.set_mode("sparse")

    def build(executor_cls):
        with reference_cpu_runtime():
            return TF._step(model, x1, t, executor=executor_cls())
    return model, build


def test_early_marks_after_an_mma_sync_launch_are_rejected_by_name():
    """Without `Lowering._post`'s correction (an executor that calls every launch a wgmma one), the conv2 after the widening
    block's mma.sync shortcut keeps its early mark on src[0], which conv1, two launches back, may still be writing."""
    Planned = _planned(TF._modulated_sim())

    class NoCorrection(Planned):
        def takes_wgmma(self, fc):
            return True

    model, build = _narrow_ddpm()
    step = build(Planned)
    es = ph.entries(step)
    assert any(es[i - 1].kernel == "mma.sync" and es[i].kernel == "wgmma" for i in range(1, len(es)))
    ph.verify(step, "ddpm ch 32", model)
    step = build(NoCorrection)
    es = ph.entries(step)
    assert any(es[i - 1].kernel == "mma.sync" and es[i].early for i in range(1, len(es)))
    with pytest.raises(AssertionError, match=r"main launch \d+ \(down\.1\.block\.0\.scatter, wgmma\) reads early group 0 src0 before its wait, "
                                             r"which main launch \d+ \(down\.1\.block\.0\.scatter_gather, mma\.sync\) may still be writing"):
        ph.check(es, ph.storage_names(step, model))


def test_a_pre_wait_read_of_the_predecessors_destination_is_rejected_by_name():
    model, x1, t = TF._prepared()
    step = TF._step(model, x1, t, executor=_planned()())
    es = ph.entries(step)
    i = next(i for i in range(1, len(es)) if es[i].pdl and es[i - 1].writes and es[i - 1].kernel != "eager")
    es[i].reads.append(("planted operand", es[i - 1].writes[0][1]))
    with pytest.raises(AssertionError, match="%s reads planted operand before its wait, which %s may still be writing"
                                             % (re.escape(es[i].label), re.escape(es[i - 1].label))):
        ph.check(es, ph.storage_names(step, model))
