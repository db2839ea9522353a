"""A compiled DDPM step on the descriptor simulator, walked launch by launch against float64 restatements of its records
(tests/fused_step_contract.py), and mutants of the simulator that each break one launch, which the walk must name."""
import copy
import os
import re
import sys
import types
import warnings

import pytest
import torch

from conftest import REPO

sys.path.insert(0, os.path.join(REPO, "tests"))

import fused_step_contract as fsc  # noqa: E402


def _model():
    from sige_b200.workloads.ddpm import DDPMConfig, SIGEDDPMUNet, init_deterministic

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return init_deterministic(SIGEDDPMUNet(DDPMConfig.small()), seed=0).eval()


def _prepared(ratio=0.05):
    from sige.utils import downsample_mask
    from sige_b200.workloads.ddpm import DDPMConfig, synthetic_inputs

    model = _model()
    x0, x1, mask, t = synthetic_inputs(DDPMConfig.small(), ratio, seed=0)
    with torch.no_grad():
        model.set_mode("full")
        model(x0, t)
        model.set_masks(downsample_mask(mask, min_res=8))
        model.set_mode("sparse")
    return model, x1, t


def _sim(base=None):
    from sim_executor import SimExecutor

    return fsc.recording(base or SimExecutor)


def _step(model, *args, executor=None, **opts):
    from sige_b200.fused import FusedStep

    with torch.no_grad():
        return FusedStep(model, *args, executor=executor or _sim()(), **opts)


def _walk(step, tag, program=None, model=None):
    res = fsc.walk(step, program, model=model)
    print(fsc.summary(tag, res))
    fsc.checked_all(step, res, program)
    return res


@pytest.mark.parametrize("opts", [{}, {"producer_preop": False}, {"fuse_shortcut": False, "sparse_stem": False}, {"tc5": False},
                                  {"fused_attention": False}])
def test_every_launch_of_a_ddpm_step_meets_its_record(opts):
    model, x1, t = _prepared()
    step = _step(model, x1, t, **opts)
    res = _walk(step, "ddpm_small %s" % opts)
    assert res["kinds"]["conv"].launches == len(step.fused) >= 34
    if not opts.get("fused_attention", True):
        assert res["eager"] > 0 and "attention" not in res["kinds"]
    else:
        assert res["eager"] == 0 and res["kinds"]["attention"].launches == 4


def test_sparse_attention_inside_the_step_meets_its_record():
    class NoClusterAttention(_sim()):
        def attention_supported(self, n_tokens, channels):
            return False

    model, x1, t = _prepared()
    step = _step(model, x1, t, executor=NoClusterAttention())
    res = _walk(step, "ddpm_small sparse attention")
    assert res["kinds"]["sparse_attention"].launches == 4


def test_batch_of_three_edits_meets_its_records():
    from sige.utils import downsample_mask
    from sige_b200.masks import stack_mask_pyramids
    from sige_b200.workloads.ddpm import DDPMConfig, synthetic_inputs

    cfg = DDPMConfig.small()
    model, _, t = _prepared()
    edits = []
    for e, (ratio, shift) in enumerate([(0.05, (0, 0)), (0.02, (-14, 9)), (0.09, (11, -13))]):
        x0, x1, mask, _ = synthetic_inputs(cfg, ratio, seed=0, edit_seed=e)
        edits.append((x0 + torch.roll(x1 - x0, shift, (2, 3)), torch.roll(mask, shift, (0, 1))))
    model.set_masks(stack_mask_pyramids([downsample_mask(m, min_res=8) for _, m in edits]))
    step = _step(model, torch.cat([x for x, _ in edits], 0), t)
    assert any(f.spec.tile_img is not None for f in step.fused)
    _walk(step, "ddpm_small batch of 3")


def _second_edit(model):
    from sige.utils import downsample_mask
    from sige_b200.workloads.ddpm import DDPMConfig, synthetic_inputs

    cfg = DDPMConfig.small()
    x0, _, _, _ = synthetic_inputs(cfg, 0.05, seed=0)
    _, x_b, mask_b, _ = synthetic_inputs(cfg, 0.03, seed=0, edit_seed=5)
    mask_b = torch.roll(mask_b, (9, -11), (0, 1))
    x_b = x0 + torch.roll(x_b - x0, (9, -11), (2, 3))
    model.set_masks(downsample_mask(mask_b, min_res=8))
    return x_b


def test_rebind_restores_the_cached_state_and_its_launches_meet_their_records():
    model, x1, t = _prepared()
    step = _step(model, x1, t, headroom=0.6)
    _walk(step, "ddpm_small headroom 0.6")
    x_b = _second_edit(model)
    with torch.no_grad():
        assert step.rebind()
    assert any(sl.cap - sl.n >= 8 for sl in step.low.slots.values()), "the padded lists must hold whole blocks of SIGE_TILE_NONE"
    r = fsc.cached_state_after_rebind(step)
    print("[fused step contract] cached views after rebind: worst error / bound %.3f" % r)
    step.static_inputs[0].copy_(x_b)
    _walk(step, "ddpm_small after rebind")


def _writeback_class():
    import test_sparse_update_fused as TSU

    return type(TSU._writeback_sim())


def _sparse_update_step(executor_cls):
    import test_sparse_update_fused as TSU
    from sige.utils import downsample_mask
    from sige_b200.workloads.ddpm import DDPMConfig

    cfg = DDPMConfig.small()
    x0, t, edits = TSU._edits(cfg)
    model = TSU._model("intree", cfg)
    with torch.no_grad():
        TSU._dense(model, x0, t)
        model.set_cache_id(1)
        model.set_masks(downsample_mask(edits[0][1], min_res=8))
    step = _step(model, edits[0][0] * 1.1, t + 10, executor=executor_cls())
    assert step.sparse_update_supported, step.sparse_update_reason
    return model, step


def test_sparse_update_epilogue_meets_its_records():
    model, step = _sparse_update_step(_sim(_writeback_class()))
    _walk(step, "ddpm_small main", model=model)
    kinds = [k for k, _ in step.low.epilogue]
    assert kinds.count("writeback") == 1 and kinds.count("conv") > 0
    _walk(step, "ddpm_small sparse_update epilogue", step.low.epilogue, model=model)


# ---------------------------------------------------------------------------------------------------------------------
# mutants: one launch of a chosen kind breaks its record; the walk must fail and name that launch
# ---------------------------------------------------------------------------------------------------------------------
def _first_real(s):
    for r, (iy, ix) in enumerate(s.idx.tolist()):
        if iy > fsc.NONE_BELOW:
            return r, iy, ix
    raise AssertionError(s.name)


def _out_origin(s, iy, ix):
    return (s.off + iy) // s.stride, (s.off + ix) // s.stride


def _mutant_off_by_one(s, run):
    src, up = s.srcs[0]
    shifted = torch.empty_like(src)
    m = types.SimpleNamespace(**vars(s))
    m.srcs = [(shifted, up)] + list(s.srcs[1:])

    def go(stream):
        shifted.copy_(torch.roll(src, 1, dims=3))
        run(m, stream)
    return go


def _mutant_skip_residual(s, run):
    def go(stream):
        res = s.residual.clone()
        run(s, stream)
        _, iy, ix = _first_real(s)
        oy, ox = _out_origin(s, iy, ix)
        ro = (s.block - s.k) // s.stride + 1
        s.dst.raw[0, :, oy:oy + ro, ox:ox + ro] -= res[0, :, oy:oy + ro, ox:ox + ro]
    return go


def _mutant_write_past(s, run):
    """One pixel past the bottom edge of a real tile, (oy + ro, ox), where that pixel belongs to no tile of the list."""
    def go(stream):
        run(s, stream)
        ro = (s.block - s.k) // s.stride + 1
        dst = s.dst.raw
        Hd, Wd = dst.shape[2], dst.shape[3]
        covered = torch.zeros((Hd, Wd), dtype=torch.bool)
        origins = [_out_origin(s, iy, ix) for iy, ix in s.idx.tolist() if iy > fsc.NONE_BELOW]
        for oy, ox in origins:
            covered[max(oy, 0):max(oy + ro, 0), max(ox, 0):max(ox + ro, 0)] = True
        oy, ox = next((oy, ox) for oy, ox in origins if 0 <= oy + ro < Hd and 0 <= ox < Wd and not covered[oy + ro, ox])
        dst[0, 0, oy + ro, ox] += 1.0
    return go


def _mutant_none_as_origin(s, run):
    real = {tuple(r) for r in s.idx.tolist() if r[0] > fsc.NONE_BELOW}
    H, W = s.H, s.W
    spare = next((iy, ix) for iy in range(-s.off, H, 4) for ix in range(-s.off, W, 4) if (iy, ix) not in real)
    idx = s.idx.clone()
    idx[idx[:, 0] <= fsc.NONE_BELOW] = torch.tensor(spare, dtype=idx.dtype)
    m = types.SimpleNamespace(**vars(s))
    m.idx = idx
    return lambda stream: run(m, stream)


def _mutant_shortcut_everywhere(s, run):
    srcs, w, b, flags = s.shortcut
    m = types.SimpleNamespace(**vars(s))
    m.shortcut = (srcs, w, b, torch.ones_like(flags))
    return lambda stream: run(m, stream)


def _mutant_no_row_scale(s, run):
    m = types.SimpleNamespace(**vars(s))
    m.out_row_scale = None
    return lambda stream: run(m, stream)


def _offset(t):
    t.add_(0.5)


MUTANTS = {
    # name: (which conv launch, how it breaks, what to move off its cached value first so that the break shows).  Recomputing an
    # unchanged tile reproduces the cache, and the fresh shortcut of an unchanged tile equals its cached residual: the walk's
    # expectations follow the live buffers, so offsetting one makes the two differ.
    "reads_one_pixel_off": (lambda s: not s.src_is_stack and s.idx is not None, _mutant_off_by_one, None),
    "skips_the_residual_on_a_tile": (lambda s: s.residual is not None and s.dst is not None and s.dst.has_raw and s.shortcut is None,
                                     _mutant_skip_residual, None),
    "writes_one_pixel_past_its_tile": (lambda s: s.dst is not None and s.dst.has_raw and s.slot is not None and s.tile_img is None,
                                       _mutant_write_past, None),
    "takes_a_padding_row_as_an_origin": (lambda s: s.slot is not None and s.slot.cap - s.slot.n >= 1 and s.dst is not None and s.dst.has_raw
                                         and s.tile_img is None, _mutant_none_as_origin, lambda s: _offset(s.dst.raw)),
    "applies_the_shortcut_on_an_unflagged_tile": (lambda s: s.shortcut is not None and s.shortcut[3] is not None and bool((s.shortcut[3] == 0).any())
                                                  and s.residual is not None, _mutant_shortcut_everywhere, lambda s: _offset(s.residual)),
    "ignores_out_row_scale": (lambda s: s.out_row_scale is not None, _mutant_no_row_scale, None),
}


def _mutant_sim(which):
    from sim_executor import SimExecutor

    pick, breaks, _ = MUTANTS[which]

    class Mutant(fsc.recording(SimExecutor)):
        armed = False
        victim = None

        def prepare_conv(self, fc):
            super().prepare_conv(fc)
            if not self.armed or self.victim is not None or not pick(fc.spec):
                return
            self.victim, self.victim_spec = fc.name, fc.spec

            def run(spec, stream):
                shim = types.SimpleNamespace(spec=spec, launch_fn=None)
                SimExecutor.prepare_conv(self, shim)
                shim.launch_fn(stream)

            fc.launch_fn = breaks(fc.spec, run)

    return Mutant


@pytest.mark.parametrize("which", sorted(MUTANTS))
def test_a_broken_conv_launch_is_rejected_by_name(which):
    model, x1, t = _prepared()
    Mutant = _mutant_sim(which)
    ex = Mutant()
    ex.armed = True
    step = _step(model, x1, t, executor=ex, headroom=0.6)
    assert ex.victim is not None, "no launch of this step has what the mutant breaks"
    offset = MUTANTS[which][2]
    if offset is not None:
        with torch.no_grad():
            offset(ex.victim_spec)
    with pytest.raises(AssertionError, match=r"conv launch \d+ \(%s\)" % ex.victim.replace(".", r"\.")):
        fsc.walk(step)


# ---------------------------------------------------------------------------------------------------------------------
# the GauGAN miniatures: separable, narrow, ReLU-epilogue, modulated and channel-window launches, SPADE modulation launches
# ---------------------------------------------------------------------------------------------------------------------
def _gaugan_gc_step(executor_cls):
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import dilate_mask, downsample_mask
    from sige_b200.workloads import gaugan_gc as G

    net = G.build_gaugan_gc("mini")
    with reference_cpu_runtime():
        G.run_gaugan_gc(net, downsample_mask, dilate_mask, size="mini", fused=lambda n: n.set_fused(False))
    return _step(net, G.gaugan_gc_inputs("mini")[1], executor=executor_cls())


def _gaugan_spade_step(executor_cls):
    import consumers
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import dilate_mask, downsample_mask
    from sige_b200.workloads import gaugan_spade as GS

    net = GS.build_gaugan_spade("mini")
    with reference_cpu_runtime():
        consumers.run_gaugan(net, downsample_mask, dilate_mask, size="mini", fused=lambda n: n.set_fused(False))
    return _step(net, consumers.gaugan_inputs("mini")[1], executor=executor_cls())


def _modulated_sim():
    import test_modulated_tile_conv as TM

    return TM._mod_sim()[0]


def _strided_sim():
    import test_spade_generator as TSG

    return TSG._sims()[0]


def test_sub_mobile_gaugan_step_meets_its_records():
    step = _gaugan_gc_step(_sim(_modulated_sim()))
    res = _walk(step, "gaugan_gc mini")
    specs = [f.spec for f in step.fused]
    assert res["kinds"]["separable"].launches > 0 and res["kinds"]["spade"].launches == 6
    assert any(s.modulation is not None for s in specs) and any(s.epilogue_act == "relu" for s in specs)
    assert any(s.Cin % 64 for s in specs) and res["eager"] > 0


def test_spade_generator_step_meets_its_records():
    import test_spade_generator as TSG

    step = _gaugan_spade_step(_sim(_strided_sim()))
    res = _walk(step, "gaugan_spade mini")
    assert sum(1 for f in step.fused if f.spec.modulation is not None) == 12 and len(TSG._windowed(step)) == 12
    assert res["kinds"]["conv"].launches == len(step.fused)


def test_a_broken_modulated_launch_is_rejected_by_name():
    """The modulated launch is handed gamma and beta the wrong way round."""
    class Swapped(_sim(_modulated_sim())):
        victim = None

        def prepare_conv(self, fc):
            s = fc.spec
            if self.victim is not None or s.modulation is None:
                return super().prepare_conv(fc)
            self.victim = fc.name
            m = copy.copy(s)
            m.modulation = (s.modulation[1], s.modulation[0], s.modulation[2])
            fc.spec = m
            try:
                super().prepare_conv(fc)
            finally:
                fc.spec = s

    step = _gaugan_gc_step(Swapped)
    assert step.ex.victim is not None
    with pytest.raises(AssertionError, match=r"conv launch \d+ \(%s\)" % step.ex.victim.replace(".", r"\.")):
        fsc.walk(step)


def test_a_writeback_into_the_wrong_cache_is_rejected_by_name():
    import test_sparse_update_fused as TSU

    class WrongCache(_sim(_writeback_class())):
        def prepare_writeback(self, entries):
            entries = list(entries)
            same = next((i, j) for i in range(len(entries)) for j in range(i + 1, len(entries))
                        if entries[i][1].shape == entries[j][1].shape and entries[i][1].dtype == entries[j][1].dtype)
            i, j = same
            swapped = list(entries)
            swapped[i] = (entries[i][0], entries[j][1]) + tuple(entries[i][2:])
            fn = super().prepare_writeback(entries)
            self.records[id(fn)] = ("writeback", entries, fn)

            def run(_stream, fn=fn):
                self.launches += 1
                TSU.torch_writeback(swapped)
            self.records[id(run)] = ("writeback", entries, run)
            return run

    model, step = _sparse_update_step(WrongCache)
    fsc.walk(step, model=model)
    with pytest.raises(AssertionError, match=r"writeback launch \d+ \(writeback\)"):
        fsc.walk(step, step.low.epilogue, model=model)


# ---------------------------------------------------------------------------------------------------------------------
# the Stable Diffusion decoder (a q stack of fixed capacity, the D = 512 sparse attention), batches of label edits (per-image
# separable and modulated launches) and the cache load of a new edit
# ---------------------------------------------------------------------------------------------------------------------
def _sd_step(executor_cls):
    import test_sd_decoder as TSD

    return TSD._steps(executor_cls())


def _sd_rebind(net, step):
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import downsample_mask
    from sige_b200.workloads import sd_decoder as SD

    _, z1, mask = SD.sd_decoder_inputs("mini")
    mask2 = torch.zeros_like(mask)
    mask2[12:20, 6:15] = True                    # the second mask of test_sd_decoder.py: fewer tiles than the first
    with reference_cpu_runtime(), torch.no_grad():
        net.set_masks(downsample_mask(mask2, min_res=(4, 4), dilation=0))
        assert step.rebind()
    step.static_inputs[0].copy_(z1)


def _sd_checks(step, res):
    assert res["kinds"]["sparse_attention"].launches == 1 and res["poisoned"] > 0
    stems = [r for r in step.low.conv_ins if int(r.weight.shape[0]) == 512]
    assert len(stems) == 1 and res["kinds"]["conv_in"].launches >= 1


def test_sd_decoder_step_meets_its_records_before_and_after_a_rebind():
    import test_sd_decoder as TSD

    _, net, step = _sd_step(fsc.recording(TSD.TileListSim))
    _sd_checks(step, _walk(step, "sd_decoder mini"))
    live = {sl.n for sl in step.low.slots.values()}
    _sd_rebind(net, step)
    assert {sl.n for sl in step.low.slots.values()} != live
    _sd_checks(step, _walk(step, "sd_decoder mini after rebind"))


def _no_tiles_batch(pyramid_of, masks):
    """The set_masks argument of a batch whose last edit has no tiles: its pyramid all False.  (A mask without a set pixel is
    not that: downsample_mask thresholds at min(0.3, max - eps), so an all-zero mask selects the whole image, as in the
    reference.)"""
    from sige_b200.masks import stack_mask_pyramids

    pyrs = [pyramid_of(m) for m in masks]
    pyrs[-1] = {k: torch.zeros_like(v) for k, v in pyrs[-1].items()}
    return stack_mask_pyramids(pyrs)


def _batched_gaugan(which, executor_cls):
    import test_batched_gaugan as TBG
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige_b200.workloads import gaugan_gc as G

    net = TBG._generator(which)
    s0, s1s, masks = G.gaugan_gc_edits("mini", TBG.E + 2)
    with reference_cpu_runtime(), torch.no_grad():
        net.set_mode("full")
        net(s0)
        net.set_mode("sparse")
        net.set_masks(_no_tiles_batch(TBG._pyramid, masks[:TBG.E]))       # the third edit has no tiles
        step = _step(net, s1s[:TBG.E], executor=executor_cls(), headroom=0.5)
    return net, step, s1s, masks


def _batched_class():
    import test_batched_gaugan as TBG

    return TBG._sims()[0]


@pytest.mark.parametrize("which", ["gc", "spade"])
def test_batched_gaugan_step_meets_its_records_and_the_next_batch_too(which):
    import test_batched_gaugan as TBG
    from oracle.cpu_runtime import reference_cpu_runtime

    net, step, s1s, masks = _batched_gaugan(which, fsc.recording(_batched_class()))
    res = _walk(step, "gaugan_%s mini batch of %d, the third edit without tiles" % (which, TBG.E))
    assert any(f.spec.tile_img is not None for f in step.fused)
    assert all(bool((sl.buf.view(TBG.E, sl.cap, 2)[2, :, 0] <= fsc.NONE_BELOW).all()) for sl in step.low.slots.values())
    if which == "gc":
        assert res["kinds"]["separable"].launches > 0 and all(r.tile_img is not None for r in step.low.separable)
    order = [1, 3, 4]
    with reference_cpu_runtime(), torch.no_grad():
        net.set_masks(TBG._batch_masks(masks[order]))
        assert step.rebind()
    step.static_inputs[0].copy_(s1s[order])
    _walk(step, "gaugan_%s mini next batch" % which)


def _load_sim(base=None):
    import test_cache_refresh as TCR

    return fsc.recording(type(TCR._sim(base)))


def _spade_base():
    import test_spade_generator as TSG

    return TSG._sims()[0]


def _walk_loads(step, tag, model):
    res = fsc.walk_loads(step, model=model)
    print(fsc.summary(tag, res) + "; %d entries" % res["entries"])
    assert res["kinds"]["cache_load"].launches == 1 and res["entries"] > 0
    return res


def test_cache_loads_meet_their_records_at_build_after_a_rebind_and_after_a_refresh():
    from sige.utils import downsample_mask
    from sige_b200.workloads.ddpm import DDPMConfig, synthetic_inputs

    model, x1, t = _prepared()
    step = _step(model, x1, t, executor=_load_sim()(), headroom=0.6)
    _walk_loads(step, "ddpm_small loads at build", model)
    _second_edit(model)
    with torch.no_grad():
        assert step.rebind()
    _walk_loads(step, "ddpm_small loads after rebind", model)
    x0, _, _, _ = synthetic_inputs(DDPMConfig.small(), 0.05, seed=0)
    with torch.no_grad():
        model.set_mode("full")
        model(x0 * 0.7, t)
        model.set_mode("sparse")
        assert step.refresh()
    _walk_loads(step, "ddpm_small loads after refresh", model)
    assert fsc.cached_state_after_rebind(step) <= 1.0


def test_spade_generator_cache_loads_meet_their_records():
    import consumers
    import test_spade_generator as TS
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige_b200.workloads import gaugan_spade as GS

    net = GS.build_gaugan_spade("mini")
    s0, s1, mask = consumers.gaugan_inputs("mini")
    with reference_cpu_runtime(), torch.no_grad():
        net.set_mode("full")
        net(s0)
        net.set_masks(TS._pyramid(mask))
        net.set_mode("sparse")
        step = _step(net, s1, executor=_load_sim(_spade_base())())
    _walk_loads(step, "gaugan_spade mini loads at build", net)
    with reference_cpu_runtime(), torch.no_grad():
        net.set_mode("full")
        net(s1)
        net.set_mode("sparse")
        assert step.refresh()
    _walk_loads(step, "gaugan_spade mini loads after refresh", net)
    with reference_cpu_runtime(), torch.no_grad():
        assert step.rebind()
    _walk_loads(step, "gaugan_spade mini loads after rebind", net)


# mutants of the new launch kinds: each must be rejected with the kind and the position of its launch
def test_a_separable_launch_that_reads_image_0s_list_for_every_image_is_rejected_by_name():
    import test_batched_gaugan as TBG

    class OneList(fsc.recording(_batched_class())):
        victim = None

        def prepare_separable(self, rec):
            if self.victim is not None or rec.tile_img is None:
                return super().prepare_separable(rec)
            self.victim = rec.name
            n = rec.idx.shape[0] // rec.batch
            m = copy.copy(rec)
            m.idx = rec.idx.clone()
            fn = super().prepare_separable(rec)
            inner = _batched_class().prepare_separable(self, m)

            def run(stream):
                m.idx.copy_(rec.idx[:n].repeat(rec.batch, 1))       # image 0's list, read at launch time
                inner(stream)
            self.records[id(run)] = ("separable", rec, run)
            del self.records[id(fn)]
            return run

    _, step, _, _ = _batched_gaugan("gc", OneList)
    assert step.ex.victim is not None and TBG.E > 1
    with pytest.raises(AssertionError, match=r"separable launch \d+ \(%s\)" % re.escape(step.ex.victim)):
        fsc.walk(step)


def test_a_sparse_attention_with_a_wrong_scale_is_rejected_by_name():
    import test_sd_decoder as TSD

    class WrongScale(fsc.recording(TSD.TileListSim)):
        def prepare_sparse_attention(self, q, k, v, scale, out):
            fn = TSD.TileListSim.prepare_sparse_attention(self, q, k, v, scale * 1.01, out)
            return self._keep("sparse_attention", fn, dict(q=q, k=k, v=v, scale=scale, out=out))

    _, _, step = _sd_step(WrongScale)
    with pytest.raises(AssertionError, match=r"sparse_attention launch \d+ \(sparse_attention\)"):
        fsc.walk(step)


def test_a_q_stack_conv_that_writes_its_padding_rows_is_rejected_by_name():
    import test_sd_decoder as TSD

    class WritesPadding(fsc.recording(TSD.TileListSim)):
        victim = None

        def prepare_conv(self, fc):
            s = fc.spec
            if s.dst_stack is None or s.src_is_stack:
                return super().prepare_conv(fc)
            self.victim = fc.name
            SimExecutor = TSD.SimExecutor
            SimExecutor.prepare_conv(self, fc)                        # the plain simulator writes every row of its stack
            self._records()[id(fc)] = ("conv", False, fc)

    _, _, step = _sd_step(WritesPadding)
    assert step.ex.victim is not None and any(sl.cap > sl.n for sl in step.low.slots.values())
    with pytest.raises(AssertionError, match=r"conv launch \d+ \(%s\): wrote outside its record" % re.escape(step.ex.victim)):
        fsc.walk(step)


def _load_mutant(change):
    Base = _load_sim()

    class Mutant(Base):
        def prepare_cache_load(self, entries):
            entries = [(src, raw, list(views)) for (src, raw, views) in entries]
            fn = super(fsc.RecordingMixin, self).prepare_cache_load(change(entries))
            return self._keep("cache_load", fn, entries)

    return Mutant


def _drop_a_shift(entries):
    out = [(src, raw, list(views)) for (src, raw, views) in entries]
    i, j = next((i, j) for i, (_, _, vs) in enumerate(out) for j, v in enumerate(vs) if v[2] is not None and float(v[2].abs().max()) > 0)
    v, sc, _, act = out[i][2][j]
    out[i][2][j] = (v, sc, None, act)
    return out


def _also_writes_its_source(entries):
    src = entries[0][0]
    return entries + [(src, None, [(src, None, torch.ones(src.shape[1]), "identity")])]      # cache + 1 into the cache itself


@pytest.mark.parametrize("change", [_drop_a_shift, _also_writes_its_source], ids=["drops_a_views_shift", "writes_its_source_cache"])
def test_a_broken_cache_load_is_rejected_by_name(change):
    model, x1, t = _prepared()
    step = _step(model, x1, t, executor=_load_mutant(change)())
    with pytest.raises(AssertionError, match=r"cache_load launch 0 \(cache_load\)"):
        fsc.walk_loads(step, model=model)
