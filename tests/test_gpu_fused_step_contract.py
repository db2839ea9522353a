"""Compiled fused steps on the H100, walked launch by launch against float64 restatements of their records
(tests/fused_step_contract.py): every launch within its bound and nothing else of the whole state touched; then the captured
graph (with programmatic dependent launch where the step uses it) and the eager launch sequence each leave the whole state
bitwise where the synchronised walk left it.  Two mutants of the executor, each breaking one launch's translation, must be
rejected by name."""
import copy
import os
import re
import sys
import time
import warnings

import pytest
import torch

from conftest import REPO

sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "baseline"))

import fused_step_contract as fsc  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _exact_fp32_dense_pass():
    saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _recording():
    from sige_b200.fused import CudaExecutor

    return fsc.recording(CudaExecutor)


def _model(cfg, dtype):
    from sige_b200.workloads.ddpm import SIGEDDPMUNet, init_deterministic

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model = init_deterministic(SIGEDDPMUNet(cfg), seed=0).eval()
    return model.to(DEV).to(dtype).to(memory_format=torch.channels_last)


def _prepared(cfg, dtype, ratio=0.05):
    from sige.utils import downsample_mask
    from sige_b200.workloads.ddpm import synthetic_inputs

    model = _model(cfg, dtype)
    x0, x1, mask, t = synthetic_inputs(cfg, ratio, seed=0)
    with torch.no_grad():
        model.set_mode("full")
        model(x0.to(DEV).to(dtype), t.to(DEV))
        model.set_masks(downsample_mask(mask.to(DEV), min_res=8))
        model.set_mode("sparse")
    return model, x1.to(DEV).to(dtype), t.to(DEV)


def _step(model, *args, step_dtype, executor_cls=None, **opts):
    from sige_b200.fused import FusedStep

    with torch.no_grad():
        return FusedStep(model, *args, executor=(executor_cls or _recording())(torch.device(DEV), step_dtype), dtype=step_dtype, **opts)


def _walk_and_replay(step, tag, program=None, model=None, replays=True):
    """(a) the walk, (c) every non-eager entry checked, (b) graph replay and eager run bitwise equal to the walk; then (d) the walk
    again from the start with the program's write footprint poisoned, which must end where the first walk ended outside the
    padding rows, and (e) graph replay and eager run from that poisoned start bitwise equal to the poisoned walk.  The start
    holds every intermediate a run on the same inputs left there, so only (d) and (e) see a launch that reads a byte before the
    launch that writes it (in program order, or under programmatic dependent launch) has written it."""
    t0 = time.perf_counter()
    fsc.poison_padding(step)                 # (the walk poisons them too: replays start from the same padding rows)
    state = fsc.State(step, model)
    start = state.snapshot()
    res = fsc.walk(step, program, model=model, state=state)
    fsc.checked_all(step, res, program)
    walked = state.snapshot()
    if replays:
        assert program is None or program is step.low.epilogue
        # the sparse_update epilogue: its first call runs it and captures it, the second replays the captured graph
        runs = ([("replay", step.replay), ("run_eager", step.run_eager)] if program is None else
                [("sparse_update (launches)", step.sparse_update), ("sparse_update (graph replay)", step.sparse_update)])
        _replay(state, start, walked, runs, tag, "the synchronised walk")
    t1 = time.perf_counter()
    res2, poisoned, walked2, n = fsc.poisoned_walk(step, res, start, walked, program, model=model, state=state)
    fsc.checked_all(step, res2, program)
    if replays:
        runs = ([("replay", step.replay), ("run_eager", step.run_eager)] if program is None else
                [("sparse_update (graph replay)", step.sparse_update), ("sparse_update (launches)", lambda: step._run(step.low.epilogue))])
        _replay(state, poisoned, walked2, runs, tag + " (poisoned)", "the poisoned walk")
    print(fsc.summary(tag, res) + "; %.2f s with replays; %d bytes poisoned, +%.2f s" % (time.perf_counter() - t0, n, time.perf_counter() - t1))
    return res


def _replay(state, start, walked, runs, tag, what):
    for name, run in runs:
        state.restore(start)
        torch.cuda.synchronize()
        with torch.no_grad():
            run()
        torch.cuda.synchronize()
        diff = state.differs(walked)
        assert diff is None, "%s: %s leaves the state different from %s: %s" % (tag, name, what, diff)


def _walk_loads_and_replay(step, tag, model):
    """walk_loads, then again from its write footprint poisoned, then `load_caches` from that poisoned start: bitwise equal to
    the poisoned walk."""
    t0 = time.perf_counter()
    state = fsc.State(step, model)
    start = state.snapshot()
    res = fsc.walk_loads(step, model=model, state=state)
    walked = state.snapshot()
    t1 = time.perf_counter()
    _, poisoned, walked2, n = fsc.poisoned_walk(step, res, start, walked, model=model, state=state, loads=True)
    stream = torch.cuda.current_stream().cuda_stream
    _replay(state, poisoned, walked2, [("load_caches", lambda: step.low.load_caches(stream))], tag + " (poisoned)", "the poisoned walk")
    print(fsc.summary(tag, res) + "; %d bytes poisoned, +%.2f s" % (n, time.perf_counter() - t1))
    return res


GPU_OPTS = [
    {"tc5": False, "producer_preop": False, "pdl": False, "fused_attention": False, "sparse_stem": False},
    {"tc5": False, "producer_preop": True, "pdl": False},
    {"tc5": True, "producer_preop": True, "pdl": False, "fuse_shortcut": False},
    {"tc5": True, "producer_preop": True, "pdl": True},
    {"tc5": True, "producer_preop": False, "pdl": True},
]


@pytest.mark.parametrize("opts", GPU_OPTS)
def test_fp16_ddpm_small_step_meets_its_records(opts):
    from sige_b200.workloads.ddpm import DDPMConfig

    model, x1, t = _prepared(DDPMConfig.small(), torch.float16)
    step = _step(model, x1, t, step_dtype=torch.float16, **opts)
    res = _walk_and_replay(step, "ddpm_small fp16 %s" % opts, model=model)
    assert res["kinds"]["conv"].launches == len(step.fused)
    assert (res["eager"] > 0) == (not opts.get("fused_attention", True))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("tag", ["ddpm_small", "ddpm256"])
def test_fp32_model_step_as_benchmarked_meets_its_records(tag, dtype):
    from sige_b200.workloads.ddpm import DDPMConfig

    cfg = DDPMConfig.small() if tag == "ddpm_small" else DDPMConfig()
    model, x1, t = _prepared(cfg, torch.float32)
    step = _step(model, x1, t, step_dtype=dtype)
    res = _walk_and_replay(step, "%s fp32 model, %s step" % (tag, dtype), model=model)
    assert res["eager"] == 0
    if tag == "ddpm256":
        assert res["kinds"]["conv"].launches == 86
        assert res["kinds"].get("attention", fsc.KindStats()).launches + res["kinds"].get("sparse_attention", fsc.KindStats()).launches == 6


def test_sparse_attention_inside_the_step_meets_its_records():
    from sige_b200.workloads.ddpm import DDPMConfig

    class NoClusterAttention(_recording()):
        def attention_supported(self, n_tokens, channels):
            return False

    model, x1, t = _prepared(DDPMConfig.small(), torch.float16)
    step = _step(model, x1, t, step_dtype=torch.float16, executor_cls=NoClusterAttention)
    res = _walk_and_replay(step, "ddpm_small sparse attention", model=model)
    assert res["kinds"]["sparse_attention"].launches == 4 and res["eager"] == 0


def test_batch_of_three_edits_meets_its_records():
    from sige.utils import downsample_mask
    from sige_b200.masks import stack_mask_pyramids
    from sige_b200.workloads.ddpm import DDPMConfig, synthetic_inputs

    cfg = DDPMConfig.small()
    model, _, t = _prepared(cfg, torch.float16)
    edits = []
    for e, (ratio, shift) in enumerate([(0.05, (0, 0)), (0.02, (-14, 9)), (0.09, (11, -13))]):
        x0, x1, mask, _ = synthetic_inputs(cfg, ratio, seed=0, edit_seed=e)
        edits.append((x0 + torch.roll(x1 - x0, shift, (2, 3)), torch.roll(mask, shift, (0, 1))))
    model.set_masks(stack_mask_pyramids([downsample_mask(m.to(DEV), min_res=8) for _, m in edits]))
    xb = torch.cat([x for x, _ in edits], 0).to(DEV).half()
    step = _step(model, xb, t, step_dtype=torch.float16)
    assert any(f.spec.tile_img is not None for f in step.fused)
    _walk_and_replay(step, "ddpm_small batch of 3", model=model)


def test_rebound_edits_meet_their_records():
    from sige.utils import downsample_mask
    from sige_b200.workloads.ddpm import DDPMConfig, synthetic_inputs

    cfg = DDPMConfig.small()
    model, x1, t = _prepared(cfg, torch.float16)
    step = _step(model, x1, t, step_dtype=torch.float16, headroom=0.6)
    _walk_and_replay(step, "ddpm_small headroom 0.6", model=model)
    x0, _, _, _ = synthetic_inputs(cfg, 0.05, seed=0)
    _, x_b, mask_b, _ = synthetic_inputs(cfg, 0.03, seed=0, edit_seed=5)
    mask_b = torch.roll(mask_b, (9, -11), (0, 1))
    x_b = (x0 + torch.roll(x_b - x0, (9, -11), (2, 3))).to(DEV).half()
    masks = downsample_mask(mask_b.to(DEV), min_res=8)
    model.set_masks(masks)
    with torch.no_grad():
        assert step.rebind()
    fsc.cached_state_after_rebind(step)
    step.static_inputs[0].copy_(x_b)
    _walk_and_replay(step, "ddpm_small after rebind", model=model)
    with torch.no_grad():
        assert step.rebind_device(masks)
    assert step.async_ok()
    fsc.cached_state_after_rebind(step)
    _walk_and_replay(step, "ddpm_small after rebind_device", model=model)


def test_sparse_update_epilogue_meets_its_records():
    import test_sparse_update_fused as TSU
    from sige.utils import downsample_mask
    from sige_b200.workloads.ddpm import DDPMConfig

    cfg = DDPMConfig.small()
    x0, t, edits = TSU._edits(cfg)
    model = _model(cfg, torch.float16)
    x0, t = x0.to(DEV).half(), t.to(DEV)
    with torch.no_grad():
        TSU._dense(model, x0, t)
        model.set_cache_id(1)
        model.set_masks(downsample_mask(edits[0][1].to(DEV), min_res=8))
    step = _step(model, (edits[0][0].to(DEV) * 1.1).half(), t + 10, step_dtype=torch.float16)
    assert step.sparse_update_supported, step.sparse_update_reason
    _walk_and_replay(step, "ddpm_small main (sparse_update)", model=model)
    kinds = [k for k, _ in step.low.epilogue]
    assert kinds.count("writeback") == 1 and kinds.count("conv") > 0
    _walk_and_replay(step, "ddpm_small sparse_update epilogue", step.low.epilogue, model=model)


# ---------------------------------------------------------------------------------------------------------------------
# the GauGAN miniatures from an fp32 model: separable, narrow, ReLU-epilogue and modulated launches (sub-mobile), channel-window
# and wgmma-modulated launches (SPADE generator)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_sub_mobile_gaugan_step_meets_its_records(dtype):
    from sige.utils import dilate_mask, downsample_mask
    from sige_b200.workloads import gaugan_gc as G

    net = G.build_gaugan_gc("mini").to(DEV)
    G.run_gaugan_gc(net, downsample_mask, dilate_mask, device=DEV, size="mini", fused=lambda n: n.set_fused(False))
    step = _step(net, G.gaugan_gc_inputs("mini")[1].to(DEV), step_dtype=dtype)
    res = _walk_and_replay(step, "gaugan_gc mini %s" % dtype, model=net)
    specs = [f.spec for f in step.fused]
    # the dense blocks' SPADE modulations stay recorded torch calls here (sige_spade_modulate declines their operands): eager
    assert res["kinds"]["separable"].launches == 12 and res["eager"] > 0
    assert any(s.modulation is not None for s in specs) and any(s.epilogue_act == "relu" for s in specs) and any(s.Cin % 64 for s in specs)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_spade_generator_step_meets_its_records(dtype):
    import consumers
    from sige.utils import dilate_mask, downsample_mask
    from sige_b200.workloads import gaugan_spade as GS

    net = GS.build_gaugan_spade("mini").to(DEV)
    consumers.run_gaugan(net, downsample_mask, dilate_mask, device=DEV, size="mini", fused=lambda n: n.set_fused(False))
    step = _step(net, consumers.gaugan_inputs("mini")[1].to(DEV), step_dtype=dtype)
    res = _walk_and_replay(step, "gaugan_spade mini %s" % dtype, model=net)
    windowed = [f for f in step.fused if not f.spec.src_is_stack and not f.spec.srcs[0][0].is_contiguous(memory_format=torch.channels_last)]
    assert sum(1 for f in step.fused if f.spec.modulation is not None) == 12 and len(windowed) == 12
    assert res["kinds"]["conv"].launches == len(step.fused)


# ---------------------------------------------------------------------------------------------------------------------
# mutants: the executor hands one launch a wrong translation of its record
# ---------------------------------------------------------------------------------------------------------------------
def _flip_flag(s):
    if s.shortcut is None or s.shortcut[3] is None or not bool((s.shortcut[3] != 0).any()):
        return None
    src, w, b, flags = s.shortcut
    f = flags.clone()
    i = int((f != 0).nonzero()[0])
    f[i] = 0
    m = copy.copy(s)
    m.shortcut = (src, w, b, f)
    return m


def _zero_bias(s):
    if s.bias is None or float(s.bias.abs().max()) == 0:
        return None
    m = copy.copy(s)
    m.bias = torch.zeros_like(s.bias)
    return m


@pytest.mark.parametrize("mutate", [_flip_flag, _zero_bias], ids=["flipped_shortcut_flag", "zero_bias"])
def test_a_mistranslated_launch_is_rejected_by_name(mutate):
    from sige_b200.workloads.ddpm import DDPMConfig

    class Mutant(_recording()):
        victim = None

        def prepare_conv(self, fc):
            m = None if self.victim is not None else mutate(fc.spec)
            if m is None:
                return super().prepare_conv(fc)
            self.victim = fc.name
            orig, fc.spec = fc.spec, m
            try:
                super().prepare_conv(fc)
            finally:
                fc.spec = orig

    model, x1, t = _prepared(DDPMConfig.small(), torch.float16)
    step = _step(model, x1, t, step_dtype=torch.float16, executor_cls=Mutant)
    assert step.ex.victim is not None
    with pytest.raises(AssertionError, match=r"conv launch \d+ \(%s\)" % step.ex.victim.replace(".", r"\.")) as err:
        fsc.walk(step, model=model)
    print("[fused step contract] mutant %s rejected: %s" % (mutate.__name__, str(err.value).splitlines()[0][:200]))


# ---------------------------------------------------------------------------------------------------------------------
# the Stable Diffusion decoder (its fixed-capacity q stack, the D = 512 sparse attention, the 4 -> 512 stem), batches of label
# edits and the cache load of a new edit
# ---------------------------------------------------------------------------------------------------------------------
def _sd(size="mini"):
    from sige.utils import downsample_mask
    from sige_b200.workloads import sd_decoder as SD

    net = SD.build_sd_decoder(size).to(DEV)
    z0, z1, mask = (t.to(DEV) for t in SD.sd_decoder_inputs(size))
    with torch.no_grad():
        net.set_mode("full")
        net(z0)
        net.set_mode("sparse")
        net.set_masks(downsample_mask(mask, min_res=(4, 4), dilation=0))
    return net, z1, mask


def _sd_launches(step, res):
    assert res["kinds"]["sparse_attention"].launches == 1 and res["poisoned"] > 0
    assert sum(1 for r in step.low.conv_ins if int(r.weight.shape[0]) == 512) == 1 and res["kinds"]["conv_in"].launches >= 1


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_sd_decoder_step_meets_its_records_before_and_after_a_rebind(dtype):
    from sige.utils import downsample_mask

    net, z1, mask = _sd()
    step = _step(net, z1, step_dtype=dtype)
    _sd_launches(step, _walk_and_replay(step, "sd_decoder mini %s" % dtype, model=net))
    mask2 = torch.zeros_like(mask)
    mask2[12:20, 6:15] = True
    net.set_masks(downsample_mask(mask2, min_res=(4, 4), dilation=0))
    with torch.no_grad():
        assert step.rebind()
    _walk_loads_and_replay(step, "sd_decoder mini %s loads after rebind" % dtype, net)
    _sd_launches(step, _walk_and_replay(step, "sd_decoder mini %s after rebind" % dtype, model=net))


def test_full_sd_decoder_step_meets_its_records():
    """The in-tree "full" decoder: 4096 keys, so the D = 512 attention splits its key range over a cluster."""
    import step_kernel_contracts as skc

    net, z1, _ = _sd("full")
    torch.cuda.reset_peak_memory_stats()
    step = _step(net, z1, step_dtype=torch.float16)
    (rec,) = [r for k, r, _ in step.ex.records.values() if k == "sparse_attention"]
    nq, nk = int(rec["q"].shape[-2]), int(rec["k"].shape[-2])
    cs = skc.wide_cluster(nq, nk, 1, torch.cuda.get_device_properties(0).multi_processor_count)
    res = _walk_and_replay(step, "sd_decoder full fp16 (Nq %d, Nk %d, cluster %d)" % (nq, nk, cs), model=net)
    print("[fused step contract] sd_decoder full: peak %.2f GB" % (torch.cuda.max_memory_allocated() / 2 ** 30))
    _sd_launches(step, res)
    assert nk == 4096 and cs > 1


def _batched(which):
    import test_fused_step_contract as TF
    import test_gpu_batched_gaugan as TG
    from sige_b200.workloads import gaugan_gc as G

    net = TG._net(which)
    s0, s1s, masks = (t.to(DEV) for t in G.gaugan_gc_edits("mini", 5))
    with torch.no_grad():
        net.set_mode("full")
        net(s0)
        net.set_mode("sparse")
        net.set_masks(TF._no_tiles_batch(TG._pyr, masks[[0, 1, 2]]))       # the third edit has no tiles
    return TG, net, s1s, masks


@pytest.mark.parametrize("which", ["gc", "spade"])
def test_batched_gaugan_step_meets_its_records(which):
    TG, net, s1s, masks = _batched(which)
    step = _step(net, s1s[[0, 1, 2]], step_dtype=torch.float16, headroom=0.5)
    res = _walk_and_replay(step, "gaugan_%s mini fp16 batch of 3, the third edit without tiles" % which, model=net)
    assert any(f.spec.tile_img is not None for f in step.fused)
    assert all(bool((sl.buf.view(3, sl.cap, 2)[2, :, 0] <= fsc.NONE_BELOW).all()) for sl in step.low.slots.values())
    assert (res["kinds"].get("separable", fsc.KindStats()).launches > 0) == (which == "gc")
    net.set_masks(TG._batch(masks[[1, 3, 4]]))
    with torch.no_grad():
        assert step.rebind()
    step.static_inputs[0].copy_(s1s[[1, 3, 4]])
    _walk_and_replay(step, "gaugan_%s mini fp16 next batch" % which, model=net)


def test_cache_loads_meet_their_records_after_a_refresh_and_after_a_rebind():
    from sige_b200.workloads.ddpm import DDPMConfig, synthetic_inputs

    model, x1, t = _prepared(DDPMConfig.small(), torch.float16)
    step = _step(model, x1, t, step_dtype=torch.float16)
    x0, _, _, _ = synthetic_inputs(DDPMConfig.small(), 0.05, seed=0)
    with torch.no_grad():
        model.set_mode("full")
        model((x0 * 0.7).to(DEV).half(), t)
        model.set_mode("sparse")
        assert step.refresh()
    res = _walk_loads_and_replay(step, "ddpm_small fp16 loads after refresh", model)
    assert res["kinds"]["cache_load"].launches == 1

    import consumers
    from sige.utils import dilate_mask, downsample_mask
    from sige_b200.workloads import gaugan_spade as GS

    net = GS.build_gaugan_spade("mini").to(DEV)
    consumers.run_gaugan(net, downsample_mask, dilate_mask, device=DEV, size="mini", fused=lambda n: n.set_fused(False))
    step = _step(net, consumers.gaugan_inputs("mini")[1].to(DEV), step_dtype=torch.float16)
    with torch.no_grad():
        assert step.rebind()
    res = _walk_loads_and_replay(step, "gaugan_spade mini fp16 loads after rebind", net)
    assert res["kinds"]["cache_load"].launches == 1


# mutants of the separable and sparse-attention translations; every access stays inside its allocation
def test_a_separable_launch_without_per_image_operands_is_rejected_by_name():
    """The batch's separable launch without SIGE_CONV_PER_IMAGE_OPERANDS: its E lists read as one shared list of E * cap rows, so
    every image takes the tiles of every edit (all of them inside each image, which share one extent)."""
    from sige_b200._cabi import CONV_PER_IMAGE_OPERANDS

    class NoPerImage(_recording()):
        victim = None

        def prepare_separable(self, rec):
            if self.victim is not None or rec.tile_img is None:
                return super().prepare_separable(rec)
            self.victim = rec.name
            fn = super().prepare_separable(rec)
            ops, branches = self.ops, [self._separable_weights(dw, w, b) + (d.raw,) for (dw, w, b, d) in rec.branches]
            src = rec.src[:, rec.c0:rec.c0 + rec.Cin]

            def run(_stream):
                ops.separable_conv(src, branches, rec.idx, src_stack=False, offset=rec.off, batch=rec.batch, flags=0)
            del self.records[id(fn)]
            return self._keep("separable", run, rec)

    assert CONV_PER_IMAGE_OPERANDS == 128
    TG, net, s1s, _ = _batched("gc")
    step = _step(net, s1s[[0, 1, 2]], step_dtype=torch.float16, executor_cls=NoPerImage)
    assert step.ex.victim is not None
    (rec,) = [r for r in step.low.separable if r.name == step.ex.victim]
    with torch.no_grad():
        for br in rec.branches:      # the stray tiles rewrite what the build's run left there: move it off first
            br[3].raw.add_(0.5)
    with pytest.raises(AssertionError, match=r"separable launch \d+ \(%s\)" % re.escape(step.ex.victim)) as err:
        fsc.walk(step, model=net)
    print("[fused step contract] mutant separable without per-image operands rejected: %s" % str(err.value).splitlines()[0][:200])


def test_a_sparse_attention_over_one_key_fewer_is_rejected_by_name():
    class OneKeyShort(_recording()):
        def prepare_sparse_attention(self, q, k, v, scale, out):
            fn = super().prepare_sparse_attention(q, k[..., :-1, :], v[..., :-1, :], scale, out)
            del self.records[id(fn)]
            return self._keep("sparse_attention", fn, dict(q=q, k=k, v=v, scale=scale, out=out))

    net, z1, _ = _sd()
    step = _step(net, z1, step_dtype=torch.float16, executor_cls=OneKeyShort)
    with pytest.raises(AssertionError, match=r"sparse_attention launch \d+ \(sparse_attention\)") as err:
        fsc.walk(step, model=net)
    print("[fused step contract] mutant sparse attention over Nk - 1 keys rejected: %s" % str(err.value).splitlines()[0][:200])
