"""The reference samplers' per-step flow on the GPU: a dense pass on the original, then a sparse pass on the edit, at every
denoising step (diffusion/samplers/ddim_ddpm_sampler.py `model_step`).  One compiled fused step serves every step
(`FusedStep.refresh`), bitwise equal to a step compiled afresh on the same caches, within TOL_MAX of the eager modules."""
import os
import sys
import warnings

import pytest
import torch

from conftest import REPO

sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "baseline"))
pytestmark = pytest.mark.gpu
DEV = "cuda:0"
STEPS = 4
TOL_MAX = 5e-3            # tests/test_gpu_fused.py: fp16 step vs the reference, max-normalised
TOL_CACHE = 4e-3          # tests/test_gpu_sparse_update_fused.py: caches after an applied edit, max-normalised


@pytest.fixture(autouse=True)
def _exact_fp32_dense_pass():
    saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _err(a, b):
    a, b = a.float(), b.float()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-6))


def _models(kind, cfg):
    """(fused model, eager model) with the same weights: the reference's fp32 file with an fp16 step, or the in-tree model in
    fp16."""
    import loader
    from sige_b200.workloads.ddpm import SIGEDDPMUNet, init_deterministic

    out = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for _ in range(2):
            if kind == "reference":
                if not loader.available():
                    pytest.skip("baseline/_ref absent (python baseline/build_ref.py)")
                m = init_deterministic(loader.reference_ddpm_on_this_repo(cfg), seed=0).eval().to(DEV)
            else:
                m = init_deterministic(SIGEDDPMUNet(cfg), seed=0).eval().to(DEV).half()
            out.append(m)
    out[0].set_fused(True, dtype=torch.float16)
    out[1].set_fused(False)
    return out


def _flow(cfg, ratio, dtype, n_edits=1):
    from sige_b200.workloads.ddpm import synthetic_inputs

    x0, x1, mask, t = synthetic_inputs(cfg, ratio, seed=0)
    edits, masks = [x1], [mask]
    for e in range(1, n_edits):
        _, xe, me, _ = synthetic_inputs(cfg, ratio, seed=0, edit_seed=e)
        edits.append(xe)
        masks.append(me)
    steps = []
    for s in range(STEPS):
        g = torch.Generator().manual_seed(s)
        noise = 0.1 * s * torch.randn(x0.shape, generator=g)
        xt = torch.cat([x0] + edits, 0) * (1.0 - 0.1 * s) + noise
        steps.append((xt.to(DEV, dtype), (t + 97 * s).to(DEV)))
    return masks, steps


def _pyramid(masks):
    from sige.utils import downsample_mask
    from sige_b200.masks import stack_mask_pyramids

    pyr = [downsample_mask(m.to(DEV), min_res=8) for m in masks]
    return pyr[0] if len(pyr) == 1 else stack_mask_pyramids(pyr)


def _dense(model, xt, t):
    model.set_mode("full")
    model(xt[:1], t)
    model.set_mode("sparse")


@pytest.mark.parametrize("kind,ratio,n_edits", [("reference", 0.012, 1), ("intree", 0.012, 1), ("intree", 0.012, 4)])
def test_one_step_serves_the_sampler_flow(kind, ratio, n_edits):
    from sige_b200.fused import FusedStep
    from sige_b200.workloads.ddpm import DDPMConfig

    cfg = DDPMConfig()
    fused, eager = _models(kind, cfg)
    masks, flow = _flow(cfg, ratio, torch.float32 if kind == "reference" else torch.float16, n_edits)
    first = None
    with torch.no_grad():
        for s, (xt, t) in enumerate(flow):
            for m in (fused, eager):
                _dense(m, xt, t)
                if s == 0:
                    m.set_masks(_pyramid(masks))
            if first is None:
                out = fused(xt[1:], t)
                first = fused.fused_step
                assert first is not None and first.refresh_reason is None, first.refresh_reason
            else:
                torch.cuda.synchronize()
                torch.cuda.set_sync_debug_mode("error")
                try:
                    out = fused(xt[1:], t)               # refresh + replay: only enqueued work
                finally:
                    torch.cuda.set_sync_debug_mode("default")
                assert fused.fused_step is first, "step %d recompiled" % s
            fresh = FusedStep(fused, xt[1:], t, dtype=torch.float16).output
            assert torch.equal(out.to(torch.float16), fresh), "step %d: %g" % (s, _err(out, fresh))
            if n_edits == 1:          # (the eager operator modules take one edit at a time)
                ref = eager(xt[1:], t)
                assert _err(out, ref) <= TOL_MAX, "step %d: %g" % (s, _err(out, ref))


def test_apply_after_a_refresh_writes_the_new_caches_and_a_new_mask_rebinds():
    from sige_b200.fused import FusedStep
    from sige_b200.parallel import cache_tensors
    from sige_b200.workloads.ddpm import DDPMConfig, synthetic_inputs

    cfg = DDPMConfig()
    fused, eager = _models("intree", cfg)
    masks, flow = _flow(cfg, 0.012, torch.float16)
    with torch.no_grad():
        xt, t = flow[0]
        for m in (fused, eager):
            _dense(m, xt, t)
            m.set_masks(_pyramid(masks))
        fused(xt[1:], t)
        step = fused.fused_step
        assert step.sparse_update_supported, step.sparse_update_reason
        old = [(v, v.clone()) for _, v in cache_tensors(fused)]
        xt, t = flow[1]
        for m in (fused, eager):
            _dense(m, xt, t)
            m.set_sparse_update(True)
        fused(xt[1:], t)
        eager(xt[1:], t)
        assert fused.fused_step is step
        for (v, keep) in old:
            assert torch.equal(v, keep), "a cache of the previous dense pass was written"
        for (n, a), (_, b) in zip(cache_tensors(fused), cache_tensors(eager)):
            assert _err(a, b) <= TOL_CACHE, "%s: %g" % (n, _err(a, b))
        for m in (fused, eager):
            m.set_sparse_update(False)
        # the next dense pass with a new (smaller) mask: refresh, then rebind, in place
        xt, t = flow[2]
        _, _, mask_b, _ = synthetic_inputs(cfg, 0.008, seed=0, edit_seed=3)
        for m in (fused, eager):
            _dense(m, xt, t)
            m.set_masks(_pyramid([mask_b]))
        out = fused(xt[1:], t)
        assert fused.fused_step is step, "refresh + rebind recompiled"
        # (a step compiled for this smaller mask plans its launches for fewer tiles: the same sums in another order)
        fresh = FusedStep(fused, xt[1:], t, dtype=torch.float16).output
        assert _err(out, fresh) <= TOL_MAX and _err(out, eager(xt[1:], t)) <= TOL_MAX


@pytest.mark.parametrize("variant", ["trace_time", "eager_cache", "cache_layout", "stack_math"])
def test_model_call_refreshes_or_recompiles_the_one_block_models(variant):
    """Through the model call: a step that declines (statically, or when the new cache is looked up) reports why and the call
    recompiles; one that refreshes serves the call itself.  Either way the result is the eager modules'."""
    from sige.utils import downsample_mask
    from test_cache_refresh import _block_model, _toy_inputs

    Block = _block_model()
    torch.manual_seed(0)
    if variant == "stack_math":
        model = Block.StackMath("plain")
    else:
        model = Block(variant if variant != "cache_layout" else "plain")
    model = model.eval().to(DEV).half()
    x0, x1, _ = _toy_inputs()
    x0, x1 = x0.to(DEV).half(), x1.to(DEV).half()
    mask = (x1 != x0).any(1)[0]
    with warnings.catch_warnings(), torch.no_grad():
        warnings.simplefilter("ignore")
        model.set_mode("full")
        model(x0)
        model.set_masks(downsample_mask(mask, min_res=6))
        model.set_mode("sparse")
        model(x1)
        first = model.fused_step
        assert first is not None
        model.set_mode("full")
        model(x0 * 0.7 + 0.3)
        if variant == "cache_layout":         # (a cache in the other dense layout: the step was built for NCHW strides)
            c = model.scatter.original_outputs[0]
            assert c.is_contiguous()
            model.scatter.original_outputs[0] = c.contiguous(memory_format=torch.channels_last)
        model.set_mode("sparse")
        out = model(x1)
        if variant == "stack_math":
            assert model.fused_step is first and first.refresh_reason is None, first.refresh_reason
        else:
            assert model.fused_step is not first and first.refresh_reason is not None
        model.set_fused(False)
        ref = model(x1)
    assert _err(out, ref) <= TOL_MAX, _err(out, ref)


def test_spade_gaugan_miniature_refreshes_to_a_fresh_compile():
    """The in-tree SPADE GauGAN generator (fp32 model, fp16 step): its step takes a second dense pass in place, bitwise equal to a
    step compiled afresh on the new caches."""
    import consumers
    from sige.utils import dilate_mask, downsample_mask
    from sige_b200.fused import FusedStep
    from sige_b200.workloads import gaugan_spade as GS

    net = GS.build_gaugan_spade("mini").to(DEV)
    s0, s1, mask = (t.to(DEV) for t in consumers.gaugan_inputs("mini"))
    with torch.no_grad():
        net.set_fused(True, dtype=torch.float16)
        net.set_mode("full")
        net(s0)
        net.set_masks(downsample_mask(dilate_mask(mask, 1), min_res=(4, 8), dilation=0))
        net.set_mode("sparse")
        net(s1)
        first = net.fused_step
        assert first is not None and first.refresh_reason is None, first.refresh_reason
        net.set_mode("full")
        net(s1)                                  # another original: new caches and statistics
        net.set_mode("sparse")
        out = net(s1)
        assert net.fused_step is first
        fresh = FusedStep(net, s1, dtype=torch.float16).output
    assert torch.equal(out.to(torch.float16), fresh), _err(out, fresh)
