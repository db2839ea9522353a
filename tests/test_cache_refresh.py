"""A compiled fused step takes a new dense pass in place (`FusedStep.refresh`), checked on the CPU.

The reference's samplers run a dense pass on the original and a sparse pass on the edit at every denoising step
(diffusion/samplers/ddim_ddpm_sampler.py `model_step`): new caches and new GroupNorm statistics each time.  Here that flow
runs through the launch records with the CPU simulator of tests/sim_executor.py, extended by the refresh hooks of the
product executor (`cache_load_supported` / `prepare_cache_load` / `repack_conv`) as torch restatements.
"""
import os
import sys
import warnings

import pytest
import torch

from conftest import REPO
from sige_b200.fused import FusedStep

sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "baseline"))

STEPS = 4
TOL = 2e-5         # tests/test_fused_cpu.py: simulated fp32 step vs the eager operator modules


def _sim(base=None):
    """A descriptor simulator (`base`, default tests/sim_executor.py's) with the refresh hooks."""
    from sim_executor import SimExecutor

    class RefreshSim(base or SimExecutor):
        """The simulator with `sige_cache_load` and the weight re-pack, restated in torch."""

        def __init__(self):
            super().__init__()
            self.loads = 0

        def cache_load_supported(self, cache=None):
            return True

        def prepare_cache_load(self, entries):
            def run(_stream):
                self.loads += 1
                for (src, raw, views) in entries:
                    if raw is not None:
                        raw.copy_(src.to(raw.dtype).expand(raw.shape[0], *src.shape[1:]))
                    for (v, sc, sh, act) in views:
                        z = src.float()
                        if sc is not None:
                            z = z * sc.view(1, -1, 1, 1)
                        if sh is not None:
                            z = z + sh.view(1, -1, 1, 1)
                        if act == "swish":
                            z = z * torch.sigmoid(z)
                        v.copy_(z)

            return run

        def repack_conv(self, fc):
            pass            # the simulator reads spec.weight / spec.bias at every launch

    return RefreshSim()


def _exact_or_declines(model, dense_inputs, sparse_args, masks, make_ex):
    """Two dense passes (the second on another original); after the second the compiled step either declines, reporting why,
    or refreshes to exactly what a step compiled afresh on the new caches computes."""
    with warnings.catch_warnings(), torch.no_grad():
        warnings.simplefilter("ignore")
        model.set_mode("full")
        model(*dense_inputs[0])
        model.set_masks(masks)
        model.set_mode("sparse")
        step = FusedStep(model, *sparse_args, executor=make_ex())
        first = step(*sparse_args).clone()
        model.set_mode("full")
        model(*dense_inputs[1])
        model.set_mode("sparse")
        fresh = FusedStep(model, *sparse_args, executor=make_ex()).output.clone()
        if step.refresh_reason is not None:
            assert not step.refresh()
            return step
        assert step.refresh()
        out = step(*sparse_args).clone()
    assert not torch.equal(first, fresh), "the second dense pass must change the result"
    assert torch.equal(out, fresh), float((out - fresh).abs().max())
    return step


def _model(kind, cfg):
    import loader
    from sige_b200.workloads.ddpm import SIGEDDPMUNet, init_deterministic

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if kind == "reference":
            if not loader.available():
                pytest.skip("baseline/_ref absent (python baseline/build_ref.py)")
            model = loader.reference_ddpm_on_this_repo(cfg)
        else:
            model = SIGEDDPMUNet(cfg)
        return init_deterministic(model, seed=0).eval()


def _flow(cfg):
    """(mask, [(x_t, t)] per step): the sampler's x_t pair [original, edit] and its timestep, different every step."""
    from sige_b200.workloads.ddpm import synthetic_inputs

    x0, x1, mask, t = synthetic_inputs(cfg, 0.05, seed=0)
    steps = []
    for s in range(STEPS):
        g = torch.Generator().manual_seed(s)
        noise = torch.randn(x0.shape, generator=g)
        xt = torch.cat([x0, x1], 0) * (1.0 - 0.1 * s) + 0.1 * s * noise
        steps.append((xt, t + 37 * s))
    return mask, steps


@pytest.mark.parametrize("kind", ["reference", "intree"])
def test_one_step_object_serves_every_denoising_step(kind):
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import downsample_mask
    from sige_b200.fused import FusedStep
    from sige_b200.workloads.ddpm import DDPMConfig
    from sim_executor import SimExecutor

    cfg = DDPMConfig.small()
    model = _model(kind, cfg)
    mask, flow = _flow(cfg)
    step = None
    with torch.no_grad():
        for s, (xt, t) in enumerate(flow):
            model.set_mode("full")
            model(xt[:1], t)
            if s == 0:
                model.set_masks(downsample_mask(mask, min_res=8))
            model.set_mode("sparse")
            if step is None:
                step = FusedStep(model, xt[1:], t, executor=_sim())
                assert step.refresh_reason is None, step.refresh_reason
                assert step.eager_nodes == [] and any(f.spec.refold for f in step.fused)
            else:
                loads = step.ex.loads
                assert step.refresh(), "a dense pass with the same shapes is taken in place"
                assert step.ex.loads == loads + 1, "every cached buffer is reloaded by one cache-load launch"
            out = step(xt[1:], t).clone()
            fresh = FusedStep(model, xt[1:], t, executor=_sim()).output
            assert torch.equal(out, fresh), "step %d: %g" % (s, float((out - fresh).abs().max()))
            with reference_cpu_runtime():
                eager = model(xt[1:], t)
            assert torch.allclose(out, eager, atol=TOL), "step %d: %g" % (s, float((out - eager).abs().max()))
            if s:
                assert float((out - prev).abs().max()) > 1e-3, "the refreshed step must follow the new dense pass"
            prev = out
        # the simulator without the hooks keeps the torch restatement and refreshes as well
        plain = FusedStep(model, xt[1:], t, executor=SimExecutor())
        assert plain.refresh_reason == "the executor cannot re-pack folded weights"
        assert not plain.refresh()


# ---------------------------------------------------------------------------------------------------------------------
# declines: each one recompiles and gives today's result
# ---------------------------------------------------------------------------------------------------------------------
def _block_model():
    """A one-block model: Gather(scale, shift from the dense pass) -> 3x3 conv -> Scatter into the dense pass's cache."""
    import sige.nn as snn

    class Block(snn.SIGEModel):
        def __init__(self, variant):
            super().__init__()
            self.variant = variant
            self.conv = snn.SIGEConv2d(64, 64, 3, padding=1)
            self.gather = snn.Gather(self.conv, (6, 6), activation_name="swish")
            self.scatter = snn.Scatter(self.gather)
            self.stats = {}

        def forward(self, x):
            if self.mode == "full":
                self.gather(x)
                self.stats[0] = 1.0 + 0.1 * x.mean((0, 2, 3)).view(1, -1, 1, 1)
                return self.scatter(self.conv(x * self.stats[0]))
            scale = self.stats[0]
            if self.variant == "trace_time":
                scale = scale * torch.ones_like(scale)           # made by the forward at trace time: held by no module
            h = self.gather(x, scale, None)
            y = self.scatter(self.conv(h))
            if self.variant == "eager_cache":
                y = torch.maximum(y, self.scatter.original_outputs[0])          # an eager node reading a cache
            return y

    class StackMath(Block):
        """The statistics reach a Gather whose tile stack is then pointwise math the lowering runs as recorded (GauGAN's
        `main_gather(x, norm_0.scale, ...)` before its SPADE math): the materialised gather reads them."""

        def forward(self, x):
            if self.mode == "full":
                return super().forward(x)
            h = torch.nn.functional.leaky_relu(self.gather(x, self.stats[0], None), 0.2)
            return self.scatter(self.conv(h))

    Block.StackMath = StackMath

    return Block


@pytest.mark.parametrize("variant", ["trace_time", "eager_cache", "cache_dtype"])
def test_a_step_that_cannot_take_a_dense_pass_declines_and_recompiles(variant):
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import downsample_mask
    from sige_b200.fused import FusedStep

    torch.manual_seed(0)
    model = _block_model()("trace_time" if variant == "trace_time" else ("eager_cache" if variant == "eager_cache" else "plain")).eval()
    x0 = torch.randn(1, 64, 24, 24)
    mask = torch.zeros(24, 24, dtype=torch.bool)
    mask[5:11, 13:20] = True
    x1 = x0 + 0.5 * mask * torch.randn(1, 64, 24, 24)
    with warnings.catch_warnings(), torch.no_grad():
        warnings.simplefilter("ignore")
        model.set_mode("full")
        model(x0)
        model.set_masks(downsample_mask(mask, min_res=6))
        model.set_mode("sparse")
        step = FusedStep(model, x1, executor=_sim())
        if variant == "cache_dtype":
            assert step.refresh_reason is None, step.refresh_reason     # known only when the new cache is looked up
        else:
            assert step.refresh_reason is not None
            assert ("held by no module" in step.refresh_reason) if variant == "trace_time" else ("read as it is" in step.refresh_reason)
        model.set_mode("full")
        model(x0 * 0.7)
        if variant == "cache_dtype":
            model.scatter.original_outputs[0] = model.scatter.original_outputs[0].double()
        model.set_mode("sparse")
        before = step(x1).clone()
        assert not step.refresh(), "nothing may change when the step declines"
        assert step.refresh_reason is not None
        if variant == "cache_dtype":
            assert "torch.float64" in step.refresh_reason, step.refresh_reason
        assert torch.equal(step(x1), before)
        if variant == "cache_dtype":
            model.scatter.original_outputs[0] = model.scatter.original_outputs[0].float()
        fresh = FusedStep(model, x1, executor=_sim()).output
        with reference_cpu_runtime():
            eager = model(x1)
    assert torch.allclose(fresh, eager, atol=TOL), float((fresh - eager).abs().max())


def _toy_inputs():
    from sige.utils import downsample_mask

    torch.manual_seed(0)
    x0 = torch.randn(1, 64, 24, 24)
    mask = torch.zeros(24, 24, dtype=torch.bool)
    mask[5:11, 13:20] = True
    x1 = x0 + 0.5 * mask * torch.randn(1, 64, 24, 24)
    return x0, x1, downsample_mask(mask, min_res=6)


def test_statistics_read_by_a_materialised_gather_are_refreshed():
    from oracle.cpu_runtime import reference_cpu_runtime

    model = _block_model().StackMath("plain").eval()
    x0, x1, masks = _toy_inputs()
    with reference_cpu_runtime():
        step = _exact_or_declines(model, [(x0,), (x0 * 0.7 + 0.3,)], (x1,), masks, _sim)
        assert step.refresh_reason is None and any(n.startswith("gather(") for n in step.eager_nodes)
        with torch.no_grad():
            eager = model(x1)
    assert torch.allclose(step.outputs, eager, atol=TOL), float((step.outputs - eager).abs().max())


@pytest.mark.parametrize("which", ["spade-intree", "spade-reference", "gaugan-mini", "sd-mini"])
def test_gaugan_and_sd_steps_refresh_exactly_or_decline(which):
    """Every GauGAN / Stable Diffusion step this repository compiles: exact after a refresh, or declined with a reason."""
    import consumers
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import downsample_mask

    if which != "spade-intree" and not consumers.available():
        pytest.skip("baseline/_ref absent (python baseline/build_ref.py)")
    make_ex = _sim
    if which.startswith("spade"):
        import test_spade_generator as TS
        from sige_b200.workloads import gaugan_spade as GS

        StridedSim, _ = TS._sims()
        make_ex = lambda: _sim(StridedSim)           # noqa: E731
        net = GS.build_gaugan_spade("mini") if which == "spade-intree" else consumers.build_gaugan("mini")
        s0, s1, mask = consumers.gaugan_inputs("mini")
        dense, args, masks = [(s0,), (s1,)], (s1,), TS._pyramid(mask)
    elif which == "gaugan-mini":
        import test_spade_generator as TS

        net = consumers.build_gaugan_mini()
        s0, s1, mask = consumers.gaugan_inputs()
        dense, args, masks = [(s0,), (s1,)], (s1,), TS._pyramid(mask)
    else:
        net = consumers.build_sd_mini()
        x0, x1, mask, ts, ctx = consumers.sd_inputs()
        dense, args, masks = [(x0, ts, ctx), (x0 * 0.7 + 0.3 * x1, ts, ctx)], (x1, ts, ctx), downsample_mask(mask, min_res=(4, 4), dilation=1)
    with reference_cpu_runtime():
        step = _exact_or_declines(net, dense, args, masks, make_ex)
    if which in ("gaugan-mini", "sd-mini"):
        assert step.refresh_reason is not None, "eager operator modules in these steps read their caches"
