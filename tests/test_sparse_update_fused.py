"""sparse_update on the fused step, checked on the CPU: the argument checks of `sige_tile_writeback`, and the reference's
multi-step apply flow (one cache per sampler step, an edit applied with `sparse_update=True`, a second edit on top of it)
driven through `FusedStep` on a simulator of the launch descriptors with a torch write-back, against the reference's CPU
runtime (oracle/cpu_runtime.py) running the eager operator modules."""
import os
import sys
import warnings

import pytest
import torch

from conftest import REPO

sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "baseline"))

STEPS = [0, 1, 2]


# ---------------------------------------------------------------------------------------------------------------------
# sige_tile_writeback: argument errors before any device call
# ---------------------------------------------------------------------------------------------------------------------
def _entry(**kw):
    from sige_b200 import _cabi

    e = _cabi.WritebackEntry()
    e.src, e.dst, e.idx = 0x10000, 0x20000, 0x30000        # never dereferenced: validation fails (or N == 0) first
    e.N, e.B, e.C, e.H, e.W = 4, 1, 64, 16, 16
    e.src_dtype, e.dst_dtype, e.dst_layout = _cabi.F16, _cabi.F32, _cabi.NCHW
    e.offH = e.offW = 1
    e.strideH = e.strideW = 1
    e.Ro = e.So = 4
    for k, v in kw.items():
        setattr(e, k, v)
    return e


def _call(entries):
    from sige_b200 import _cabi

    lib = _cabi.lib()
    table = (_cabi.WritebackEntry * max(1, len(entries)))(*entries)
    rc = lib.sige_tile_writeback(table, len(entries), None)
    return rc, lib.sige_last_error()


def test_tile_writeback_argument_errors_need_no_device(cabi_lib):
    from sige_b200 import _cabi

    lib = _cabi.lib()
    assert lib.sige_tile_writeback(None, 1, None) != 0 and b"null entry table" in lib.sige_last_error()
    assert lib.sige_tile_writeback(None, 0, None) == 0
    rc, msg = _call([_entry(N=0)] * (_cabi.WRITEBACK_MAX_ENTRIES + 1))
    assert rc != 0 and b"at most 64" in msg
    rc, msg = _call([_entry(N=0, src=0, dst=0, idx=0)] * _cabi.WRITEBACK_MAX_ENTRIES)
    assert rc == 0                                            # N == 0 entries are no-ops, their pointers are not looked at
    rc, msg = _call([_entry(src_dtype=_cabi.BF16, dst_dtype=_cabi.F16)])
    assert rc != 0 and b"would round" in msg
    rc, msg = _call([_entry(src_dtype=_cabi.F32, dst_dtype=_cabi.F32)])
    assert rc != 0 and b"f16 or bf16" in msg
    rc, msg = _call([_entry(C=60)])
    assert rc != 0 and b"multiple of 8" in msg
    rc, msg = _call([_entry(N=0), _entry(src=0)])
    assert rc != 0 and b"entry 1: null buffer" in msg
    rc, msg = _call([_entry(Ro=9)])
    assert rc != 0 and b"output tile" in msg
    rc, msg = _call([_entry(dst_layout=5)])
    assert rc != 0 and b"layout" in msg
    rc, msg = _call([_entry(dst=0x20008)])
    assert rc != 0 and b"16-byte aligned" in msg


# ---------------------------------------------------------------------------------------------------------------------
# the apply flow on the simulator
# ---------------------------------------------------------------------------------------------------------------------
def _cdiv(a: int, b: int) -> int:
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def torch_writeback(entries) -> None:
    """Restatement of sige_tile_writeback (include/sige_b200.h) on torch tensors."""
    from sige_b200._cabi import TILE_NONE

    def pair(v):
        return (int(v[0]), int(v[1])) if isinstance(v, (tuple, list)) else (int(v), int(v))

    for (src, dst, idx, off, stride, tile) in entries:
        (oh, ow), (sh, sw), (ro, so) = pair(off), pair(stride), pair(tile)
        H, W = src.shape[2], src.shape[3]
        for ih, iw in idx.tolist():
            if ih == TILE_NONE:
                continue
            y, x = _cdiv(oh + ih, sh), _cdiv(ow + iw, sw)
            r0, r1, c0, c1 = max(y, 0), min(y + ro, H), max(x, 0), min(x + so, W)
            if r0 < r1 and c0 < c1:
                dst[:, :, r0:r1, c0:c1] = src[:, :, r0:r1, c0:c1].to(dst.dtype)


def _writeback_sim():
    from sim_executor import SimExecutor

    class WritebackSim(SimExecutor):
        def writeback_supported(self):
            return True

        def prepare_writeback(self, entries):
            def run(_stream):
                self.launches += 1
                torch_writeback(entries)

            return run

    return WritebackSim()


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


def _edits(cfg):
    from sige_b200.workloads.ddpm import synthetic_inputs

    x0, xa, mask_a, t = synthetic_inputs(cfg, 0.05, seed=0, edit_seed=1)
    _, xb, mask_b, _ = synthetic_inputs(cfg, 0.10, seed=0, edit_seed=2)
    xb = xa + (xb - x0)                                  # the second edit on top of the first
    return x0, t, ((xa, mask_a), (xb, mask_a | mask_b))


def _dense(model, x0, t):
    model.set_mode("full")
    for s in STEPS:                                      # a dense pass per sampler step, cached under its id
        model.set_cache_id(s)
        model(x0 * (1.0 + 0.1 * s), t + 10 * s)
    model.set_mode("sparse")


def _eager_flow(kind, cfg):
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import downsample_mask
    from sige_b200.parallel import cache_tensors

    x0, t, edits = _edits(cfg)
    outs = []
    with reference_cpu_runtime(), torch.no_grad():
        model = _model(kind, cfg)
        _dense(model, x0, t)
        model.set_sparse_update(True)
        for x_edit, mask in edits:
            model.set_masks(downsample_mask(mask, min_res=8))
            for s in STEPS:
                model.set_cache_id(s)
                outs.append(model(x_edit * (1.0 + 0.1 * s), t + 10 * s).clone())
    return outs, [(n, v.detach().float().clone()) for n, v in cache_tensors(model)]


def _fused_flow(kind, cfg):
    """The same flow through FusedStep: one step per cache id, compiled on the first edit with room for the second, which is
    installed in place (`rebind`) — the cached buffers then restart from the caches the first apply wrote."""
    from sige.utils import downsample_mask
    from sige_b200.fused import FusedStep
    from sige_b200.parallel import cache_tensors

    x0, t, edits = _edits(cfg)
    outs, steps = [], {}
    with torch.no_grad():
        model = _model(kind, cfg)
        _dense(model, x0, t)
        for e, (x_edit, mask) in enumerate(edits):
            model.set_masks(downsample_mask(mask, min_res=8))
            for s in STEPS:
                model.set_cache_id(s)
                args = (x_edit * (1.0 + 0.1 * s), t + 10 * s)
                if e == 0:
                    steps[s] = FusedStep(model, *args, executor=_writeback_sim(), headroom=2.0)
                else:
                    assert steps[s].rebind()
                st = steps[s]
                assert st.sparse_update_supported, st.sparse_update_reason
                assert st.eager_nodes == []
                outs.append(st(*args).clone())
                st.sparse_update()
    return outs, [(n, v.detach().float().clone()) for n, v in cache_tensors(model)], steps


@pytest.mark.parametrize("kind", ["intree", "reference"])
def test_fused_sparse_update_flow_matches_the_reference_cpu_runtime(kind):
    from sige_b200.workloads.ddpm import DDPMConfig

    cfg = DDPMConfig.small()
    fused_outs, fused_caches, steps = _fused_flow(kind, cfg)
    ref_outs, ref_caches = _eager_flow(kind, cfg)
    st = steps[0]
    kinds = [k for k, _ in st.low.epilogue]
    n_sc = sum(1 for f in st.fused if f.spec.shortcut is not None and f.spec.dst is not None and f.spec.dst.cached_init is not None)
    assert n_sc > 0 and kinds.count("writeback") == 1
    # the shortcuts fused into a sparse block's conv2, and the launches whose cached destination exists only as views, run again in the epilogue
    assert sum(1 for f in st.low.epilogue_fused if f.name.endswith(".shortcut")) == n_sc
    assert any(f.name.endswith(".raw") for f in st.low.epilogue_fused)
    assert len(fused_outs) == len(ref_outs) == 2 * len(STEPS)
    for i, (a, b) in enumerate(zip(fused_outs, ref_outs)):
        err = float((a - b).abs().max() / b.abs().max())
        assert err <= 2e-5, "output %d: %g" % (i, err)
    assert [n for n, _ in fused_caches] == [n for n, _ in ref_caches] and len(fused_caches) > 3 * 10
    for (n, a), (_, b) in zip(fused_caches, ref_caches):
        err = float((a - b).abs().max() / max(1.0, float(b.abs().max())))
        assert err <= 2e-5, "cache %s: %g" % (n, err)


def test_plain_simulator_declines_and_lowers_as_before():
    """An executor without the write-back predicate gets the same main program; the step says why it cannot apply edits."""
    from sige.utils import downsample_mask
    from sige_b200.fused import FusedStep
    from sige_b200.workloads.ddpm import DDPMConfig
    from sim_executor import SimExecutor

    cfg = DDPMConfig.small()
    x0, t, edits = _edits(cfg)
    progs = []
    with torch.no_grad():
        model = _model("intree", cfg)
        _dense(model, x0, t)
        model.set_cache_id(1)
        model.set_masks(downsample_mask(edits[0][1], min_res=8))
        for ex, writes_back in ((SimExecutor(), False), (_writeback_sim(), True)):
            st = FusedStep(model, edits[0][0] * 1.1, t + 10, executor=ex)
            progs.append(([k for k, _ in st.steps], [(f.name, f.spec.N, f.spec.off, f.spec.Cin, f.spec.Cout) for f in st.fused], st.launches_per_step,
                          st.output.clone()))
            if writes_back:
                assert st.sparse_update_supported
            else:
                assert not st.sparse_update_supported and "write-back" in st.sparse_update_reason and st.low.epilogue == []
                with pytest.raises(RuntimeError, match="cannot write back"):
                    st.sparse_update()
    assert progs[0][:3] == progs[1][:3]
    assert torch.equal(progs[0][3], progs[1][3])


def test_step_declines_a_cache_it_cannot_take_exactly():
    """A bf16 cache under an fp32 step would round: the step declines with the reason, and the main program is unaffected."""
    from sige.utils import downsample_mask
    from sige_b200.fused import FusedStep
    from sige_b200.workloads.ddpm import DDPMConfig

    cfg = DDPMConfig.small()
    x0, t, edits = _edits(cfg)
    with torch.no_grad():
        model = _model("intree", cfg)
        _dense(model, x0, t)
        model.set_cache_id(0)
        model.set_masks(downsample_mask(edits[0][1], min_res=8))
        mods = [m for m in model.modules() if hasattr(m, "original_outputs")]
        mods[3].original_outputs[0] = mods[3].original_outputs[0].to(torch.bfloat16)
        st = FusedStep(model, edits[0][0], t, executor=_writeback_sim())
    assert not st.sparse_update_supported and "exactly" in st.sparse_update_reason
