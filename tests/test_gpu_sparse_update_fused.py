"""sparse_update on the fused path, on the GPU: `sige_tile_writeback` against a torch restatement, and the reference's apply
flow (a cache per sampler step; each edit previewed, then applied with `sparse_update=True`; a second edit on top of the first)
through the public model call, against the reference's CPU runtime running the eager operator modules."""
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
STEPS = [0, 1, 2]
TOL_MAX = 5e-3            # tests/test_gpu_fused.py: fp16 step vs the reference, max-normalised
# caches after two applied edits, max-normalised per cache (fp16 step of an fp32 model vs the reference's fp32 CPU runtime): measured
# 1.9e-3 at worst on an H100; the bound is about twice that
TOL_CACHE = 4e-3


@pytest.fixture(autouse=True)
def _exact_fp32_dense_pass():
    saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


# ---------------------------------------------------------------------------------------------------------------------
# the kernel
# ---------------------------------------------------------------------------------------------------------------------
GUARD = 64          # elements of random guard band on both sides of every destination (a multiple of 16 bytes)


def _guarded(shape, dtype, nhwc, gen):
    B, C, H, W = shape
    n = B * C * H * W
    base = torch.randn(n + 2 * GUARD, generator=gen).to(dtype).to(DEV)
    inner = base[GUARD:GUARD + n]
    t = inner.view(B, H, W, C).permute(0, 3, 1, 2) if nhwc else inner.view(B, C, H, W)
    return base, t


def _tiles(n, H, W, gen, pad):
    """n tile origins from one grid step beyond the top-left corner to beyond the bottom-right one, plus `pad` SIGE_TILE_NONE rows."""
    from sige_b200._cabi import TILE_NONE

    ih = torch.randint(-6, H + 2, (n,), generator=gen)
    iw = torch.randint(-6, W + 2, (n,), generator=gen)
    idx = torch.stack([ih, iw], 1)
    idx[0] = torch.tensor([-6, -6])                     # wholly outside: writes nothing
    idx[1 % n] = torch.tensor([H - 2, W - 3])           # past the bottom-right border: clipped
    idx = torch.cat([idx, torch.full((pad, 2), TILE_NONE)], 0)
    return idx.to(torch.int32).to(DEV)


def _bits(t):
    return t.view({4: torch.int32, 2: torch.int16}[t.element_size()]).cpu()


def _case(B, nhwc, dst_dtype, src_dtype, seed):
    """Entries over C = 8, 72, 128, 512 with 4x4 tiles (offset 1, stride 1) and 2x2 tiles (offset 0, stride 2, origins in the
    stride-2 conv's input frame); padded lists, one of them padding only, and an empty one."""
    gen = torch.Generator().manual_seed(seed)
    entries, bases = [], []
    #        C,   H,  W, off, stride, tile, tiles, padding
    geoms = [(8, 12, 20, 1, 1, 4, 5, 3), (72, 16, 16, 1, 1, 4, 9, 0), (128, 10, 14, 0, 2, 2, 7, 3), (512, 8, 8, 1, 1, 4, 6, 2),
             (72, 9, 13, 0, 2, 2, 0, 8), (8, 8, 8, 1, 1, 4, 0, 0)]
    for (C, H, W, off, stride, ro, n, pad) in geoms:
        src = torch.randn(B, C, H, W, generator=gen).to(src_dtype).to(DEV).contiguous(memory_format=torch.channels_last)
        base, dst = _guarded((B, C, H, W), dst_dtype or src_dtype, nhwc, gen)
        idx = _tiles(max(n, 2), H * stride, W * stride, gen, pad)
        idx = idx if n else idx[2:]
        entries.append((src, dst, idx, off, stride, ro))
        bases.append(base)
    return entries, bases


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("src_dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("dst_dtype", [torch.float32, None])
@pytest.mark.parametrize("nhwc", [False, True])
def test_tile_writeback_matches_torch_restatement(nhwc, dst_dtype, src_dtype, B):
    """Written elements are exactly the converted source; every other element of the guard-banded destinations, and every
    source, is bitwise unchanged; a graph replay writes what the eager launch wrote."""
    from sige_b200 import ops
    from test_sparse_update_fused import torch_writeback

    entries, bases = _case(B, nhwc, dst_dtype, src_dtype, seed=B * 7 + nhwc)
    initial = [b.clone() for b in bases]
    src_before = [_bits(e[0]) for e in entries]
    want = [b.clone().cpu() for b in bases]
    want_entries = []
    for (src, dst, idx, off, stride, ro), w in zip(entries, want):
        Bb, C, H, W = dst.shape
        inner = w[GUARD:GUARD + dst.numel()]
        wd = inner.view(Bb, H, W, C).permute(0, 3, 1, 2) if nhwc else inner.view(Bb, C, H, W)
        want_entries.append((src.cpu(), wd, idx.cpu(), off, stride, ro))
    torch_writeback(want_entries)
    assert any(not torch.equal(_bits(w), _bits(b)) for w, b in zip(want, initial))
    run = ops.tile_writeback_launcher(entries)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):                # (capture runs nothing)
        run(torch.cuda.current_stream().cuda_stream)
    run(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for k, (b, w) in enumerate(zip(bases, want)):
        assert torch.equal(_bits(b), _bits(w)), "entry %d (eager launch)" % k
    for (src, *_), s0 in zip(entries, src_before):
        assert torch.equal(_bits(src), s0)
    for b, b0 in zip(bases, initial):
        b.copy_(b0)
    g.replay()
    torch.cuda.synchronize()
    for k, (b, w) in enumerate(zip(bases, want)):
        assert torch.equal(_bits(b), _bits(w)), "entry %d (graph replay)" % k


def test_tile_writeback_splits_more_entries_than_one_launch_takes():
    from sige_b200 import _cabi, ops
    from test_sparse_update_fused import torch_writeback

    gen = torch.Generator().manual_seed(3)
    n = _cabi.WRITEBACK_MAX_ENTRIES + 9
    entries, want = [], []
    for k in range(n):
        src = torch.randn(1, 16, 8, 8, generator=gen).half().to(DEV).contiguous(memory_format=torch.channels_last)
        dst = torch.randn(1, 16, 8, 8, generator=gen).to(DEV)
        idx = _tiles(3, 8, 8, gen, pad=1)
        entries.append((src, dst, idx, 1, 1, 4))
        want.append((src, dst.clone(), idx.cpu(), 1, 1, 4))
    before = ops.launch_count
    ops.tile_writeback(entries)
    assert ops.launch_count - before == 2
    torch_writeback(want)
    for (_, d, _, _, _, _), (_, w, _, _, _, _) in zip(entries, want):
        assert torch.equal(d, w)


# ---------------------------------------------------------------------------------------------------------------------
# the apply flow
# ---------------------------------------------------------------------------------------------------------------------
def _model(cfg):
    from sige_b200.workloads.ddpm import SIGEDDPMUNet, init_deterministic

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return init_deterministic(SIGEDDPMUNet(cfg), seed=0).eval()


def _edits(cfg):
    from sige_b200.workloads.ddpm import synthetic_inputs

    x0, xa, mask_a, t = synthetic_inputs(cfg, 0.05, seed=0, edit_seed=1)
    _, xb, mask_b, _ = synthetic_inputs(cfg, 0.10, seed=0, edit_seed=2)
    xb = xa + (xb - x0)
    return x0, t, ((xa, mask_a), (xb, mask_a | mask_b))


def _dense(model, x0, t, dev, steps=STEPS):
    model.set_mode("full")
    for s in steps:
        model.set_cache_id(s)
        model((x0 * (1.0 + 0.1 * s)).to(dev), (t + 10 * s).to(dev))
    model.set_mode("sparse")


def _caches(model):
    from sige_b200.parallel import cache_tensors

    return [(n, v) for n, v in cache_tensors(model)]


def _written(step, masks):
    """Accumulate, per module cache (by address), the union of the output tiles the step's write-back covers."""
    from sige_b200._cabi import TILE_NONE

    for (buf, slot, off, stride, ro) in step.low.cache_writers:
        c = buf.cached_init
        m = masks.setdefault(c.data_ptr(), torch.zeros(c.shape[2:], dtype=torch.bool))
        for ih, iw in slot.buf.tolist():
            if ih == TILE_NONE:
                continue
            y, x = int((off + ih) / stride), int((off + iw) / stride)
            m[max(y, 0):max(y + ro, 0), max(x, 0):max(x + ro, 0)] = True


@pytest.fixture(scope="module")
def flows():
    """The fused flow (each edit previewed, then applied) and the reference CPU runtime's eager flow."""
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import downsample_mask
    from sige_b200.workloads.ddpm import DDPMConfig

    cfg = DDPMConfig.small()
    x0, t, edits = _edits(cfg)
    model = _model(cfg).to(DEV)
    res = {"outs": [], "steps": [], "masks": {}}
    with torch.no_grad():
        _dense(model, x0, t, DEV)
        res["dense"] = {n: v.detach().clone() for n, v in _caches(model)}
        model.set_fused(True, dtype=torch.float16)
        for x_edit, mask in edits:
            model.set_masks(downsample_mask(mask.to(DEV), min_res=8))
            for s in STEPS:
                model.set_cache_id(s)
                args = ((x_edit * (1.0 + 0.1 * s)).to(DEV), (t + 10 * s).to(DEV))
                model.set_sparse_update(False)
                before = {n: v.clone() for n, v in _caches(model)}
                model(*args)                                                 # preview
                preview_step = model.fused_step
                assert all(torch.equal(v, before[n]) for n, v in _caches(model)), "a preview wrote a cache"
                model.set_sparse_update(True)
                res["outs"].append(model(*args).float().cpu())               # apply
                assert model.fused_step is preview_step and preview_step.eager_nodes == []
                assert preview_step.sparse_update_supported, preview_step.sparse_update_reason
                res["steps"].append(preview_step)
                _written(preview_step, res["masks"])
        res["caches"] = {n: v.detach().float().cpu() for n, v in _caches(model)}
        res["addr"] = {n: v.data_ptr() for n, v in _caches(model)}
    res["model"], res["args"] = model, args
    with reference_cpu_runtime(), torch.no_grad():
        cpu = _model(cfg)
        _dense(cpu, x0, t, "cpu")
        cpu.set_sparse_update(True)
        ref_outs = []
        for x_edit, mask in edits:
            cpu.set_masks(downsample_mask(mask, min_res=8))
            for s in STEPS:
                cpu.set_cache_id(s)
                ref_outs.append(cpu(x_edit * (1.0 + 0.1 * s), t + 10 * s).clone())
        res["ref_outs"], res["ref_caches"] = ref_outs, {n: v.detach().float().clone() for n, v in _caches(cpu)}
    return res


def test_apply_flow_matches_the_reference_cpu_runtime(flows):
    assert len(flows["outs"]) == len(flows["ref_outs"]) == 2 * len(STEPS)
    for i, (a, b) in enumerate(zip(flows["outs"], flows["ref_outs"])):
        err = float((a - b).abs().max() / b.abs().max())
        assert err <= TOL_MAX, "output %d: %g" % (i, err)
    worst = 0.0
    assert sorted(flows["caches"]) == sorted(flows["ref_caches"]) and len(flows["caches"]) > 3 * 10
    for n, a in flows["caches"].items():
        b = flows["ref_caches"][n]
        err = float((a - b).abs().max() / max(float(b.abs().max()), 1e-12))
        worst = max(worst, err)
        assert err <= TOL_CACHE, "cache %s: %g" % (n, err)
    print("worst cache error, max-normalised: %.3g" % worst)


def test_apply_writes_only_the_output_tiles(flows):
    changed_any = 0
    for n, after in flows["caches"].items():
        dense = flows["dense"][n].float().cpu()
        m = flows["masks"].get(flows["addr"][n])
        diff = after != dense
        if m is None:
            assert not bool(diff.any()), "cache %s changed without a writer" % n
            continue
        changed_any += int(diff.any())
        outside = diff & ~m.view(1, 1, *m.shape)
        assert not bool(outside.any()), "cache %s: %d elements outside the written tiles changed" % (n, int(outside.sum()))
    assert changed_any > 10


def test_apply_is_idempotent_and_a_plain_call_writes_nothing(flows):
    model, args = flows["model"], flows["args"]
    with torch.no_grad():
        model.set_sparse_update(True)
        first = model(*args)
        caches = {n: v.clone() for n, v in _caches(model)}
        again = model(*args)
        assert torch.equal(first, again)
        assert all(torch.equal(v, caches[n]) for n, v in _caches(model))
        model.set_sparse_update(False)
        model(*args)
        assert all(torch.equal(v, caches[n]) for n, v in _caches(model))


def test_main_program_is_the_one_a_model_without_the_flag_compiles(flows):
    from sige.utils import downsample_mask
    from sige_b200.workloads.ddpm import DDPMConfig

    cfg = DDPMConfig.small()
    x0, t, edits = _edits(cfg)
    steps = {}
    for used in (False, True):
        model = _model(cfg).to(DEV)
        with torch.no_grad():
            _dense(model, x0, t, DEV, steps=[0])
            model.set_fused(True, dtype=torch.float16)
            model.set_masks(downsample_mask(edits[0][1].to(DEV), min_res=8))
            model.set_sparse_update(used)
            model(edits[0][0].to(DEV), t.to(DEV))
        st = model.fused_step
        steps[used] = ([k for k, _ in st.steps], [(f.name, f.spec.N, f.spec.off, f.spec.k, f.spec.Cin, f.spec.Cout, len(f.spec.aux), f.spec.dst is not None and f.spec.dst.has_raw)
                                                    for f in st.fused], st.launches_per_step)
    assert steps[False][0] == steps[True][0] and steps[False][2] == steps[True][2]
    # (the epilogue gives raw buffers to destinations the main program writes only as views: compare all but that)
    assert [f[:7] for f in steps[False][1]] == [f[:7] for f in steps[True][1]]


def test_eager_modules_continue_from_the_applied_caches(flows):
    """After the fused applies, the next edit through the eager operator modules agrees with the fused preview of it."""
    from sige.utils import downsample_mask
    from sige_b200.workloads.ddpm import DDPMConfig, synthetic_inputs

    model, (_, t) = flows["model"], flows["args"]
    _, x_c, mask_c, _ = synthetic_inputs(DDPMConfig.small(), 0.08, seed=0, edit_seed=5)
    with torch.no_grad():
        model.set_sparse_update(False)
        model.set_masks(downsample_mask(mask_c.to(DEV), min_res=8))
        x_c = (x_c * (1.0 + 0.1 * STEPS[-1])).to(DEV)
        model.set_fused(True, dtype=torch.float16)
        fused = model(x_c, t).float()
        model.set_fused(False)
        eager = model(x_c, t).float()
        model.set_fused(True, dtype=torch.float16)
    err = float((fused - eager).abs().max() / eager.abs().max())
    assert err <= TOL_MAX, err


def test_next_edit_applied_without_a_host_sync():
    """The second edit installed by `set_masks_async` and applied under sync debugging gives bitwise what `set_masks` gives."""
    from sige.utils import downsample_mask
    from sige_b200.workloads.ddpm import DDPMConfig

    cfg = DDPMConfig.small()
    x0, t, edits = _edits(cfg)
    (xa, mask_a), (xb, mask_b) = edits
    results = []
    for use_async in (True, False):
        model = _model(cfg).to(DEV)
        with torch.no_grad():
            _dense(model, x0, t, DEV, steps=[0])
            model.set_cache_id(0)
            model.set_fused(True, dtype=torch.float16, headroom=2.0)
            model.set_sparse_update(True)
            model.set_masks(downsample_mask(mask_a.to(DEV), min_res=8))
            model(xa.to(DEV), t.to(DEV))
            step = model.fused_step
            pyr = downsample_mask(mask_b.to(DEV), min_res=8)
            xb_d, t_d = xb.to(DEV), t.to(DEV)
            torch.cuda.synchronize()
            if use_async:
                torch.cuda.set_sync_debug_mode("error")
                try:
                    assert model.set_masks_async(pyr) is True
                    out = model(xb_d, t_d)
                finally:
                    torch.cuda.set_sync_debug_mode("default")
                assert model.fused_step is step and model.masks_async_ok()
            else:
                model.set_masks(pyr)
                out = model(xb_d, t_d)
            results.append((out.clone(), {n: v.clone() for n, v in _caches(model)}))
    (oa, ca), (ob, cb) = results
    assert torch.equal(oa, ob)
    assert sorted(ca) == sorted(cb) and all(torch.equal(ca[n], cb[n]) for n in ca)
