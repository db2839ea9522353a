"""A batch of independent label edits through one fused GauGAN step (both generators), on the descriptor simulator.

The SPADE launches of a batch — the separable gamma / beta convs of the sub-mobile generator, the windowed `mlp_gamma_beta` conv of the
full SPADE and the modulated convs that read gamma / beta — read the per-edit fixed-capacity lists of the batch's `IdxSlot`s over
operands of E images (SIGE_CONV_PER_IMAGE_OPERANDS).  Checked here: the batched step has the launches of the single-edit step, all
on per-edit lists, and no eager operator-module node; each edit of its output equals that edit's own step; a second batch that fits
goes in by `rebind` and equals a fresh compile; an executor without the per-image operands still refuses the batch.  The C-ABI's
refusals of the new flag are checked without a device."""
import copy
import ctypes
import os
import sys
import types
from collections import Counter

import pytest
import torch
from torch.nn import functional as F

from conftest import REPO

sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "baseline"))

import consumers  # noqa: E402

E = 3


def _sims():
    """(BatchSim, NoPerImageSim): the simulator of test_spade_generator.py (separable, narrow, modulated and strided launches) taught
    to read a batch's per-edit lists, with and without the per-image operands of the SPADE launches."""
    import test_spade_generator as TSG

    from sige_b200._cabi import TILE_NONE

    StridedSim, _ = TSG._sims()

    class NoPerImageSim(StridedSim):
        def batch_slots_supported(self):
            return True

        def prepare_conv(self, fc):
            """A batched launch: the real rows of its per-edit lists (a SIGE_TILE_NONE row reads zeros and writes nothing), read when
            the launch runs; a modulated one on leaky((x*scale + shift) * (1 + gamma) + beta) of every image at its logical extent."""
            s = fc.spec
            if s.tile_img is None:
                return super().prepare_conv(fc)
            assert s.slot is not None and s.idx is s.slot.buf and s.N == s.slot.E * s.slot.cap, s.name
            inner = copy.copy(s)
            z = None
            if s.modulation is not None:
                gamma, beta, slope = s.modulation
                assert len(s.srcs) == 1 and s.act == "identity" and s.shortcut is None
                z = torch.empty(tuple(gamma.shape), dtype=torch.float32)
                inner.srcs, inner.scale, inner.shift, inner.modulation = [(z, 0)], None, None, None
            shim = types.SimpleNamespace(spec=inner, launch_fn=None)
            super().prepare_conv(shim)

            def run(stream):
                if z is not None:
                    x, up = s.srcs[0]
                    a = F.interpolate(x.float(), scale_factor=2.0, mode="nearest") if up else x.float()
                    B = a.shape[0]
                    if s.scale is not None:
                        a = a * (s.scale.view(1, -1, 1, 1) if s.scale.dim() == 1 else s.scale.view(B, -1, 1, 1))
                    if s.shift is not None:
                        a = a + (s.shift.view(1, -1, 1, 1) if s.shift.dim() == 1 else s.shift.view(B, -1, 1, 1))
                    m = a * (1 + gamma.float()) + beta.float()
                    z.copy_(torch.where(m > 0, m, m * slope))
                real = s.idx[:, 0] > TILE_NONE
                inner.idx, inner.tile_img, inner.N = s.idx[real], s.tile_img[real], int(real.sum())
                shim.launch_fn(stream)

            fc.launch_fn = run

    class BatchSim(NoPerImageSim):
        def per_image_operands_supported(self):
            return True

        def prepare_separable(self, rec):
            """sige_separable_conv with per-image lists: row m of idx is a tile of image tile_img[m]."""
            if rec.tile_img is None:
                return super().prepare_separable(rec)

            def run(_stream):
                self.launches += 1
                src = rec.src[:, rec.c0:rec.c0 + rec.Cin].float()
                P = 8
                padded = F.pad(src, (P, P, P, P))
                rows = [(int(b), iy, ix) for b, (iy, ix) in zip(rec.tile_img.tolist(), rec.idx.tolist()) if iy > TILE_NONE]
                assert len(rec.idx) == rec.batch * (len(rec.idx) // rec.batch)
                if not rows:
                    return
                X = torch.stack([padded[b, :, iy + P:iy + P + 6, ix + P:ix + P + 6] for b, iy, ix in rows])
                for dw, pw_w, pw_b, dst in rec.branches:
                    y = F.conv2d(X, dw.weight.float(), None if dw.bias is None else dw.bias.float(), groups=X.shape[1])
                    if dw.scale is not None:
                        y = y * dw.scale.view(1, -1, 1, 1)
                    if dw.shift is not None:
                        y = y + dw.shift.view(1, -1, 1, 1)
                    y = F.conv2d(y, pw_w.float(), None if pw_b is None else pw_b.float())
                    out = dst.raw
                    H, W = out.shape[2], out.shape[3]
                    for m, (b, iy, ix) in enumerate(rows):
                        oy, ox = iy + rec.off, ix + rec.off
                        y0, x0, y1, x1 = max(oy, 0), max(ox, 0), min(oy + 4, H), min(ox + 4, W)
                        if y1 > y0 and x1 > x0:
                            out[b, :, y0:y1, x0:x1] = y[m, :, y0 - oy:y1 - oy, x0 - ox:x1 - ox].to(out.dtype)

            return run

    return BatchSim, NoPerImageSim


def _generator(which, size="mini"):
    if which == "gc":
        from sige_b200.workloads import gaugan_gc as G

        return G.build_gaugan_gc(size)
    if which == "spade":
        from sige_b200.workloads import gaugan_spade as GS

        return GS.build_gaugan_spade(size)
    if not consumers.available():
        pytest.skip("baseline/_ref absent (python baseline/build_ref.py)")
    return consumers.build_gaugan(size)


def _pyramid(mask):
    from sige.utils import dilate_mask, downsample_mask

    return downsample_mask(dilate_mask(mask, 1), min_res=(4, 8), dilation=0)


def _batch_masks(masks):
    from sige_b200.masks import stack_mask_pyramids

    return stack_mask_pyramids([_pyramid(m) for m in masks])


def _kinds(step):
    n = Counter(step.eager_nodes)
    return {"separable": [k for k, _ in step.steps].count("separable"), "modulated": sum(1 for f in step.fused if f.spec.modulation is not None),
            "strided": sum(1 for f in step.fused if not f.spec.src_is_stack and not f.spec.srcs[0][0].is_contiguous(memory_format=torch.channels_last)),
            "launches": len(step.fused), "eager": dict(n)}


def _per_image(step):
    """Every launch of the step that reads a tile list of the batch reads its slot's per-edit lists."""
    low = step.low
    batched = [f for f in step.fused if f.spec.tile_img is not None]
    for f in batched:
        sl = f.spec.slot
        assert sl is not None and f.spec.idx is sl.buf and sl.E == E and f.spec.N == E * sl.cap, f.name
    for r in low.separable:
        sl = next(sl for sl in low.slots.values() if sl.buf is r.idx)
        assert r.tile_img is sl.tile_img and sl.E == E and r.batch == E, r.name
    return batched


@pytest.mark.parametrize("which", ["gc", "spade", "reference"])
def test_batch_of_label_edits_runs_as_one_step_and_takes_the_next_batch_in_place(which):
    """E = 3 edits of the scene (the workload's, a smaller one elsewhere, one along the image border) in one compiled step: the
    launches of the single-edit step, each on per-edit lists; every edit's output equals its own single-edit step; a second batch
    that fits is installed by `rebind` into the same step object and equals a fresh compile exactly."""
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige_b200.fused import FusedStep
    from sige_b200.workloads import gaugan_gc as G

    BatchSim, _ = _sims()
    net = _generator(which)
    s0, s1s, masks = G.gaugan_gc_edits("mini", E + 2)
    sizes = [int(m.sum()) for m in masks[:E]]
    assert min(sizes) * 1.8 < max(sizes) and bool(masks[2][:, 0].any())       # one much smaller edit, one on the border
    with reference_cpu_runtime(), torch.no_grad():
        net.set_mode("full")
        net(s0)
        net.set_mode("sparse")
        singles = []
        for e in range(E):
            net.set_masks(_pyramid(masks[e]))
            single = FusedStep(net, s1s[e:e + 1], executor=BatchSim())
            singles.append((single, single.output.clone()))
        net.set_masks(_batch_masks(masks[:E]))
        step = FusedStep(net, s1s[:E], executor=BatchSim(), headroom=0.5)
        out = step.output.clone()

        # batch B: edits 1, 3 and 4 of the scene, each list within the capacities of the first batch
        order = [1, 3, 4]
        net.set_masks(_batch_masks(masks[order]))
        assert step.rebind(), "a batch that fits is installed in place"
        out_b = step(s1s[order]).clone()
        fresh_b = FusedStep(net, s1s[order], executor=BatchSim(), headroom=0.5).output.clone()

    assert not any(n.startswith(("sige.", "gather(")) for n in step.eager_nodes), step.eager_nodes
    one = _kinds(singles[0][0])
    got = _kinds(step)
    assert {k: v for k, v in got.items() if k != "eager"} == {k: v for k, v in one.items() if k != "eager"}
    assert got["eager"] == one["eager"]
    assert got["modulated"] > 0 and (got["separable"] > 0 if which == "gc" else got["strided"] > 0)
    batched = _per_image(step)
    assert {f.name for f in batched} >= {f.name for f in step.fused if f.spec.modulation is not None}
    assert out.shape[0] == E
    for e, (_, want) in enumerate(singles):
        scale = want.abs().max().item()
        assert (out[e:e + 1] - want).abs().max().item() <= 2e-5 * scale, e
    assert torch.equal(out_b, fresh_b)


@pytest.mark.parametrize("which", ["gc", "spade"])
def test_executor_without_per_image_operands_still_refuses_the_batch(which):
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige_b200.fused import FusedStep
    from sige_b200.lazy import TraceUnsupported
    from sige_b200.workloads import gaugan_gc as G

    _, NoPerImageSim = _sims()
    net = _generator(which)
    s0, s1s, masks = G.gaugan_gc_edits("mini", E)
    with reference_cpu_runtime(), torch.no_grad():
        net.set_mode("full")
        net(s0)
        net.set_masks(_batch_masks(masks))
        net.set_mode("sparse")
        with pytest.raises(TraceUnsupported):
            FusedStep(net, s1s, executor=NoPerImageSim())


# ---------------------------------------------------------------------------------------------------------------- C-ABI (CPU)
def test_per_image_operands_flag_refusals_come_before_any_cuda_call(cabi_lib):
    """With the flag clear a window or a modulated source keeps refusing per-image lists ("per-image"); the flag is refused without
    per-image lists or on stacks, for sige_tile_conv and sige_separable_conv.  The descriptors' pointers are not device memory, so a
    descriptor the checks accept is only ever passed with N = 0 (a no-op that returns 0 after the checks)."""
    import test_modulated_tile_conv as TM
    import test_spade_generator as TSG
    from sige_b200 import _cabi

    lib = _cabi.lib()
    PER = _cabi.CONV_PER_IMAGE_OPERANDS
    assert PER == 128 and lib.sige_abi_version() == 3

    def window():
        d = TSG._host_desc()
        d.src_pixel_stride = 384
        return d

    def modulated():
        return TM._host_desc()[0]

    def verdict(d, fn="sige_tile_conv"):
        rc = getattr(lib, fn)(ctypes.byref(d), None)
        return rc, lib.sige_last_error() if rc else b""

    def accepted(d, fn="sige_tile_conv"):
        d.N = 0
        return verdict(d, fn) == (0, b"")

    for make in (window, modulated):
        d = make()
        d.idx_per_image, d.B = 1, 2
        rc, msg = verdict(d)
        assert rc != 0 and b"per-image" in msg and b"SIGE_CONV_PER_IMAGE_OPERANDS" in msg, msg
        d.flags |= PER
        assert accepted(d)
        for change in (lambda d: setattr(d, "idx_per_image", 0), lambda d: setattr(d, "src_is_stack", 1), lambda d: setattr(d, "dst_is_stack", 1)):
            d = make()
            d.idx_per_image, d.B, d.flags = 1, 2, d.flags | PER
            change(d)
            rc, msg = verdict(d)
            assert rc != 0 and b"SIGE_CONV_PER_IMAGE_OPERANDS" in msg, msg
    d = TSG._host_desc()                                      # a plain per-image launch is accepted with the flag too
    d.idx_per_image, d.B, d.flags = 1, 2, d.flags | PER
    assert accepted(d)

    def sep(src_stack=0, dst_stack=0):
        s = _cabi.SeparableConv()
        s.dtype, s.src, s.src_is_stack, s.src_C, s.B, s.H, s.W, s.idx, s.N = _cabi.F16, 0x10000, src_stack, 64, 2, 32, 32, 0x20000, 8
        s.Cin, s.Cout, s.offH, s.offW, s.nbranch, s.flags = 64, 64, 1, 1, 1, PER
        b = s.branch[0]
        b.dw_weight, b.pw_weight, b.dst, b.dst_is_stack, b.dH, b.dW, b.dst_C = 0x30000, 0x40000, 0x50000, dst_stack, 32, 32, 64
        return s

    for kw in ({"src_stack": 1}, {"dst_stack": 1}):
        rc, msg = verdict(sep(**kw), "sige_separable_conv")
        assert rc != 0 and b"SIGE_CONV_PER_IMAGE_OPERANDS" in msg, msg
    assert accepted(sep(), "sige_separable_conv")
