"""A compiled step of a batch of independent edits takes the next batch in place: per-edit fixed-capacity tile lists
(`IdxSlot` with `tile_images`), rewritten by `FusedStep.rebind` — checked on the descriptor simulator with the in-tree DDPM
miniature and E = 4 edits."""
import os
import sys
import warnings

import torch

from conftest import REPO

sys.path.insert(0, os.path.join(REPO, "tests"))

E = 4


def _model():
    from sige_b200.workloads.ddpm import DDPMConfig, SIGEDDPMUNet, init_deterministic, synthetic_inputs

    cfg = DDPMConfig.small()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model = init_deterministic(SIGEDDPMUNet(cfg), seed=0).eval()
    x0, _, _, t = synthetic_inputs(cfg, 0.05, seed=0)
    with torch.no_grad():
        model.set_mode("full")
        model(x0, t)
        model.set_mode("sparse")
    return model, cfg, x0, t


def _batch(cfg, x0, plan):
    """plan: (ratio, shift) per edit -> (inputs [E, ...], mask pyramids {res: [E, H, W]})."""
    from sige.utils import downsample_mask
    from sige_b200.masks import stack_mask_pyramids
    from sige_b200.workloads.ddpm import synthetic_inputs

    xs, pyramids = [], []
    for e, (ratio, shift) in enumerate(plan):
        _, x1, mask, _ = synthetic_inputs(cfg, ratio, seed=0, edit_seed=e)
        xs.append(x0 + torch.roll(x1 - x0, shift, (2, 3)))
        pyramids.append(downsample_mask(torch.roll(mask, shift, (0, 1)), min_res=8))
    return torch.cat(xs, 0), stack_mask_pyramids(pyramids)


A = [(0.05, (0, 0)), (0.03, (-14, 9)), (0.08, (11, -13)), (0.02, (6, 6))]
B = [(0.04, (9, -11)), (0.06, (-7, 3)), (0.03, (2, 14)), (0.05, (-12, -12))]


def _batch_sim():
    """The descriptor simulator, taught to read a batch's per-edit fixed-capacity lists: a batched launch runs on the real rows of
    its lists (a SIGE_TILE_NONE row reads zeros and writes nothing, include/sige_b200.h), read when the launch runs."""
    import copy
    from types import SimpleNamespace

    from sige_b200._cabi import TILE_NONE
    from sim_executor import SimExecutor

    class BatchSlotSim(SimExecutor):
        def batch_slots_supported(self):
            return True

        def prepare_conv(self, fc):
            s = fc.spec
            if s.tile_img is None:
                return super().prepare_conv(fc)
            inner = SimpleNamespace(spec=copy.copy(s))
            super().prepare_conv(inner)

            def run(stream):
                real = s.idx[:, 0] > TILE_NONE
                v = inner.spec
                v.idx, v.tile_img, v.N = s.idx[real], s.tile_img[real], int(real.sum())
                if s.shortcut is not None:
                    v.shortcut = tuple(s.shortcut[:3]) + (s.shortcut[3][real],)
                inner.launch_fn(stream)

            fc.launch_fn = run

    return BatchSlotSim()


def _step(model, x, t, executor=None, **opts):
    from sige_b200.fused import FusedStep

    with torch.no_grad():
        return FusedStep(model, x, t, executor=executor or _batch_sim(), **opts)


def _batched(step):
    return [f for f in step.fused if f.spec.tile_img is not None]


def _per_image_layout(g, cap):
    """The per-image layout of a Gather's concatenated lists, restated: row e*cap + i = tile i of edit e, SIGE_TILE_NONE behind."""
    from sige_b200._cabi import TILE_NONE

    rows = torch.full((E * cap, 2), TILE_NONE, dtype=torch.int32)
    img = g.tile_images.long()
    for e in range(E):
        sel = g.active_indices[img == e]
        rows[e * cap:e * cap + sel.shape[0]] = sel
    return rows


def test_batched_step_with_headroom_reads_slot_buffers_and_takes_the_next_batch_in_place():
    model, cfg, x0, t = _model()
    xa, ma = _batch(cfg, x0, A)
    model.set_masks(ma)
    step = _step(model, xa, t, headroom=0.5)
    batched = _batched(step)
    assert len(batched) > 10 and step.eager_nodes == []
    for f in batched:
        s, sl = f.spec, f.spec.slot
        assert sl is not None and s.idx is sl.buf and sl.E == E and sl.padded, s.name
        counts = torch.bincount(sl.gather.tile_images.long(), minlength=E)
        assert sl.cap % 8 == 0 and sl.cap >= int(counts.max()) * 1.5 and s.N == E * sl.cap, s.name
        assert torch.equal(s.tile_img, torch.arange(E * sl.cap, dtype=torch.int32) // sl.cap), s.name
        assert torch.equal(sl.buf, _per_image_layout(sl.gather, sl.cap)), s.name
        if s.shortcut is not None:
            assert s.shortcut[3].shape == (E * sl.cap,)
    assert any(f.spec.shortcut is not None for f in batched), "the DDPM step fuses its 1x1 shortcuts"
    stem = step.low.conv_ins[0]
    assert stem.tiles is not None and any(stem.tiles is sl.buf for sl in step.low.slots.values())

    # batch B: other places and sizes, every per-edit list within the capacities of batch A
    xb, mb = _batch(cfg, x0, B)
    model.set_masks(mb)
    with torch.no_grad():
        assert step.rebind(), "batch B fits: installed in place"
        for f in batched:
            assert torch.equal(f.spec.slot.buf, _per_image_layout(f.spec.slot.gather, f.spec.slot.cap)), f.spec.name
        out_b = step(xb, t).clone()
    fresh = _step(model, xb, t).output
    assert torch.allclose(out_b, fresh, atol=2e-5), float((out_b - fresh).abs().max())

    # one edit with no change at all: its lists are empty at every resolution
    empty = {res: m.clone() for res, m in mb.items()}
    for m in empty.values():
        m[2] = False
    model.set_masks(empty)
    with torch.no_grad():
        assert step.rebind(), "an edit with empty lists installs"
        out_e = step(xb, t).clone()
    fresh = _step(model, xb, t).output
    assert torch.allclose(out_e, fresh, atol=2e-5), float((out_e - fresh).abs().max())

    # too many tiles for one edit: recompile
    xc, mc = _batch(cfg, x0, [(0.05, (0, 0)), (0.30, (0, 0)), (0.03, (2, 14)), (0.05, (-12, -12))])
    model.set_masks(mc)
    assert not step.rebind()

    # another number of edits: recompile
    xd, md = _batch(cfg, x0, B[:3])
    model.set_masks(md)
    assert not step.rebind()


def test_batched_step_without_headroom_has_the_per_image_lists_of_the_longest_edit():
    """headroom 0: every batched launch's list length per edit is the longest edit's count, the per-image layout is the one the
    launches always had (padded with SIGE_TILE_NONE), and no launch claims whole CTAs of padding."""
    model, cfg, x0, t = _model()
    xa, ma = _batch(cfg, x0, A)
    model.set_masks(ma)
    step = _step(model, xa, t)
    wide = _step(model, xa, t, headroom=0.5)
    assert [f.name for f in step.fused] == [f.name for f in wide.fused]
    assert torch.allclose(step.output, wide.output, atol=2e-5)
    # an executor that does not read per-edit fixed-capacity lists gets the concatenated lists with a per-row image index: the same
    # launches, which the per-image layout gives the same rows (the longest edit's count per edit, SIGE_TILE_NONE behind)
    from sim_executor import SimExecutor

    plain = _step(model, xa, t, executor=SimExecutor())
    assert not plain.low.slots and [f.name for f in plain.fused] == [f.name for f in step.fused]
    assert torch.allclose(step.output, plain.output, atol=2e-5)
    batched = _batched(step)
    assert len(batched) > 10
    for f, p in zip(step.fused, plain.fused):
        assert (f.spec.tile_img is None) == (p.spec.tile_img is None), f.name
        if f.spec.tile_img is None:
            continue
        sl = f.spec.slot
        counts = torch.bincount(p.spec.tile_img.long(), minlength=E)
        assert sl.cap == int(counts.max()) and f.spec.N == E * sl.cap and not sl.padded, f.name
        assert torch.equal(sl.buf, _per_image_layout(sl.gather, sl.cap)), f.name
        shortcut = f.spec.shortcut
        if shortcut is not None:              # the shortcut flags of the concatenated rows, at their rows of the per-image layout
            rows = p.spec.tile_img.long() * sl.cap + torch.cat([torch.arange(int(c)) for c in counts])
            want = torch.zeros(E * sl.cap, dtype=torch.uint8)
            want[rows] = p.spec.shortcut[3]
            assert torch.equal(shortcut[3], want), f.name
    # an executor without the per-edit lists recompiles for a new batch, as before
    with torch.no_grad():
        assert not plain.rebind()
    # a later batch whose lists are no longer than these installs in place as well
    model.set_masks(ma)
    with torch.no_grad():
        assert step.rebind()
        assert torch.allclose(step(xa, t), wide.output, atol=2e-5)
