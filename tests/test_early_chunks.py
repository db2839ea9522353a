"""Early source groups (sige_tile_conv_t.early), checked without a GPU: which launches of a DDPM-256 step the lowering marks,
and the K partition the wgmma kernel's host plan derives from a mask (sige_tile_conv_plan)."""
import ctypes
import os
import sys

import pytest
import torch

from conftest import REPO, golden

sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "baseline"))

SHORTCUT_CONV2 = ["down.2.block.0.scatter", "n76.conv3x3", "n194.conv3x3", "n207.conv3x3", "n220.conv3x3", "n237.conv3x3",
                  "n266.conv3x3", "n295.conv3x3", "n328.conv3x3", "n341.conv3x3", "n354.conv3x3"] + \
                 ["up.%d.block.%d.scatter" % (u, b) for u in (2, 1, 0) for b in (0, 1, 2)]
SKIP_CONV1 = ["n189.conv3x3", "n202.conv3x3", "n215.conv3x3", "n232.conv3x3", "n261.conv3x3", "n290.conv3x3", "n323.conv3x3",
              "n336.conv3x3", "n349.conv3x3"] + ["up.%d.block.%d.scatter_gather" % (u, b) for u in (2, 1, 0) for b in (0, 1, 2)]


def _ddpm256(**opts):
    from test_fused_cpu import _prepared

    import fused_step_contract as fsc
    import pdl_hazards as ph
    from sige_b200.fused import FusedStep
    from sige_b200.workloads.ddpm import DDPMConfig
    from sim_executor import SimExecutor

    G = golden("ddpm256_golden.npz")
    model, x1, t = _prepared("intree", DDPMConfig(), float(G["ratio"][0]))
    with torch.no_grad():
        return model, FusedStep(model, x1, t, executor=fsc.recording(ph.planned(SimExecutor))(), **opts)


def test_ddpm256_step_marks_the_shortcut_and_skip_launches(cabi_lib):
    """Exactly the 20 fused-shortcut conv2s (bit 2) and the 18 up-path conv1s on cat([h, skip]) (bit 1) get a mask, each after a
    wgmma tile conv; their predecessors, and only those, release early; and no launch of the step reads, before its wait, a line
    that a launch possibly running beside it writes (tests/pdl_hazards.py)."""
    import pdl_hazards as ph

    model, step = _ddpm256()
    assert len(step.fused) == 86
    marked = {f.name: f.spec.early for f in step.fused if f.spec.early}
    assert marked == {**{n: 4 for n in SHORTCUT_CONV2}, **{n: 2 for n in SKIP_CONV1}}
    kinds = [k for k, _ in step.steps]
    es = {e.pos: e for e in ph.entries(step)}
    for f in step.fused:
        if f.spec.early:
            assert kinds[f.pos - 1] == "conv" and es[f.pos - 1].kernel == "wgmma", "%s follows a %s" % (f.name, es[f.pos - 1].kernel)
    assert {f.pos for f in step.fused if f.spec.early_release} == {f.pos - 1 for f in step.fused if f.spec.early}
    st = ph.verify(step, "ddpm256", model)["main then main"]
    assert st.early == 2 * 38
    # without programmatic dependent launch there is nothing to overlap
    _, plain = _ddpm256(pdl=False)
    assert not any(f.spec.early or f.spec.early_release for f in plain.fused)
    assert not any(e.pdl for e in ph.entries(plain) if e.kernel in ("wgmma", "mma.sync"))


def test_early_marks_that_ignore_what_the_predecessor_writes_are_rejected_by_name(cabi_lib, monkeypatch):
    """`_early_masks` marking every group, `written` or not: each skip conv1 then reads h, which its predecessor writes, before
    its wait."""
    import pdl_hazards as ph
    from sige_b200.fused import Lowering

    def every_group(self):
        self._conv_at = {fc.pos: fc for fc in self.fused}
        for fc in self.fused:
            s, prev = fc.spec, self._conv_at.get(fc.pos - 1)
            if s.pdl and s.tc5 and prev is not None and prev.spec.pdl and prev.spec.tc5:
                s.early = sum(1 << g for g, views in enumerate(ph.early_groups(s)) if views)
                prev.spec.early_release = bool(s.early)

    monkeypatch.setattr(Lowering, "_early_masks", every_group)
    model, step = _ddpm256()
    seq = ph.entries(step)
    found = ph.hazards(seq, ph.storage_names(step, model))
    for name in SKIP_CONV1:
        assert any(h.startswith("main launch") and "(%s, wgmma) reads early group 0 src0 before its wait" % name in h for h in found), name
    with pytest.raises(AssertionError, match=r"PDL hazards; the first: main launch \d+ \(.*, wgmma\) reads early group \d"):
        ph.check(seq)


def _desc(cin, cout, n_tiles, *, srcs=None, cin2=0, early=0, ksplit=0, res=64):
    from sige_b200 import _cabi

    d = _cabi.TileConv()
    d.dtype = _cabi.F16
    d.B, d.H, d.W = 1, res, res
    srcs = srcs or (cin,)
    d.n_src = len(srcs)
    for i, c in enumerate(srcs):
        d.src[i].C = c
    d.N, d.R, d.S = n_tiles, 6, 6
    d.Cin, d.Cout, d.kH, d.kW, d.stride = cin, cout, 3, 3, 1
    d.dH, d.dW, d.dC = res, res, cout
    d.ksplit, d.flags = ksplit, _cabi.CONV_PDL | _cabi.CONV_TC5 | (early << 4)
    if cin2:
        d.n_src2, d.Cin2 = 1, cin2
        d.src2[0].C = cin2
    return d


def _plan(d):
    from sige_b200 import _cabi

    p = _cabi.TileConvPlan()
    assert _cabi.lib().sige_tile_conv_plan(ctypes.byref(d), ctypes.byref(p)) == 0
    return p


def slices(cin, c0, cin2, early, ks):
    """Restatement of the K partition of a narrow 3x3 launch: the ring steps of each group (src[0], src[1], shortcut) in the natural
    order, a step = (chunk, kind); early groups first; rank r takes floor(n r / ks) .. floor(n (r+1) / ks) of the early steps,
    then the same share of the late ones."""
    steps = [[("m", j // 3) for j in range(c0 // 64 * 3)], [("m", j // 3) for j in range(c0 // 64 * 3, cin // 64 * 3)],
             [("s", c) for c in range(cin2 // 64)]]
    e = [s for g in range(3) if (early >> g) & 1 for s in steps[g]]
    late = [s for g in range(3) if not (early >> g) & 1 for s in steps[g]]
    return [e[len(e) * r // ks:len(e) * (r + 1) // ks] + late[len(late) * r // ks:len(late) * (r + 1) // ks] for r in range(ks)]


def halo_fills(cin, c0, cin2, early, ks):
    """Halo fills (distinct chunks) of each rank's slice."""
    return [sum(1 for i, s in enumerate(mine) if i == 0 or s != mine[i - 1]) for mine in slices(cin, c0, cin2, early, ks)]


def test_plan_splits_k_by_the_early_partition(cabi_lib):
    """sige_tile_conv_plan: the automatic split of a launch with early groups halves until every rank of the partition has a ring
    step (three taps); with no early group the plan is the one it always was."""
    # up.1.block.0.scatter of a DDPM-256 step (32 tiles at 64^2, 128 -> 128, shortcut 128): 8-way without early groups; with the
    # shortcut early, rank 0 of an 8-way split would get none of the 2 early and none of the 6 late steps
    assert min(len(s) for s in slices(128, 128, 128, 4, 8)) == 0 and min(len(s) for s in slices(128, 128, 128, 4, 4)) > 0
    assert _plan(_desc(128, 128, 32, cin2=128)).ksplit == 8
    assert _plan(_desc(128, 128, 32, cin2=128, early=4)).ksplit == 4
    for n_tiles in (1, 4, 16, 32, 64):
        for cin, srcs, cin2, masks in ((512, (512,), 512, (1, 4, 5)), (1024, (512, 512), 0, (1, 2, 3)), (768, (512, 256), 0, (2,)),
                                       (384, (256, 128), 0, (2,)), (256, (128, 128), 256, (2, 4, 6, 7)), (128, (128,), 128, (4,)),
                                       (128, (64, 64), 64, (1, 2, 4, 7))):
            for cout in (128, 256, 512):
                base = _plan(_desc(cin, cout, n_tiles, srcs=srcs, cin2=cin2))
                for early in masks:
                    p = _plan(_desc(cin, cout, n_tiles, srcs=srcs, cin2=cin2, early=early))
                    want = base.ksplit
                    while want > 1 and min(len(s) for s in slices(cin, srcs[0], cin2, early, want)) == 0:
                        want //= 2
                    assert (p.path, p.bn, p.ksplit, p.deep_ring) == (1, base.bn, want, int(want > 1 and base.bn == 64)), \
                        (n_tiles, cin, srcs, cin2, cout, early)
