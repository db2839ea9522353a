"""Early source groups (sige_tile_conv_t.early), checked without a GPU: which launches of a DDPM-256 step the lowering marks,
and the K partition the wgmma kernel's host plan derives from a mask (sige_tile_conv_plan)."""
import ctypes
import os
import sys

import torch

from conftest import REPO, golden

sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "baseline"))

SHORTCUT_CONV2 = ["down.2.block.0.scatter", "n76.conv3x3", "n194.conv3x3", "n207.conv3x3", "n220.conv3x3", "n237.conv3x3",
                  "n266.conv3x3", "n295.conv3x3", "n328.conv3x3", "n341.conv3x3", "n354.conv3x3"] + \
                 ["up.%d.block.%d.scatter" % (u, b) for u in (2, 1, 0) for b in (0, 1, 2)]
SKIP_CONV1 = ["n189.conv3x3", "n202.conv3x3", "n215.conv3x3", "n232.conv3x3", "n261.conv3x3", "n290.conv3x3", "n323.conv3x3",
              "n336.conv3x3", "n349.conv3x3"] + ["up.%d.block.%d.scatter_gather" % (u, b) for u in (2, 1, 0) for b in (0, 1, 2)]


def test_ddpm256_step_marks_the_shortcut_and_skip_launches():
    """Exactly the 20 fused-shortcut conv2s (bit 2) and the 18 up-path conv1s on cat([h, skip]) (bit 1) get a mask; no marked group
    is written by the preceding step, which is always a tile conv; their predecessors, and only those, release early."""
    from test_fused_cpu import _prepared

    from sige_b200.fused import FusedStep
    from sige_b200.workloads.ddpm import DDPMConfig
    from sim_executor import SimExecutor

    G = golden("ddpm256_golden.npz")
    model, x1, t = _prepared("intree", DDPMConfig(), float(G["ratio"][0]))
    with torch.no_grad():
        step = FusedStep(model, x1, t, executor=SimExecutor())
    assert len(step.fused) == 86
    marked = {f.name: f.spec.early for f in step.fused if f.spec.early}
    assert marked == {**{n: 4 for n in SHORTCUT_CONV2}, **{n: 2 for n in SKIP_CONV1}}
    by_pos = {f.pos: f for f in step.fused}
    kinds = [k for k, _ in step.steps]
    releasers = set()
    for f in step.fused:
        if not f.spec.early:
            continue
        assert kinds[f.pos - 1] == "conv", "%s follows a %s step" % (f.name, kinds[f.pos - 1])
        prev = by_pos[f.pos - 1].spec
        written = {v.untyped_storage().data_ptr() for (v, _, _, _) in prev.aux}
        if prev.dst is not None and prev.dst.has_raw:
            written.add(prev.dst.raw.untyped_storage().data_ptr())
        groups = [[t_] for t_, _ in f.spec.srcs] + [[]] * (2 - len(f.spec.srcs)) + [list(f.spec.shortcut[0]) if f.spec.shortcut else []]
        for g, reads in enumerate(groups):
            if (f.spec.early >> g) & 1:
                assert reads and not any(r.untyped_storage().data_ptr() in written for r in reads), (f.name, g)
        releasers.add(f.pos - 1)
    assert {f.pos for f in step.fused if f.spec.early_release} == releasers
    # after an attention core or a glue step nothing is marked
    for f in step.fused:
        if f.pos > 0 and kinds[f.pos - 1] != "conv":
            assert f.spec.early == 0
    # without programmatic dependent launch there is nothing to overlap
    with torch.no_grad():
        plain = FusedStep(model, x1, t, executor=SimExecutor(), pdl=False)
    assert not any(f.spec.early or f.spec.early_release for f in plain.fused)


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
