"""A batch of independent edits of one latent through one fused Stable Diffusion VAE decoder step, on the descriptor simulator.

The mid block's attention of a batch lowers as for one edit: the q conv writes an [E * cap] tile stack over the slot's per-edit lists,
ONE sparse attention runs at B = E (each edit's queries against its own k / v maps) and proj_out reads the output stack through the
same lists (sige_tile_conv_t.idx_per_image with a stack on one side).  Checked here: the batched step has the single-edit step's
launches, on per-edit lists, and no eager node; each edit equals its own single-edit step and edit 0 the golden; a second batch that
fits goes in by `rebind`; an executor without the per-image stacks refuses the batch; the program meets its launch records and has no
PDL hazard, before and after the next batch; the C-ABI's acceptance and refusals of per-image stacks, without a device."""
import copy
import ctypes
import os
import sys
import types
from collections import Counter

import numpy as np
import pytest
import torch

from conftest import REPO, golden

sys.path.insert(0, os.path.join(REPO, "tests"))

import fused_step_contract as fsc  # noqa: E402
import pdl_hazards as ph  # noqa: E402
from sim_executor import SimExecutor  # noqa: E402
from test_sd_decoder import TileListSim  # noqa: E402

from sige_b200._cabi import TILE_NONE  # noqa: E402

E = 3


class _Image:
    """Image e of a destination buffer, as a one-image buffer (what the simulator writes through)."""

    def __init__(self, buf, e):
        self.buf, self.e = buf, e

    shape = property(lambda self: (1,) + tuple(self.buf.shape[1:]))
    has_raw = property(lambda self: self.buf.has_raw)
    raw = property(lambda self: self.buf.raw[self.e:self.e + 1])


class NoStackSim(TileListSim):
    """The simulator with a batch's per-edit lists (a SIGE_TILE_NONE row reads zeros and writes nothing; a stack row b*N + i is list
    row b*N + i), but without the per-image stacks of SIGEAttnBlock's launches."""

    def batch_slots_supported(self):
        return True

    def prepare_conv(self, fc):
        s = fc.spec
        if s.tile_img is None:
            return super().prepare_conv(fc)
        sl = s.slot
        assert sl is not None and s.idx is sl.buf and s.N == sl.E * sl.cap and not (s.src_is_stack and s.dst_stack is not None), s.name
        if s.src_is_stack:                 # one launch per edit on that edit's real rows, into image e of every destination
            shims = []
            for e in range(sl.E):
                inner = copy.copy(s)
                inner.B, inner.tile_img, inner.dst = 1, None, _Image(s.dst, e)
                inner.residual = None if s.residual is None else s.residual[e:e + 1]
                inner.aux = [(v[e:e + 1], sc, sh, act) for (v, sc, sh, act) in s.aux]
                shim = types.SimpleNamespace(spec=inner, launch_fn=None)
                SimExecutor.prepare_conv(self, shim)
                shims.append(shim)

            def run_stack(stream):
                for e, shim in enumerate(shims):
                    rows = torch.arange(e * sl.cap, (e + 1) * sl.cap)
                    rows = rows[s.idx[rows, 0] > TILE_NONE]
                    shim.spec.idx, shim.spec.srcs, shim.spec.N = s.idx[rows], [(s.srcs[0][0][rows], 0)], int(rows.numel())
                    if rows.numel():
                        shim.launch_fn(stream)

            fc.launch_fn = run_stack
            return
        inner = copy.copy(s)
        shim = types.SimpleNamespace(spec=inner, launch_fn=None)
        SimExecutor.prepare_conv(self, shim)

        def run(stream):
            real = s.idx[:, 0] > TILE_NONE
            inner.idx, inner.tile_img, inner.N = s.idx[real], s.tile_img[real], int(real.sum())
            if s.shortcut is not None and s.shortcut[3] is not None:       # one fused-shortcut flag per list row
                inner.shortcut = s.shortcut[:3] + (s.shortcut[3][real],)
            if s.dst_stack is not None:
                inner.dst_stack = torch.empty((inner.N,) + tuple(s.dst_stack.shape[1:]), dtype=s.dst_stack.dtype)
            if inner.N:
                shim.launch_fn(stream)
            if s.dst_stack is not None and inner.N:
                s.dst_stack[real] = inner.dst_stack

        fc.launch_fn = run


class BatchSim(NoStackSim):
    def per_image_stacks_supported(self):
        return True

    def prepare_sparse_attention(self, q, k, v, scale, out):
        self.attention_shapes = getattr(self, "attention_shapes", []) + [tuple(q.shape)]
        return super().prepare_sparse_attention(q, k, v, scale, out)


def _pyramid(mask):
    from sige.utils import downsample_mask

    return downsample_mask(mask, min_res=(4, 4), dilation=0)


def _batch(masks):
    from sige_b200.masks import stack_mask_pyramids

    return stack_mask_pyramids([_pyramid(m) for m in masks])


def _kinds(step):
    return {"steps": Counter(k for k, _ in step.steps), "eager": list(step.eager_nodes), "stems": len(step.low.conv_ins)}


def _rel(a, ref):
    return float(np.abs(np.asarray(a, dtype=np.float64) - ref).max() / np.abs(ref).max())


def _built(executor_cls=BatchSim, singles=False):
    """(net, step, singles [(step, output)], z1s, masks) of the mini decoder: a batch of E edits (headroom 0.5) after the dense pass."""
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige_b200.fused import FusedStep
    from sige_b200.workloads import sd_decoder as SD

    net = SD.build_sd_decoder("mini")
    z0, z1s, masks = SD.sd_decoder_edits("mini", E + 2)
    one = []
    with reference_cpu_runtime(), torch.no_grad():
        net.set_mode("full")
        net(z0)
        net.set_mode("sparse")
        if singles:
            for e in range(E):
                net.set_masks(_pyramid(masks[e]))
                st = FusedStep(net, z1s[e:e + 1], executor=TileListSim())
                one.append((st, st.output.clone()))
        net.set_masks(_batch(masks[:E]))
        step = FusedStep(net, z1s[:E], executor=executor_cls(), headroom=0.5)
    return net, step, one, z1s, masks


def test_batch_of_decoder_edits_runs_as_one_step_and_takes_the_next_batch_in_place():
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige_b200.fused import FusedStep

    net, step, singles, z1s, masks = _built(singles=True)
    sizes = [int(m.sum()) for m in masks[:E]]
    assert len(set(sizes)) == E and any(bool(m[:, 0].any() or m[0].any()) for m in masks[:E])      # other sizes, one on the border
    one, got = _kinds(singles[0][0]), _kinds(step)
    assert got == one and got["steps"]["sparse_attention"] == 1 and not got["eager"], (got, one)
    assert step.ex.attention_shapes == [(E, 1, _cap(step) * 16, 512)]        # B = E, heads 1, cap * 4 * 4 queries per edit
    batched = [f for f in step.fused if f.spec.tile_img is not None]
    assert len(batched) == len(step.fused), [f.name for f in step.fused if f.spec.tile_img is None]
    assert sum(1 for f in batched if f.spec.dst_stack is not None) == 1 and sum(1 for f in batched if f.spec.src_is_stack) == 1
    for f in batched:
        assert f.spec.slot.E == E and f.spec.N == E * f.spec.slot.cap, f.name
    out = step.output.clone()
    assert out.shape[0] == E
    for e, (_, want) in enumerate(singles):
        assert (out[e:e + 1] - want).abs().max().item() <= 2e-5 * want.abs().max().item(), e
    G = golden("sd_decoder_mini_golden.npz")
    assert _rel(out[0:1].numpy(), G["sparse1"]) <= 2e-5

    order = [1, 3, 4]                       # the next batch: each list within the first batch's capacities
    with reference_cpu_runtime(), torch.no_grad():
        net.set_masks(_batch(masks[order]))
        assert step.rebind(), "a batch that fits is installed in place"
        out_b = step(z1s[order]).clone()
        fresh_b = FusedStep(net, z1s[order], executor=BatchSim(), headroom=0.5).output.clone()
    assert torch.equal(out_b, fresh_b)


def _cap(step):
    (cap,) = {f.spec.slot.cap for f in step.fused if f.spec.dst_stack is not None}
    return cap


def test_executor_without_per_image_stacks_still_refuses_the_batch():
    from sige_b200.lazy import TraceUnsupported

    with pytest.raises(TraceUnsupported, match="foreign ops on the tile stack of a batch"):
        _built(NoStackSim)


def test_batched_program_meets_its_records_and_has_no_pdl_hazard_nor_the_next_batch():
    from oracle.cpu_runtime import reference_cpu_runtime

    net, step, _, z1s, masks = _built(fsc.recording(ph.planned(BatchSim)))
    res = fsc.walk(step, model=net)
    print(fsc.summary("sd_decoder mini batch of %d" % E, res))
    fsc.checked_all(step, res)
    assert res["kinds"]["sparse_attention"].launches == 1
    ph.verify(step, "sd_decoder mini batch", net)
    order = [1, 3, 4]
    with reference_cpu_runtime(), torch.no_grad():
        net.set_masks(_batch(masks[order]))
        assert step.rebind()
    step.static_inputs[0].copy_(z1s[order])
    fsc.checked_all(step, fsc.walk(step, model=net))
    ph.verify(step, "sd_decoder mini next batch", net)


# ---------------------------------------------------------------------------------------------------------------- C-ABI (CPU)
def _desc(src_stack, dst_stack):
    """A per-image 1x1 launch on 4x4 tiles (SIGEAttnBlock's q conv / proj_out) whose pointers are not device memory."""
    from sige_b200 import _cabi

    d = _cabi.TileConv()
    d.dtype = _cabi.F16
    d.n_src, d.src[0].ptr, d.src[0].C = 1, 0x10000, 512
    d.B, d.H, d.W, d.idx, d.N, d.idx_per_image = E, 16, 16, 0x20000, 16, 1
    d.R = d.S = 4
    d.w_packed, d.bias = 0x30000, 0x40000
    d.Cin, d.Cout, d.kH, d.kW, d.stride = 512, 512, 1, 1, 1
    d.dst, d.dH, d.dW, d.dC = 0x50000, 16, 16, 512
    d.src_is_stack, d.dst_is_stack = src_stack, dst_stack
    d.flags = _cabi.CONV_TC5 | _cabi.CONV_PADDED
    return d


def test_per_image_stack_descriptors_are_accepted_and_planned_and_stack_to_stack_refused(cabi_lib):
    from sige_b200 import _cabi

    lib = _cabi.lib()
    assert lib.sige_abi_version() == 3

    def verdict(d):
        rc = lib.sige_tile_conv(ctypes.byref(d), None)
        return rc, lib.sige_last_error() if rc else b""

    for tc5 in (True, False):
        for src_stack, dst_stack in ((1, 0), (0, 1)):
            d = _desc(src_stack, dst_stack)
            if not tc5:
                d.flags &= ~_cabi.CONV_TC5
            pl = _cabi.TileConvPlan()
            assert lib.sige_tile_conv_plan(ctypes.byref(d), ctypes.byref(pl)) == 0
            assert pl.path == (1 if tc5 else 0) and pl.grid_x > 0 and pl.grid_y > 0 and pl.grid_z >= 1, (tc5, src_stack)
            if tc5:
                assert pl.grid_x == E * d.N // 8
            d.N = 0                          # the checks pass; N = 0 is then a no-op that touches no pointer
            assert verdict(d) == (0, b""), (tc5, src_stack, dst_stack)
    d = _desc(1, 1)
    rc, msg = verdict(d)
    assert rc != 0 and b"stack to stack" in msg, msg
    for src_stack, dst_stack in ((1, 0), (0, 1)):
        d = _desc(src_stack, dst_stack)
        d.flags |= _cabi.CONV_PER_IMAGE_OPERANDS
        rc, msg = verdict(d)
        assert rc != 0 and b"SIGE_CONV_PER_IMAGE_OPERANDS" in msg, msg
