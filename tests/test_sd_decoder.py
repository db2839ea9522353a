"""The Stable Diffusion VAE decoder (sige_b200/workloads/sd_decoder.py) in miniature, on the CPU: the in-tree restatement against the
golden the reference's own SIGEDecoder produced (tests/golden/make_golden_sd_decoder.py), and its fused step on the descriptor
simulator — the mid block's 512-channel attention core lowered to ONE sparse-attention launch, the recorded calls kept for an
executor without that head dim, and a second mask installed in place."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import REPO, golden

sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "tests", "golden"))

from sim_executor import SimExecutor  # noqa: E402

from sige_b200._cabi import TILE_NONE  # noqa: E402


class TileListSim(SimExecutor):
    """The simulator, plus the kernel's rule for a stack source read through a fixed-capacity tile list: the SIGE_TILE_NONE rows
    that pad the list are computed and write nothing (include/sige_b200.h, sige_tile_conv_t)."""

    def prepare_conv(self, fc):
        super().prepare_conv(fc)
        s = fc.spec
        if not s.src_is_stack or s.idx is None:
            return
        inner = fc.launch_fn

        def run(stream):
            keep = (s.idx, s.srcs, s.N)
            n = int((s.idx[:, 0] != TILE_NONE).sum())          # the padding trails the real tiles
            s.idx, s.srcs, s.N = s.idx[:n], [(s.srcs[0][0][:n],) + tuple(s.srcs[0][1:])] + list(s.srcs[1:]), n
            try:
                inner(stream)
            finally:
                s.idx, s.srcs, s.N = keep

        fc.launch_fn = run


class NoWideHead(TileListSim):
    def sparse_attention_supported(self, head_dim):
        return head_dim != 512


def _decoder():
    from sige_b200.workloads import sd_decoder as SD

    return SD, SD.build_sd_decoder("mini")


def _rel(a, ref):
    return float(np.abs(np.asarray(a, dtype=np.float64) - ref).max() / np.abs(ref).max())


def test_in_tree_decoder_matches_the_reference_golden():
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import downsample_mask

    SD, net = _decoder()
    G = golden("sd_decoder_mini_golden.npz")
    with reference_cpu_runtime():
        full0, sparse1 = SD.run_sd_decoder(net, downsample_mask, fused=lambda n: n.set_fused(False))
    assert _rel(full0.numpy(), G["full0"]) <= 1e-6
    assert _rel(sparse1.numpy(), G["sparse1"]) <= 1e-6


def test_reference_decoder_file_matches_the_golden():
    sys.path.insert(0, os.path.join(REPO, "baseline"))
    import consumers

    if not consumers.available():
        pytest.skip("baseline/_ref absent (python baseline/build_ref.py)")
    from make_golden_sd_decoder import build_reference_decoder
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import downsample_mask

    SD, _ = _decoder()
    net = build_reference_decoder("mini")          # the reference's class on this repository's sige.nn
    G = golden("sd_decoder_mini_golden.npz")
    with reference_cpu_runtime():
        full0, sparse1 = SD.run_sd_decoder(net, downsample_mask, fused=lambda n: n.set_fused(False))
    assert _rel(full0.numpy(), G["full0"]) <= 1e-6
    assert _rel(sparse1.numpy(), G["sparse1"]) <= 1e-6


def _steps(executor):
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import downsample_mask
    from sige_b200.fused import FusedStep

    SD, net = _decoder()
    with reference_cpu_runtime():
        SD.run_sd_decoder(net, downsample_mask, fused=lambda n: n.set_fused(False))
        z1 = SD.sd_decoder_inputs("mini")[1]
        with torch.no_grad():
            step = FusedStep(net, z1, executor=executor)
    return SD, net, step


def test_attention_core_lowers_to_one_sparse_attention_launch():
    G = golden("sd_decoder_mini_golden.npz")
    _, _, step = _steps(TileListSim())
    _, _, plain = _steps(NoWideHead())
    kinds = [k for k, _ in step.steps]
    assert kinds.count("sparse_attention") == 1
    assert not {"bmm", "softmax", "mul", "to_nhwc"} & set(step.eager_nodes), step.eager_nodes
    assert step.refresh_reason is None
    assert _rel(step.output.numpy(), G["sparse1"]) <= 2e-5
    # the q conv's launch moves from the eager core's operand to the kernel's: one conv launch either way
    assert kinds.count("conv") == [k for k, _ in plain.steps].count("conv")
    # without the head dim: today's recorded calls, and the same result
    assert [k for k, _ in plain.steps].count("sparse_attention") == 0
    assert plain.eager_nodes == ["bmm", "mul", "softmax", "bmm", "to_nhwc"]
    assert _rel(plain.output.numpy(), G["sparse1"]) <= 2e-5


def test_second_mask_rebinds_in_place():
    from oracle.cpu_runtime import reference_cpu_runtime
    from sige.utils import downsample_mask
    from sige_b200.fused import FusedStep

    SD, net, step = _steps(TileListSim())
    z0, z1, mask = SD.sd_decoder_inputs("mini")
    mask2 = torch.zeros_like(mask)
    mask2[12:20, 6:15] = True                        # another edit that fits the lists' capacity
    with reference_cpu_runtime(), torch.no_grad():
        net.set_masks(downsample_mask(mask2, min_res=(4, 4), dilation=0))
        assert step.rebind()
        out = step(z1).clone()
        want = FusedStep(net, z1, executor=TileListSim()).output
        net.set_fused(False)
        eager = net(z1)
    assert torch.equal(out, want)
    assert _rel(out.numpy(), eager.numpy()) <= 2e-5
