"""Ours vs the REFERENCE'S OWN CUDA PATH (north star: "outputs match the reference's own CUDA path on identical inputs").
tests/golden/make_golden_ref_cuda.py ran the unmodified reference — its python package, its sige.cuda kernels built for
sm_90a, cuDNN, exact fp32 — on an H100 and stored its outputs in tests/golden/ddpm256_ref_cuda_golden.npz; this test runs
the same model on this repository's sige with the same weights and inputs (numpy-seeded).  The model is the reference's
unmodified model file when baseline/_ref is installed, else the in-tree restatement of the same architecture."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import REPO, golden

sys.path.insert(0, os.path.join(REPO, "baseline"))
pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def test_against_the_references_own_cuda_path():
    import warnings

    import loader
    from sige.utils import downsample_mask
    from sige_b200.workloads.ddpm import DDPMConfig, SIGEDDPMUNet, init_deterministic, synthetic_inputs

    ref = golden("ddpm256_ref_cuda_golden.npz")
    saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        cfg = DDPMConfig()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            net = loader.reference_ddpm_on_this_repo(cfg) if loader.available() else SIGEDDPMUNet(cfg)
            model = init_deterministic(net, seed=0).eval().to(DEV)
        x0, x1, mask, t = synthetic_inputs(cfg, float(ref["ratio"][0]), seed=0)
        with torch.no_grad():
            model.set_mode("full")
            full0 = model(x0.to(DEV), t.to(DEV))
            model.set_masks(downsample_mask(mask.to(DEV), min_res=8))
            model.set_mode("sparse")
            model.set_fused(False)
            ours_fp32 = model(x1.to(DEV), t.to(DEV))                  # eager operator modules, exact fp32 kernels
            model.set_fused(True, dtype=torch.float16)
            ours_fused = model(x1.to(DEV), t.to(DEV))                 # fused step, fp16 tensor-core arithmetic
            assert model.fused_step is not None and model.fused_step.eager_nodes == []
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved
    want = ref["sparse_out"]
    scale = np.abs(want).max()
    assert tuple(full0.shape) == tuple(ref["full0_shape"])
    e_full = np.abs(full0.cpu().numpy().reshape(-1)[ref["full0_idx"]] - ref["full0_sample"]).max() / float(ref["full0_absmax"][0])
    e32 = np.abs(ours_fp32.cpu().numpy() - want).max() / scale
    e16 = np.abs(ours_fused.cpu().numpy() - want).max() / scale
    big = np.abs(want) >= 0.05 * scale
    r16 = (np.abs(ours_fused.cpu().numpy() - want)[big] / np.abs(want[big])).max()
    print("vs the reference's CUDA path (%s): dense pass %.3g; sparse fp32 modules %.3g; sparse fp16 fused max %.3g rel(|ref|>5%%) %.3g"
          % (ref["gpu"][0], e_full, e32, e16, r16))
    assert e_full <= 1e-5, "same dense pass (same cuDNN) expected"
    assert e32 <= 1e-5, "fp32 operator modules vs the reference's CUDA kernels + cuDNN (north star: 1e-5 rel fp32)"
    assert e16 <= 5e-3, "fp16 fused step vs the reference's fp32 CUDA path"
