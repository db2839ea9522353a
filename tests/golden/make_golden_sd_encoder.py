"""Golden output of the Stable Diffusion VAE encoder, produced by RUNNING THE REFERENCE ITSELF:

    python tests/golden/make_golden_sd_encoder.py           (spawns itself in the reference environment)

In the child process `import sige` is the reference's package from baseline/_ref (its python + its sige.cpu kernels); the model
is the reference's own SIGEEncoder (stable-diffusion/ldm/modules/diffusionmodules/sige_model.py) at the "mini" size of
sige_b200/workloads/sd_encoder.py, fp32 on the CPU, with the same deterministic weights: a full pass on the original image x0,
set_masks (min_res 4 x 4, dilation 0, as the SDEdit runner), a sparse pass on the edited image x1.  Writes
tests/golden/sd_encoder_mini_golden.npz.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))


def build_reference_encoder(size="mini"):
    """The reference's SIGEEncoder class at one of the in-tree sizes, with the in-tree deterministic weights."""
    for p in (os.path.join(REPO, "baseline", "_ref", "stubs"), os.path.join(REPO, "baseline", "_ref", "stable-diffusion")):
        if p not in sys.path:
            sys.path.append(p)
    from ldm.modules.diffusionmodules.sige_model import SIGEEncoder  # the reference's file, verbatim

    from sige_b200.workloads import sd_encoder as SE

    cfg = SE.SIZES[size]
    net = SIGEEncoder(ch=cfg["ch"], out_ch=SE.IN_CH, ch_mult=cfg["ch_mult"], num_res_blocks=cfg["num_res_blocks"], attn_resolutions=[],
                      in_channels=SE.IN_CH, resolution=cfg["resolution"], z_channels=SE.Z_CHANNELS, double_z=True)
    return SE.init_deterministic(net, seed=SE.SEED).eval()


def child():
    import numpy as np
    import torch

    import sige

    assert os.path.realpath(sige.__file__).startswith(os.path.realpath(os.path.join(REPO, "baseline", "_ref"))), sige.__file__
    from sige.utils import downsample_mask

    from sige_b200.workloads import sd_encoder as SE

    torch.set_num_threads(8)
    full0, sparse1 = SE.run_sd_encoder(build_reference_encoder("mini"), downsample_mask, "mini")
    np.savez_compressed(os.path.join(HERE, "sd_encoder_mini_golden.npz"), full0=full0.numpy(), sparse1=sparse1.numpy())
    print("sd encoder mini:", tuple(sparse1.shape), float(sparse1.abs().max()))


if __name__ == "__main__":
    if "--child" in sys.argv:
        child()
    else:
        sys.path.insert(0, os.path.join(REPO, "baseline"))
        import loader

        sys.exit(subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=loader.reference_env(8)).returncode)
