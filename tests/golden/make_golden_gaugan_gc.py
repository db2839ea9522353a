"""Golden outputs of GauGAN compressed with GAN Compression (the sub-mobile SPADE generator), produced by RUNNING THE REFERENCE:

    python tests/golden/make_golden_gaugan_gc.py           (spawns itself in the reference environment)

In the child process `import sige` is the reference's package from baseline/_ref (its python + its sige.cpu kernels) and the model
is the reference's own SIGEFusedSubMobileSPADEGenerator
(gaugan/models/sub_mobile_spade_generators/sige_fused_sub_mobile_spade_generator.py) in miniature, built and driven by
sige_b200.workloads.gaugan_gc (weights by init_deterministic, the label maps and mask pyramid of the GauGAN workload).
Writes tests/golden/gaugan_gc_mini_golden.npz and nothing else.
"""
import importlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))


def child():
    import numpy as np
    import torch

    import sige

    assert os.path.realpath(sige.__file__).startswith(os.path.realpath(os.path.join(REPO, "baseline", "_ref"))), sige.__file__
    from sige.utils import dilate_mask, downsample_mask

    sys.path.insert(0, os.path.join(REPO, "baseline"))
    import consumers
    from sige_b200.workloads import gaugan_gc as G

    torch.set_num_threads(8)
    pkg = consumers._gaugan_package()
    ref_cls = importlib.import_module(pkg + ".sub_mobile_spade_generators.sige_fused_sub_mobile_spade_generator").SIGEFusedSubMobileSPADEGenerator
    full0, sparse1 = G.run_gaugan_gc(G.build_gaugan_gc("mini", cls=ref_cls), downsample_mask, dilate_mask)
    np.savez_compressed(os.path.join(HERE, "gaugan_gc_mini_golden.npz"), full0=full0.numpy(), sparse1=sparse1.numpy())
    print("gaugan sub-mobile mini:", tuple(sparse1.shape), float(sparse1.abs().max()))


if __name__ == "__main__":
    if "--child" in sys.argv:
        child()
    else:
        sys.path.insert(0, os.path.join(REPO, "baseline"))
        import loader

        sys.exit(subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=loader.reference_env(8)).returncode)
