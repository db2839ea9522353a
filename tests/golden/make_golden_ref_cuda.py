"""Golden outputs of the reference's OWN CUDA PATH on the DDPM-256 step, produced by RUNNING THE REFERENCE ITSELF.

    python tests/golden/make_golden_ref_cuda.py [OUT.npz]      (on a GPU, with baseline/_ref installed)

baseline/run_reference.py runs the unmodified reference (its python package, its sige.cuda kernels built for sm_90a,
cuDNN, exact fp32 convolutions) in a child process where `import sige` is the reference, on the numpy-seeded weights
and inputs of sige_b200.workloads.ddpm at a 1.2 % edit.  Stored: the sparse output in full, and a fixed seeded sample of
the dense output (with its max |value|) so that the file stays below 1 MB.  tests/test_gpu_vs_reference_cuda.py compares
this repository's outputs on the same inputs with them.
"""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
N_SAMPLE = 32768


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "ddpm256_ref_cuda_golden.npz")
    sys.path.insert(0, os.path.join(REPO, "baseline"))
    import loader

    assert loader.available(cuda=True), "baseline/_ref/sige/cuda.so is missing (python baseline/build_ref.py)"
    with tempfile.TemporaryDirectory() as d:
        dump = os.path.join(d, "ref.npz")
        r = subprocess.run([sys.executable, os.path.join(REPO, "baseline", "run_reference.py"), "--backend", "cuda", "--no-tf32", "--steps", "2",
                            "--warmup", "1", "--ratio", "0.012", "--dump", dump], env=loader.reference_env(), capture_output=True, text=True,
                           timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        info = json.loads(r.stdout.strip().splitlines()[-1])
        ref = np.load(dump)
        sparse, full0 = ref["sparse_out"].astype(np.float32), ref["full0_out"].astype(np.float32)
    idx = np.sort(np.random.default_rng(0).choice(full0.size, N_SAMPLE, replace=False)).astype(np.int32)
    np.savez_compressed(out, sparse_out=sparse, full0_idx=idx, full0_sample=full0.reshape(-1)[idx],
                        full0_absmax=np.array([np.abs(full0).max()], np.float64), full0_shape=np.array(full0.shape, np.int64),
                        ratio=np.array([0.012]), gpu=np.array([info["gpu"]]))
    print(out, os.path.getsize(out), info["gpu"])


if __name__ == "__main__":
    main()
