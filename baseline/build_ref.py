"""Recipe: install the UNMODIFIED reference under baseline/_ref/ (git-ignored, travels with gpurun).

BENCH / TEST INFRASTRUCTURE — nothing under sige_b200/ or sige/ imports what this produces.

    python baseline/build_ref.py [--force] [--no-cuda]

What lands in baseline/_ref/ (all of it produced from /root/reference where it lies; nothing of it is
tracked by git):

    sige/                 the reference's python package, verbatim (sige/__init__.py, __version__.py,
                          utils.py, nn/*.py) + its two native backends built from the reference's own
                          sources with the reference's own flags (setup.py:147-182):
        cpu.so            sige/cpu/*.cpp + sige/common.cpp              (-g -O3 -fopenmp)
        cuda.so           sige/cuda/*.{cpp,cu} + sige/common.cpp        (nvcc -O3, TORCH_CUDA_ARCH_LIST=9.0a;
                          the reference's setup.py only builds it when a GPU is visible at build time
                          (setup.py:164) and passes no arch flags; nvcc cross-compiles it here)
    diffusion/            models/ (the DDPM / PD U-Nets: the north-star model file
                          models/ddpm_arch/sige_fused_unet.py) + configs/
    stable-diffusion/ldm  the SD model files that use sige.nn (import / shape tests)
    gaugan/models         the GauGAN generators that use sige.nn
    example.py, assets/mask.npy
    stubs/                few-line stand-ins for `easydict`, `torchprofile`, `omegaconf.listconfig` (absent from this image,
                          no network; SURVEY.md Appendix D) — only so that the model files import

Used by: bench.py --impl reference (the reference's python + sige.cpu + oneDNN on the host cores),
bench.py --impl reference-cuda (the reference's python + sige.cuda + cuDNN on the same H100),
tests/test_gpu_reference_model.py (the reference's unmodified model file on THIS repo's sige.nn) and
tests/test_gpu_vs_reference_cuda.py (ours vs the reference's own CUDA path).
"""
from __future__ import annotations

import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = os.environ.get("SIGE_REFERENCE_ROOT", "/root/reference")
OUT = os.path.join(HERE, "_ref")

CPU_SOURCES = ["sige/cpu/gather.cpp", "sige/cpu/scatter.cpp", "sige/cpu/scatter_gather.cpp", "sige/cpu/common_cpu.cpp",
               "sige/cpu/pybind_cpu.cpp", "sige/common.cpp"]
CUDA_SOURCES = ["sige/cuda/gather.cpp", "sige/cuda/gather_kernel.cu", "sige/cuda/scatter.cpp", "sige/cuda/scatter_kernel.cu",
                "sige/cuda/scatter_gather.cpp", "sige/cuda/scatter_gather_kernel.cu", "sige/cuda/common_cuda.cu",
                "sige/cuda/pybind_cuda.cpp", "sige/common.cpp"]

PY_TREES = [  # (source relative to the reference root, destination relative to baseline/_ref, file filter)
    ("sige", "sige", (".py",)),
    ("diffusion/models", "diffusion/models", (".py",)),
    ("diffusion/configs", "diffusion/configs", (".yml",)),
    ("diffusion_demo/models", "diffusion_demo/models", (".py",)),
    ("stable-diffusion/ldm", "stable-diffusion/ldm", (".py",)),
    ("stable-diffusion/configs", "stable-diffusion/configs", (".yaml",)),
    ("gaugan/models", "gaugan/models", (".py",)),
]
FILES = ["example.py", "assets/mask.npy"]

STUBS = {
    "easydict/__init__.py": (
        "class EasyDict(dict):\n"
        "    def __init__(self, d=None, **kw):\n"
        "        super().__init__()\n"
        "        for k, v in dict(d or {}, **kw).items():\n"
        "            self[k] = v\n"
        "    def __setitem__(self, k, v):\n"
        "        if isinstance(v, dict) and not isinstance(v, EasyDict):\n"
        "            v = EasyDict(v)\n"
        "        super().__setitem__(k, v)\n"
        "    __setattr__ = __setitem__\n"
        "    def __getattr__(self, k):\n"
        "        try:\n"
        "            return self[k]\n"
        "        except KeyError:\n"
        "            raise AttributeError(k)\n"
    ),
    "torchprofile/__init__.py": "def profile_macs(*args, **kwargs):\n    return 0\n",
    # stable-diffusion/ldm/modules/diffusionmodules/sige_openaimodel.py:266 imports it only to test `type(context_dim) == ListConfig`
    "omegaconf/__init__.py": "from .listconfig import ListConfig  # noqa: F401\n",
    "omegaconf/listconfig.py": "class ListConfig(list):\n    pass\n",
}


def ref_available() -> bool:
    return all(os.path.isfile(os.path.join(REF_ROOT, s)) for s in CPU_SOURCES + CUDA_SOURCES)


def installed(need_cuda: bool = True) -> bool:
    ok = os.path.isfile(os.path.join(OUT, "sige", "cpu.so")) and os.path.isfile(os.path.join(OUT, "sige", "nn", "base.py"))
    ok = ok and os.path.isfile(os.path.join(OUT, "diffusion", "models", "ddpm_arch", "sige_fused_unet.py"))
    if need_cuda:
        ok = ok and os.path.isfile(os.path.join(OUT, "sige", "cuda.so"))
    return ok


def _copy_tree(src_rel: str, dst_rel: str, exts) -> int:
    n = 0
    src_root = os.path.join(REF_ROOT, src_rel)
    for root, dirs, files in os.walk(src_root):
        dirs[:] = [d for d in dirs if d not in ("__pycache__", "mps", "cpu", "cuda")]
        for f in files:
            if not f.endswith(tuple(exts)):
                continue
            rel = os.path.relpath(os.path.join(root, f), src_root)
            dst = os.path.join(OUT, dst_rel, rel)
            os.makedirs(os.path.dirname(dst), exist_ok=True)
            shutil.copyfile(os.path.join(root, f), dst)
            n += 1
    return n


def _build_ext(name: str, sources, with_cuda: bool, verbose: bool) -> str:
    os.environ["CXX"] = "/usr/bin/g++"      # the image's /opt/gcc wrapper cannot find libgomp.spec (SURVEY Appendix D)
    os.environ["CC"] = "/usr/bin/gcc"
    if with_cuda:
        os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0a"
    from torch.utils.cpp_extension import load

    build_dir = os.path.join(OUT, "_build_" + name)
    os.makedirs(build_dir, exist_ok=True)
    load(name=name, sources=[os.path.join(REF_ROOT, s) for s in sources],
         extra_cflags=["-g", "-O3", "-fopenmp"], extra_cuda_cflags=["-O3"] if with_cuda else None,
         extra_ldflags=["-fopenmp"], build_directory=build_dir, is_python_module=False, with_cuda=with_cuda, verbose=verbose)
    dst = os.path.join(OUT, "sige", name + ".so")
    shutil.copy2(os.path.join(build_dir, name + ".so"), dst)
    shutil.rmtree(build_dir, ignore_errors=True)
    return dst


def build(force: bool = False, cuda: bool = True, verbose: bool = False):
    """Returns baseline/_ref (or None when the reference tree is absent and nothing was prebuilt)."""
    if not ref_available():
        return OUT if installed(need_cuda=False) else None
    os.makedirs(OUT, exist_ok=True)     # python trees + stubs are refreshed every time (cheap); the extensions only when missing
    for src, dst, exts in PY_TREES:
        if os.path.isdir(os.path.join(REF_ROOT, src)):
            _copy_tree(src, dst, exts)
    for f in FILES:
        if os.path.isfile(os.path.join(REF_ROOT, f)):
            os.makedirs(os.path.dirname(os.path.join(OUT, f)) or OUT, exist_ok=True)
            shutil.copyfile(os.path.join(REF_ROOT, f), os.path.join(OUT, f))
    for rel, text in STUBS.items():
        p = os.path.join(OUT, "stubs", rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "w") as fh:
            fh.write(text)
    if force or not os.path.isfile(os.path.join(OUT, "sige", "cpu.so")):
        _build_ext("cpu", CPU_SOURCES, False, verbose)
    if cuda and (force or not os.path.isfile(os.path.join(OUT, "sige", "cuda.so"))):
        _build_ext("cuda", CUDA_SOURCES, True, verbose)
    return OUT


if __name__ == "__main__":
    print("reference install:", build(force="--force" in sys.argv, cuda="--no-cuda" not in sys.argv, verbose=True))
