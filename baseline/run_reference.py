#!/usr/bin/env python
"""Run the UNMODIFIED reference (baseline/_ref: its python package, its own native backend) on the bench workload.

    PYTHONPATH=baseline/_ref:baseline/_ref/stubs:baseline/_ref/diffusion:<repo> \
        python baseline/run_reference.py --backend cuda|cpu [--steps K --warmup W --ratio r --threads n --dump out.npz]

BENCH / TEST INFRASTRUCTURE.  Everything on the timed path is the reference's: ``sige.nn`` / ``sige.utils`` from
the reference tree (verbatim copy), ``sige.cuda`` (its five CUDA kernels recompiled for sm_90a) or ``sige.cpu`` (its
OpenMP kernels), its model file diffusion/models/ddpm_arch/sige_fused_unet.py, and PyTorch's conv (cuDNN / oneDNN) —
fp32, NCHW, stock backend flags, as the reference runs it.  This repository only contributes the deterministic
weights and synthetic inputs (sige_b200.workloads.ddpm.init_deterministic / synthetic_inputs — numpy-seeded, no
kernels involved) so that both arms see identical tensors.

Timing follows the reference's own Runner.profile (diffusion/runner.py:214-245): W warm-up sparse forwards, then K
timed sparse forwards with a device synchronize after each one, wall clock; for CUDA the same region is also timed
with CUDA events.  Prints ONE JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import warnings


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", default="cuda", choices=["cuda", "cpu"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ratio", type=float, default=0.012)
    ap.add_argument("--threads", type=int, default=0)
    ap.add_argument("--small", action="store_true", help="the 64x64 miniature (tests)")
    ap.add_argument("--workload", default="ddpm", choices=["ddpm", "sd", "gaugan"],
                    help="sd / gaugan: the reference's SIGEUNetModel / SIGEFusedSPADEGenerator at full size (BASELINE.json configs[2], [3]); --small = miniatures")
    ap.add_argument("--no-tf32", action="store_true", help="parity runs: exact fp32 convolutions")
    ap.add_argument("--dump", default=None, help="write the sparse output (and the dense one) to this .npz")
    ap.add_argument("--edit-seed", type=int, default=None)
    args = ap.parse_args()

    import numpy as np
    import torch

    import sige  # the REFERENCE package (baseline/_ref first on PYTHONPATH)

    ref_root = os.path.realpath(os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref"))
    assert os.path.realpath(sige.__file__).startswith(ref_root), "import sige resolved to %s, not the reference install" % sige.__file__
    from sige.utils import dilate_mask, downsample_mask

    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from loader import ddpm_config
    from sige_b200.workloads.ddpm import DDPMConfig, init_deterministic, synthetic_inputs

    if args.threads:
        torch.set_num_threads(args.threads)
    if args.no_tf32:
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda", 0) if args.backend == "cuda" else torch.device("cpu")
    if args.backend == "cuda":
        import sige.cuda  # noqa: F401  (fail loudly if the reference's CUDA extension did not travel)
    def sync():
        if dev.type == "cuda":
            torch.cuda.synchronize()

    size = "mini" if args.small else "full"
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if args.workload == "ddpm":
            from models.ddpm_arch.sige_fused_unet import SIGEFusedUNet

            cfg = DDPMConfig.small() if args.small else DDPMConfig()
            model = init_deterministic(SIGEFusedUNet(None, ddpm_config(cfg)), seed=0).eval().to(dev)
            x0, x1, mask, t = synthetic_inputs(cfg, args.ratio, seed=0, edit_seed=args.edit_seed)
            full_args, sparse_args = (x0.to(dev), t.to(dev)), (x1.to(dev), t.to(dev))
            masks = downsample_mask(mask.to(dev), min_res=8)
        else:
            import consumers

            if args.workload == "sd":
                model = consumers.build_sd(size).to(dev)
                x0, x1, mask, ts, ctx = (v.to(dev) for v in consumers.sd_inputs(size))
                full_args, sparse_args = (x0, ts, ctx), (x1, ts, ctx)
                masks = downsample_mask(mask, min_res=(8, 8) if size == "full" else (4, 4), dilation=1)
            else:
                model = consumers.build_gaugan(size).to(dev)
                s0, s1, mask = (v.to(dev) for v in consumers.gaugan_inputs(size))
                full_args, sparse_args = (s0,), (s1,)
                masks = downsample_mask(dilate_mask(mask, 1), min_res=(4, 8), dilation=0)

    with torch.no_grad():
        model.set_mode("full")
        full0 = model(*full_args)
        model.set_masks(masks)
        model.set_mode("sparse")
        for _ in range(args.warmup):
            out = model(*sparse_args)
            sync()
        ev = None
        if dev.type == "cuda":
            ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            ev[0].record()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            out = model(*sparse_args)
            sync()
        dt = time.perf_counter() - t0
        dev_ms = None
        if ev is not None:
            ev[1].record()
            torch.cuda.synchronize()
            dev_ms = ev[0].elapsed_time(ev[1]) / max(1, args.steps)
    if args.dump:
        np.savez_compressed(args.dump, sparse_out=out.float().cpu().numpy(), full0_out=full0.float().cpu().numpy())
    print(json.dumps({
        "backend": args.backend, "workload": args.workload, "steps": args.steps, "warmup": args.warmup, "ratio": args.ratio,
        "ms_per_step": 1e3 * dt / max(1, args.steps), "steps_per_s": args.steps / dt if dt > 0 else None, "device_ms_per_step": dev_ms,
        "threads": torch.get_num_threads(), "tf32": bool(torch.backends.cudnn.allow_tf32) and dev.type == "cuda",
        "sige_file": os.path.realpath(sige.__file__), "device": str(dev),
        "gpu": torch.cuda.get_device_name(0) if dev.type == "cuda" else None,
    }), flush=True)


if __name__ == "__main__":
    main()
