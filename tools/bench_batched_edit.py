"""Time how a compiled DDPM-256 step of a batch of independent edits takes the next batch, on one GPU.

    python tools/bench_batched_edit.py [--edits 8] [--steps 50] [--warmup 10] [--repeats 3] [--dtype fp16|bf16]

Workload: the in-tree DDPM U-Net at 256 x 256 (sige_b200/workloads/ddpm.py, the same architecture and deterministic weights as
bench.py), fp32 model and dense pass, sparse steps as a fused fp16 step in one CUDA graph.  A batch holds E edits of the one
original image with the edit ratios of BASELINE.json configs[4] (1 / 5 / 15 / 30 %, repeated up to E), each square mask shifted by
its own offset; batch B has the same ratios at other offsets, so that every mask differs from batch A's.

Four timings of a new batch, each the wall time from the mask call to the synchronised end of the first step after it
(`torch.cuda.synchronize()`), taken --repeats times alternating batch B and batch A:
  * recompile         — a step compiled for neither batch: `set_masks` + trace, lowering, three warm-up runs and graph capture;
  * set_masks in place — the step compiled on batch A with headroom 0.5 takes the batch through `set_masks` (`FusedStep.rebind`);
  * set_masks_async    — the same through `set_masks_async` (`FusedStep.rebind_device`: reduced on the device, no host sync);
and the steady-state step time (CUDA events around `model(x, t)`, an L2 flush of a 256 MiB write between steps outside the events)
of the step compiled at headroom 0 and at headroom 0.5, alternated twice, which shows what the padding rows cost when CTAs made only
of padding exit at once.  GPU name, power limit and SM clock are read in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import warnings

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))

from bench_gaugan_gc import gpu_info  # noqa: E402

RATIOS = (0.01, 0.05, 0.15, 0.30)
SHIFT_A = [(0, 0), (20, -12), (-16, 8), (10, 10), (-24, -20), (6, -30), (28, 4), (-8, 16)]
SHIFT_B = [(-30, 20), (12, 24), (24, -10), (-14, -6), (16, 28), (-26, 2), (4, -22), (20, -18)]


def batch(cfg, x0, shifts, E, dev):
    """(inputs [E, C, H, W], mask pyramids {res: [E, H, W]}) of E edits of x0 with the config #5 ratios at `shifts`."""
    import torch

    from sige_b200.masks import downsample_mask, stack_mask_pyramids
    from sige_b200.workloads.ddpm import synthetic_inputs

    xs, pyramids = [], []
    for e in range(E):
        ratio, shift = RATIOS[e % len(RATIOS)], shifts[e % len(shifts)]
        _, x1, mask, _ = synthetic_inputs(cfg, ratio, seed=0, edit_seed=e)
        xs.append(x0 + torch.roll(x1 - x0, shift, (2, 3)))
        pyramids.append(downsample_mask(torch.roll(mask, shift, (0, 1)).to(dev), min_res=8))
    return torch.cat(xs, 0).to(dev), stack_mask_pyramids(pyramids)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--edits", type=int, default=8, help="edits per batch (E)")
    ap.add_argument("--steps", type=int, default=50, help="timed steady-state steps per block")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3, help="new batches timed per install path")
    ap.add_argument("--dtype", choices=["fp16", "bf16"], default="fp16")
    args = ap.parse_args()

    import numpy as np
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_batched_edit: needs a CUDA device")
    from sige_b200.workloads.ddpm import DDPMConfig, SIGEDDPMUNet, init_deterministic, synthetic_inputs

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    dtype = torch.float16 if args.dtype == "fp16" else torch.bfloat16
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    cfg = DDPMConfig()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model = init_deterministic(SIGEDDPMUNet(cfg), seed=0).eval().to(dev)
    x0, _, _, t = synthetic_inputs(cfg, 0.05, seed=0)
    t = t.to(dev)
    with torch.no_grad():
        model.set_mode("full")
        model(x0.to(dev), t)
        model.set_mode("sparse")
    E = args.edits
    xa, ma = batch(cfg, x0, SHIFT_A, E, dev)
    xb, mb = batch(cfg, x0, SHIFT_B, E, dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def new_batch(call, masks, x):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        call(masks)
        model(x, t)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    def installs(call):
        """Seconds per new batch through `call`, alternating B and A, and whether every one ran on the step compiled on A."""
        model.set_fused(True, dtype=dtype, headroom=0.5)
        model.set_masks(ma)
        model(xa, t)
        first = model.fused_step
        secs, in_place, fit = [], True, True
        for i in range(args.repeats):
            for masks, x in ((mb, xb), (ma, xa)):
                secs.append(new_batch(call, masks, x))
                in_place = in_place and model.fused_step is first
                fit = fit and model.masks_async_ok()
        return secs, in_place and fit

    def steady(headroom):
        model.set_fused(True, dtype=dtype, headroom=headroom)
        model.set_masks(ma)
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
        for _ in range(max(1, args.warmup)):
            model(xa, t)
        for i, (a, b) in enumerate(evs):
            flush.fill_(i & 0xFF)
            a.record()
            model(xa, t)
            b.record()
        torch.cuda.synchronize()
        return [a.elapsed_time(b) for a, b in evs]

    with torch.no_grad():
        steady(0.0)                                          # loads every kernel of the step once (first compile, not timed)
        info_before = gpu_info()
        recompile = []
        for i in range(args.repeats):
            for masks, x in ((mb, xb), (ma, xa)):
                model.set_fused(True, dtype=dtype, headroom=0.5)      # drops the compiled step: the next call compiles
                recompile.append(new_batch(model.set_masks, masks, x))
        sync_s, sync_in_place = installs(model.set_masks)
        async_s, async_in_place = installs(model.set_masks_async)
        blocks = {0.0: [], 0.5: []}
        for _ in range(2):
            for h in (0.0, 0.5):
                blocks[h].append(steady(h))
        step = model.fused_step
        caps = sorted({(sl.cap, sl.E) for sl in step.low.slots.values()})
    info = gpu_info()
    med = lambda v: float(np.median(v))  # noqa: E731
    line = {
        "metric": "ddpm-256 batch of %d edits: next batch" % E, "edits": E, "ratios": [RATIOS[e % len(RATIOS)] for e in range(E)],
        "dtype": args.dtype, "gpu": info, "sm_mhz_before_timing": info_before.get("sm_mhz"),
        "recompile_seconds": recompile, "recompile_median_seconds": med(recompile),
        "set_masks_in_place_seconds": sync_s, "set_masks_in_place_median_seconds": med(sync_s), "set_masks_in_place": sync_in_place,
        "set_masks_async_seconds": async_s, "set_masks_async_median_seconds": med(async_s), "set_masks_async_in_place": async_in_place,
        "ms_per_step_headroom_0": [med(b) for b in blocks[0.0]], "ms_per_step_headroom_0.5": [med(b) for b in blocks[0.5]],
        "l2": "flushed (256 MiB write) between timed steps", "steps": args.steps, "warmup": args.warmup,
        "tile_conv_launches": len(step.fused), "slot_caps_headroom_0.5": caps,
    }
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
