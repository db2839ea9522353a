"""Time the sparse step of a GauGAN generator on one GPU: GauGAN compressed with GAN Compression (the sub-mobile SPADE generator,
the default) or the full SPADE generator.

    python tools/bench_gaugan_gc.py [--generator gc|spade] [--steps 50] [--warmup 10] [--dtype fp16|bf16] [--size full|mini]
                                    [--headroom 0.5] [--dump-outputs DIR] [--per-launch] [--edits E]

Workload (--generator gc): sige_b200/workloads/gaugan_gc.py at full size — 512 x 1024 label map, config 32_32_32_48_32_24_24_32 (the
published GAN Compression Cityscapes sub-network), 5 sparse blocks, the 2.98 % label edit of the full-size GauGAN workload.
--generator spade: sige_b200/workloads/gaugan_spade.py (ngf 64, `more` up-sampling layers, 5 sparse blocks) on the same label maps
and edit.  Either way: fp32 model and dense pass, sparse step as a fused fp16 step (`set_fused(True, dtype=torch.float16)`) in one
CUDA graph.  As bench.py: warm-up,
per-step CUDA events around `model(x)`, an L2 flush (256 MiB write) between steps outside the events, GPU name / power limit /
SM clock read in the same run, the launch mix of the compiled step, and --dump-outputs DIR (the last timed step's output as
float32 .npy).  The step is compiled with --headroom (extra tile-list capacity); after the timed steps the next-edit figure is
the wall time from `set_masks_async` of a second, smaller label edit to the synchronised end of the step that follows it (an
interactive user's next stroke), taken three times alternating with the first edit; `next_edit_in_place` says whether the
compiled step took the edit without recompiling.  --per-launch adds the CUDA-event time of every tile-conv launch of the compiled
step, each after an L2 flush (launch latency included), and the kernel it runs (from its launch plan: `wgmma bn=.. ksplit=..` or
`mma.sync`).  --edits E (E > 1) adds a batch of E independent label edits of the scene (`gaugan_gc_edits`: the workload's edit,
`edit_b`, then seeded edits elsewhere): one compiled step of the batch against the E single-edit steps, timed in the same run and
alternated (each step replayed through its own CUDA graph, an L2 flush before each), and the install of the next batch of E edits
into the batched step through `set_masks` and through `set_masks_async`, against a recompile (wall time to the synchronised end
of the step that follows).  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from collections import Counter

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)


def gpu_info() -> dict:
    import torch

    info = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        pl, sm, sm_max = (v.strip() for v in r.stdout.strip().split(","))
        info.update({"power_limit_w": float(pl), "sm_mhz": float(sm), "sm_max_mhz": float(sm_max)})
    except Exception as e:  # noqa: BLE001
        info["nvidia_smi"] = "unavailable: %s" % e
    return info


def edit_b(size: str):
    """A second label edit, smaller than the workload's and elsewhere in the image: (edited label map, its mask)."""
    from sige_b200.workloads import gaugan_gc as G

    _, s1s, masks = G.gaugan_gc_edits(size, 2)
    return s1s[1:2], masks[1]


def next_edit(net, x_a, dilate_mask, downsample_mask, size: str, dev):
    """Wall seconds from set_masks_async of the next edit to the synchronised end of the step after it, three times (edit B, edit A,
    edit B); and whether every one ran on the step compiled first."""
    import torch

    from sige_b200.workloads import gaugan_gc as G

    x_b, mask_b = (t.to(dev) for t in edit_b(size))
    mask_a = G.gaugan_gc_inputs(size)[2].to(dev)
    pyr = {k: downsample_mask(dilate_mask(m, 1), min_res=(4, 8), dilation=0) for k, m in (("a", mask_a), ("b", mask_b))}
    first = net.fused_step
    out, in_place = [], True
    with torch.no_grad():
        for k, x in (("b", x_b), ("a", x_a), ("b", x_b)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            net.set_masks_async(pyr[k])
            net(x)
            torch.cuda.synchronize()
            out.append(time.perf_counter() - t0)
            in_place = in_place and net.fused_step is first
    return out, in_place


def batch_of_edits(net, E: int, size: str, dtype, headroom: float, steps: int, warmup: int, flush, dev) -> dict:
    """The --edits figures (see the module docstring); `net` has had its dense pass and is in sparse mode."""
    import numpy as np
    import torch

    from sige.utils import dilate_mask, downsample_mask
    from sige_b200.masks import stack_mask_pyramids
    from sige_b200.workloads import gaugan_gc as G

    _, s1s, masks = G.gaugan_gc_edits(size, 2 * E)
    s1s, masks = s1s.to(dev), masks.to(dev)

    def pyr(m):
        return downsample_mask(dilate_mask(m, 1), min_res=(4, 8), dilation=0)

    def batch(sel):
        return stack_mask_pyramids([pyr(masks[e]) for e in sel])

    A, B = list(range(E)), list(range(E, 2 * E))
    singles = []
    with torch.no_grad():
        for e in A:
            net.set_fused(True, dtype=dtype, headroom=headroom)
            net.set_masks(pyr(masks[e]))
            net(s1s[e:e + 1])
            singles.append((net.fused_step, s1s[e:e + 1]))
        net.set_fused(True, dtype=dtype, headroom=headroom)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        t0 = time.perf_counter()
        net.set_masks(batch(A))
        net(s1s[A])
        torch.cuda.synchronize()
        compile_s = time.perf_counter() - t0
        peak = torch.cuda.max_memory_allocated(dev) - base
        step, xa = net.fused_step, s1s[A]

    def one(st, x):
        if flush is not None:
            flush.fill_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        st(x)
        b.record()
        return a, b

    batched, separate = [], []
    with torch.no_grad():
        for i in range(warmup + steps):
            ev_b = one(step, xa)
            ev_s = [one(st, x) for st, x in singles]
            torch.cuda.synchronize()
            if i >= warmup:
                batched.append(ev_b[0].elapsed_time(ev_b[1]))
                separate.append(sum(a.elapsed_time(b) for a, b in ev_s))

    def install(fn, pyramid, x):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn(pyramid)
        net(x)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    res = {"sync": [], "async": []}
    in_place = True
    with torch.no_grad():
        pa, pb = batch(A), batch(B)
        for _ in range(3):
            for k, fn in (("sync", net.set_masks), ("async", net.set_masks_async)):
                res[k].append(install(fn, pb, s1s[B]))
                in_place = in_place and net.fused_step is step
                install(net.set_masks, pa, xa)
        in_place = in_place and net.masks_async_ok()
        recompile = []
        for _ in range(2):
            net.set_fused(True, dtype=dtype, headroom=headroom)
            recompile.append(install(net.set_masks, pb, s1s[B]))
    return {"E": E, "mask_pixels": [int(m.sum()) for m in masks[A]], "batched_ms": float(np.median(batched)),
            "single_edit_steps_ms": float(np.median(separate)), "batched_over_singles": float(np.median(batched) / np.median(separate)),
            "rounds": len(batched), "batched_compile_seconds": compile_s, "batched_compile_peak_bytes": int(peak),
            "next_batch_set_masks_seconds": res["sync"], "next_batch_set_masks_async_seconds": res["async"],
            "next_batch_recompile_seconds": recompile, "next_batch_in_place": in_place}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--generator", choices=["gc", "spade"], default="gc", help="sub-mobile (GAN Compression) or full SPADE generator")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--dtype", choices=["fp16", "bf16"], default="fp16")
    ap.add_argument("--size", choices=["full", "mini"], default="full")
    ap.add_argument("--no-flush", action="store_true", help="do not flush L2 between timed steps")
    ap.add_argument("--headroom", type=float, default=0.5, help="extra tile-list capacity of the compiled step")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    ap.add_argument("--per-launch", action="store_true", help="time every tile-conv launch of the compiled step on its own")
    ap.add_argument("--edits", type=int, default=1, help="E > 1: also time a batch of E label edits against E single-edit steps")
    args = ap.parse_args()

    import numpy as np
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_gaugan_gc: needs a CUDA device")
    from sige.utils import dilate_mask, downsample_mask
    from sige_b200.workloads import gaugan_gc as G

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    dtype = torch.float16 if args.dtype == "fp16" else torch.bfloat16
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    if args.generator == "spade":
        from sige_b200.workloads.gaugan_spade import build_gaugan_spade

        net = build_gaugan_spade(args.size).to(dev)
    else:
        net = G.build_gaugan_gc(args.size).to(dev)
    t0 = time.time()
    G.run_gaugan_gc(net, downsample_mask, dilate_mask, device=dev, size=args.size,
                    fused=lambda n: n.set_fused(True, dtype=dtype, headroom=args.headroom))
    compile_s = time.time() - t0
    step = net.fused_step
    x = G.gaugan_gc_inputs(args.size)[1].to(dev)
    flush = None if args.no_flush else torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timed(k):
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(k)]
        out = None
        with torch.no_grad():
            for i in range(k):
                if flush is not None:
                    flush.fill_(i & 0xFF)
                evs[i][0].record()
                out = net(x)
                evs[i][1].record()
        torch.cuda.synchronize()
        return [a.elapsed_time(b) for a, b in evs], out

    timed(max(1, args.warmup))
    info_before = gpu_info()
    ms, out = timed(max(1, args.steps))
    info = gpu_info()
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        np.save(os.path.join(args.dump_outputs, "out.npy"), out.float().cpu().numpy())
    per_launch = None
    if args.per_launch:
        from sige_b200.roofline import kernel_name, plan_of

        stream = torch.cuda.current_stream(dev)
        per_launch = []
        with torch.no_grad():
            for f in step.fused:
                evs = []
                for i in range(10):
                    if flush is not None:
                        flush.fill_(i)
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(stream)
                    f.launch(stream.cuda_stream)
                    b.record(stream)
                    evs.append((a, b))
                torch.cuda.synchronize()
                per_launch.append({"launch": f.name, "us": 1e3 * float(np.median([a.elapsed_time(b) for a, b in evs])),
                                   "modulated": f.spec.modulation is not None, "Cin": f.spec.Cin, "Cout": f.spec.Cout, "k": f.spec.k,
                                   "kernel": kernel_name(plan_of(f))})
    next_edit_s, in_place = next_edit(net, x, dilate_mask, downsample_mask, args.size, dev)
    kinds = Counter(k for k, _ in step.steps) if step is not None else Counter()
    low = step.low if step is not None else None
    line = {
        "metric": "gaugan-%s %s sparse step" % (args.generator, args.size), "generator": args.generator, "ms_per_step": float(np.median(ms)), "ms_mean": float(np.mean(ms)),
        "ms_min": float(np.min(ms)), "ms_max": float(np.max(ms)), "steps": len(ms), "warmup": args.warmup,
        "dtype": args.dtype, "l2": "not flushed" if flush is None else "flushed (256 MiB write) between timed steps",
        "gpu": info, "sm_mhz_before_timing": info_before.get("sm_mhz"), "compile_seconds": compile_s,
        "next_edit_seconds": next_edit_s, "next_edit_median_seconds": float(np.median(next_edit_s)), "next_edit_in_place": in_place,
        "headroom": args.headroom,
        "launches": {"tile_conv": len(step.fused) if step else 0, "separable": kinds.get("separable", 0), "spade": kinds.get("spade", 0),
                     "modulated": sum(1 for f in step.fused if getattr(f.spec, "modulation", None) is not None) if step else 0,
                     "eager_nodes": len(step.eager_nodes) if step else None},
        "eager_node_kinds": dict(Counter(step.eager_nodes).most_common(8)) if step else None,
        "separable_branches": [len(r.branches) for r in getattr(low, "separable", [])] if low is not None else None,
    }
    if per_launch is not None:
        line["per_launch"] = per_launch
    if args.edits > 1:
        line["batch_of_edits"] = batch_of_edits(net, args.edits, args.size, dtype, args.headroom, max(1, args.steps), max(1, args.warmup), flush, dev)
        line["batch_of_edits"]["gpu"] = gpu_info()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
