"""Time the Stable Diffusion VAE decoder's (or encoder's) sparse step on one GPU.

    python tools/bench_sd_decoder.py [--model decoder|encoder] [--size full|mini] [--steps 20] [--warmup 5]

Workload: sige_b200/workloads/sd_decoder.py (the default) — "full" is the first-stage decoder of stable-diffusion/configs/sige.yaml,
z 4 x 64 x 64 -> 512 x 512 — or, with --model encoder, sige_b200/workloads/sd_encoder.py — the first-stage encoder of the same
config, image 3 x 512 x 512 -> moments 8 x 64 x 64 — with BASELINE.json's centred 15 % square edit and the SDEdit runner's mask
pyramid (min_res 4 x 4, dilation 0).
Arms, alternated step by step in one process (CUDA events around each call, an L2 flush (256 MiB write) between calls outside the
events):
  dense        the model's full (dense) pass, fp32, on the original input
  modules      the sparse pass through the eager fp32 operator modules
  fused        the compiled fused fp16 step (CUDA graph)
  fused_core_recorded   the same step with the mid block's attention core left to its recorded torch calls (an executor without
               head dim 512): what the D = 512 sparse-attention launch saves
Then the next edit (a second, smaller mask): the wall time from `set_masks` / `set_masks_async` to the synchronised end of the step
that follows, against a recompile (set_fused + the first call), three times each.  Prints the launch mix of both compiled steps,
the GPU's name, power limit and SM clock read in the same run, and one JSON line.

    python tools/bench_sd_decoder.py [--model decoder|encoder] --size full --edits E

E independent edits of the input (sd_decoder_edits / sd_encoder_edits: edit 0 is the one above, the others smaller, larger, on the border), arms
alternated as above:
  batched      ONE compiled fp16 step over the batch of E edits (per-edit tile lists, headroom 0.5)
  singles      E compiled single-edit fp16 steps, one after another
Then the next batch (edits E .. 2E-1, each list within the first batch's capacities) installed through `set_masks` and through
`set_masks_async`, against a recompile, as above.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time
from collections import Counter

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))

from bench_gaugan_gc import gpu_info  # noqa: E402


def _workload(model):
    """(build, inputs, edits) of the model: build(size) -> net, inputs(size) -> (x0, x1, mask), edits(size, E) -> (x0, x1s, masks)."""
    if model == "encoder":
        from sige_b200.workloads import sd_encoder as SE

        return SE.build_sd_encoder, SE.sd_encoder_inputs, SE.sd_encoder_edits
    from sige_b200.workloads import sd_decoder as SD

    return SD.build_sd_decoder, SD.sd_decoder_inputs, SD.sd_decoder_edits


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="decoder", choices=["decoder", "encoder"])
    ap.add_argument("--size", default="full", choices=["full", "mini"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--edits", type=int, default=1, help="E > 1: a batch of E independent edits in one step, against E single steps")
    args = ap.parse_args()
    if args.edits > 1:
        return batched(args)

    import torch

    from sige.utils import downsample_mask
    from sige_b200.fused import CudaExecutor, FusedStep

    assert torch.cuda.is_available(), "bench_sd_decoder needs a GPU"
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    build, inputs, _ = _workload(args.model)
    net = build(args.size).to(dev)
    z0, z1, mask = (t.to(dev) for t in inputs(args.size))
    res = mask.shape[0]
    mask2 = torch.zeros_like(mask)
    lo = res // 2 - res // 8
    mask2[lo:lo + res // 5, lo - res // 16:lo - res // 16 + res // 5] = True       # a 4 % square near the first edit
    m1, m2 = (downsample_mask(m, min_res=(4, 4), dilation=0) for m in (mask, mask2))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    class CoreRecorded(CudaExecutor):
        def sparse_attention_supported(self, head_dim):
            return head_dim != 512 and super().sparse_attention_supported(head_dim)

    with torch.no_grad():
        net.set_mode("full")
        net(z0)
        net.set_masks(m1)
        net.set_mode("sparse")
        net.set_fused(True, dtype=torch.float16)
        out_fused = net(z1)
        step = net.fused_step
        recorded = FusedStep(net, z1, dtype=torch.float16, executor=CoreRecorded(dev, torch.float16))

        def dense():
            net.set_mode("full")
            net(z0)
            net.set_mode("sparse")

        def modules():
            net.set_fused(False)
            net(z1)

        def fused():
            step(z1)

        def core_recorded():
            recorded(z1)

        arms = {"dense": dense, "modules": modules, "fused": fused, "fused_core_recorded": core_recorded}
        times = {k: [] for k in arms}
        for i in range(args.warmup + args.steps):
            for name, fn in arms.items():
                flush.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fn()
                b.record()
                torch.cuda.synchronize()
                if i >= args.warmup:
                    times[name].append(a.elapsed_time(b))
        err = float((recorded.output.float() - out_fused.float()).abs().max() / out_fused.float().abs().max())

        # the next edit: in place (host lists, device lists) against a recompile
        net.set_fused(True, dtype=torch.float16)
        net(z1)
        step = net.fused_step
        nxt = {"set_masks": [], "set_masks_async": [], "recompile": []}
        in_place = True
        for _ in range(3):
            for how in nxt:
                net.set_masks(m1)
                net(z1)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if how == "set_masks":
                    net.set_masks(m2)
                elif how == "set_masks_async":
                    net.set_masks_async(m2)
                else:
                    net.set_fused(True, dtype=torch.float16)
                    net.set_masks(m2)
                net(z1)
                torch.cuda.synchronize()
                nxt[how].append((time.perf_counter() - t0) * 1e3)
                if how != "recompile":
                    in_place = in_place and net.fused_step is step
                else:
                    net.set_fused(True, dtype=torch.float16)
                    net.set_masks(m1)
                    net(z1)
                    step = net.fused_step

    def mix(s):
        return {"tile_convs": len(s.fused), "steps": dict(Counter(k for k, _ in s.steps)), "eager_nodes": list(s.eager_nodes)}

    tokens = int(step.low.sparse_attention_calls)
    out = {
        "workload": "sd_%s_%s" % (args.model, args.size),
        "edit": "centred 15 %% square of the %d x %d image, min_res 4 x 4, dilation 0" % (res, res),
        "gpu": gpu_info(),
        "ms_median": {k: statistics.median(v) for k, v in times.items()},
        "ms_min": {k: min(v) for k, v in times.items()},
        "next_edit_ms_median": {k: statistics.median(v) for k, v in nxt.items()},
        "next_edit_in_place": in_place,
        "fused": mix(step),
        "fused_core_recorded": mix(recorded),
        "core_recorded_vs_fused_rel_diff": err,
        "sparse_attention_launches": tokens,
        "steps": args.steps,
    }
    print(json.dumps(out))


def _timed(arms, steps, warmup, flush):
    import torch

    times = {k: [] for k in arms}
    for i in range(warmup + steps):
        for name, fn in arms.items():
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            if i >= warmup:
                times[name].append(a.elapsed_time(b))
    return times


def batched(args):
    import torch

    from sige.utils import downsample_mask
    from sige_b200.masks import stack_mask_pyramids

    assert torch.cuda.is_available(), "bench_sd_decoder needs a GPU"
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    E = args.edits
    build, _, edits = _workload(args.model)
    net = build(args.size).to(dev)
    z0, z1s, masks = (t.to(dev) for t in edits(args.size, 2 * E))
    pyrs = [downsample_mask(m, min_res=(4, 4), dilation=0) for m in masks]
    A, B = list(range(E)), list(range(E, 2 * E))
    batch_a, batch_b = (stack_mask_pyramids([pyrs[e] for e in ids]) for ids in (A, B))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    with torch.no_grad():
        net.set_mode("full")
        net(z0)
        net.set_mode("sparse")
        singles = []
        for e in A:
            net.set_fused(True, dtype=torch.float16)
            net.set_masks(pyrs[e])
            o = net(z1s[e:e + 1]).clone()
            singles.append((net.fused_step, o))
        net.set_fused(True, dtype=torch.float16, headroom=0.5)
        net.set_masks(batch_a)
        out = net(z1s[A]).clone()
        step = net.fused_step
        x_a = z1s[A]
        err = max(float((out[i:i + 1].float() - o.float()).abs().max() / o.float().abs().max()) for i, (_, o) in enumerate(singles))

        def one_batch():
            step(x_a)

        def one_by_one():
            for e, (s, _) in enumerate(singles):
                s(z1s[e:e + 1])

        times = _timed({"batched": one_batch, "singles": one_by_one}, args.steps, args.warmup, flush)

        nxt = {"set_masks": [], "set_masks_async": [], "recompile": []}
        in_place = True
        for _ in range(3):
            for how in nxt:
                net.set_fused(True, dtype=torch.float16, headroom=0.5)
                net.set_masks(batch_a)
                net(x_a)
                step = net.fused_step
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if how == "set_masks":
                    net.set_masks(batch_b)
                elif how == "set_masks_async":
                    net.set_masks_async(batch_b)
                else:
                    net.set_fused(True, dtype=torch.float16, headroom=0.5)
                    net.set_masks(batch_b)
                net(z1s[B])
                torch.cuda.synchronize()
                nxt[how].append((time.perf_counter() - t0) * 1e3)
                if how != "recompile":
                    in_place = in_place and net.fused_step is step and net.masks_async_ok()
    caps = sorted({sl.cap for sl in step.low.slots.values()})
    out = {
        "workload": "sd_%s_%s_batch_of_%d" % (args.model, args.size, E),
        "edits": [int(m.sum()) for m in masks[:E]],
        "gpu": gpu_info(),
        "ms_median": {k: statistics.median(v) for k, v in times.items()},
        "ms_min": {k: min(v) for k, v in times.items()},
        "batched_vs_singles_max_rel_diff": err,
        "next_batch_ms_median": {k: statistics.median(v) for k, v in nxt.items()},
        "next_batch_in_place": in_place,
        "tile_list_capacities": caps,
        "batched_steps": dict(Counter(k for k, _ in step.steps)),
        "steps": args.steps,
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
