"""Live roofline measurement of the dominant kernel (the fused tile convolution), for bench.py.

achieved = ALGORITHMIC bytes per launch / average launch duration, with the duration taken from
CUDA events on the launching stream around each launch (L2 flushed before every launch).
Algorithmic bytes of one tile-conv launch (SURVEY.md §8d):
    e * [ M*Cin*R*S (tile read) + kH*kW*Cout*Cin (weights) + M*Cout*Ro*So (write) ],  e = 2 (fp16/bf16)
and its FLOPs 2*M*Ro*So*Cout*Cin*kH*kW.  Peaks come from MEASURED_PEAKS.json (driver-written),
else the H100 SXM data sheet (3350 GB/s HBM3, 989 TFLOP/s dense fp16/bf16; not measured).
"""
from __future__ import annotations

import json
import os

import torch

from . import ops
from .nn import SIGEConv2d

_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def peaks():
    p = os.path.join(_REPO, "MEASURED_PEAKS.json")
    try:
        d = json.load(open(p))
        return {"hbm_gbs": float(d["hbm_gbs"]), "bf16_tflops": float(d.get("bf16_tflops", 989.0)), "source": "measured (MEASURED_PEAKS.json)"}
    except Exception:  # noqa: BLE001
        return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "source": "H100 SXM data sheet (not measured)"}


def conv_layers_of_step(model, x, t):
    """One sparse forward with hooks: [(module, input stack shape)] for every tensor-core tile conv."""
    seen = []
    hooks = []

    def hook(mod, inp, out):
        xin = inp[0]
        if xin.is_cuda and mod.mode == "sparse" and ops.tile_conv_tc_supported(xin, mod.weight, mod.stride, mod.dilation, mod.groups):
            seen.append((mod, tuple(xin.shape)))

    for m in model.modules():
        if isinstance(m, SIGEConv2d):
            hooks.append(m.register_forward_hook(hook))
    try:
        with torch.no_grad():
            model(x, t)
    finally:
        for h in hooks:
            h.remove()
    return seen


def measure_layers(layers, dtype, flush, reps: int = 10):
    """layers: [(module, (M, Cin, R, S))].  Returns the roofline dict."""
    if not layers:
        return None
    dev = layers[0][0].weight.device
    stream = torch.cuda.current_stream(dev)
    tot_bytes = tot_flops = tot_ms = 0.0
    n_launch = 0
    cache = {}
    for mod, shape in layers:
        M, Cin, R, S = shape
        kH, kW = mod.kernel_size
        st = mod.stride[0]
        Cout = mod.out_channels
        Ro, So = (R - kH) // st + 1, (S - kW) // st + 1
        key = (shape, Cout, kH, st)
        if key not in cache:
            x = torch.randn(shape, device=dev, dtype=dtype).contiguous(memory_format=torch.channels_last)
            wp, b32 = mod._packed_weight(dtype)
            out = ops.tile_conv_stack(x, wp, b32, (kH, kW), st)
            ms = 0.0
            for i in range(reps):
                if flush is not None:
                    flush.fill_(i)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                ops.tile_conv_stack(x, wp, b32, (kH, kW), st, out=out)
                b.record(stream)
                b.synchronize()
                ms += a.elapsed_time(b)
            cache[key] = ms / reps
        tot_ms += cache[key]
        tot_bytes += 2.0 * (M * Cin * R * S + kH * kW * Cout * Cin + M * Cout * Ro * So)
        tot_flops += 2.0 * M * Ro * So * Cout * Cin * kH * kW
        n_launch += 1
    pk = peaks()
    achieved = tot_bytes / (tot_ms * 1e-3) / 1e9
    return {
        "bound": "hbm", "achieved": achieved, "peak": pk["hbm_gbs"], "unit": "GB/s", "frac": achieved / pk["hbm_gbs"], "traffic": None,
        "kernel": "sige::tile_conv_mma_kernel (all %d tensor-core tile convs of one step)" % n_launch,
        "avg_launch_us": 1e3 * tot_ms / n_launch, "algorithmic_bytes_per_step": tot_bytes, "peak_source": pk["source"],
        "tensor": {"achieved_tflops": tot_flops / (tot_ms * 1e-3) / 1e12, "peak_tflops": pk["bf16_tflops"],
                   "frac": tot_flops / (tot_ms * 1e-3) / 1e12 / pk["bf16_tflops"]},
        "note": "cold L2 (flushed before every launch); launch latency included in the event bracket",
    }


def measure_dominant_kernel(model, dtype, flush):
    from .workloads.ddpm import DDPMConfig, synthetic_inputs

    dev = next(model.parameters()).device
    _, x1, _, t = synthetic_inputs(getattr(model, "cfg", DDPMConfig()), 0.012, seed=0)
    x = x1.to(dev).to(dtype).contiguous(memory_format=torch.channels_last)
    layers = conv_layers_of_step(model, x, t.to(dev))
    return measure_layers(layers, dtype, flush)


def measure_engine(engine, flush, reps: int = 5):
    """Per-launch CUDA-event timing of every fused tile-conv launch of the step engine (cold L2).
    achieved = sum(algorithmic bytes) / sum(launch durations)."""
    dev = engine.dev
    stream = torch.cuda.current_stream(dev)
    tot_ms = 0.0
    per = []
    for f in engine.fused:
        ms = 0.0
        for i in range(reps):
            if flush is not None:
                flush.fill_(i)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            f.launch(stream.cuda_stream)
            b.record(stream)
            b.synchronize()
            ms += a.elapsed_time(b)
        per.append((f.name, ms / reps, f.bytes, f.flops, f.tiles))
        tot_ms += ms / reps
    pk = peaks()
    tot_bytes, tot_flops = float(engine.algorithmic_bytes()), float(engine.algorithmic_flops())
    achieved = tot_bytes / (tot_ms * 1e-3) / 1e9
    slow = sorted(per, key=lambda r: -r[1])[:5]
    return {
        "bound": "hbm", "achieved": achieved, "peak": pk["hbm_gbs"], "unit": "GB/s", "frac": achieved / pk["hbm_gbs"],
        "traffic": None, "algorithmic_bytes_per_launch": tot_bytes / max(1, len(per)),
        "kernel": "sige::tc5::tile_conv_tc5_kernel / sige::tile_conv_mma_kernel (all %d fused gather-conv-scatter launches of one step)" % len(per),
        "avg_launch_us": 1e3 * tot_ms / max(1, len(per)), "algorithmic_bytes_per_step": tot_bytes, "peak_source": pk["source"],
        "tensor": {"achieved_tflops": tot_flops / (tot_ms * 1e-3) / 1e12, "peak_tflops": pk["bf16_tflops"],
                   "frac": tot_flops / (tot_ms * 1e-3) / 1e12 / pk["bf16_tflops"]},
        "slowest": [{"layer": n, "us": 1e3 * ms, "tiles": t, "GBps": by / (ms * 1e-3) / 1e9} for n, ms, by, fl, t in slow],
        "note": "cold L2 (flushed before every launch); launch latency included in the event bracket",
    }


def plan_of(fc):
    """The launch plan (sige_tile_conv_plan_t) of a FusedConv: the kernel and grid its launch uses."""
    import ctypes

    from . import _cabi

    pl = _cabi.TileConvPlan()
    _cabi.check(_cabi.lib().sige_tile_conv_plan(ctypes.byref(fc.desc), ctypes.byref(pl)), "sige_tile_conv_plan")
    return pl


def kernel_name(pl) -> str:
    """'wgmma bn=<BN> ksplit=<K>' or 'mma.sync bn=<BN> ksplit=<K> grid=<X>x<Y>' for a plan_of() result."""
    if pl.path == 1:
        return "wgmma bn=%d ksplit=%d" % (pl.bn, pl.ksplit)
    return "mma.sync bn=%d ksplit=%d grid=%dx%d" % (pl.bn, pl.ksplit, pl.grid_x, pl.grid_y)


def _traced_step(model, args, options):
    """A fused, graph-captured step whose wgmma launches stamp %globaltimer per CTA (16 slots each) into a device buffer:
    (step, plans, ctas, offs, buf) with offs[i] the first slot of launch i (ctas[i] == 0: not a wgmma launch)."""
    from . import _cabi
    from .fused import FusedConv, FusedStep

    lib = _cabi.lib()
    dev = args[0].device
    order = {}

    # pass 1 (no trace): learn the grids, size the trace buffer
    opts = dict(options)
    opts.pop("use_graph", None)
    with torch.no_grad():
        probe = FusedStep(model, *args, use_graph=False, **opts)
    plans = [plan_of(f) for f in probe.fused]
    ctas = [pl.grid_x * pl.grid_y * pl.grid_z if pl.path == 1 else 0 for pl in plans]
    offs, tot = [], 0
    for c in ctas:
        offs.append(tot)
        tot += c * 16
    del probe
    buf = torch.zeros(max(tot, 16), dtype=torch.int64, device=dev)

    def hook(fc):
        i = order.setdefault(id(fc), len(order))
        lib.sige_debug_set_trace(buf.data_ptr() + offs[i] * 8 if (i < len(offs) and ctas[i] > 0) else None)

    FusedConv.trace_hook = hook
    try:
        with torch.no_grad():
            step = FusedStep(model, *args, use_graph=True, **opts)
    finally:
        FusedConv.trace_hook = None
        lib.sige_debug_set_trace(None)
    assert len(step.fused) == len(ctas)
    return step, plans, ctas, offs, buf


def measure_in_graph(model, args, options, flush, reps: int = 5):
    """IN-STEP roofline of the dominant kernel (tc5::tile_conv_tc5_kernel): a second fused step is built whose wgmma
    launches stamp %globaltimer per CTA into a trace buffer (pointer baked into the captured kernel parameters), the
    CUDA graph is replayed after an L2 flush, and per launch  start = the first CTA whose dependency resolved
    (griddepcontrol.wait returned), end = last CTA's exit.
    Programmatic dependent launch lets a layer's prologue overlap its predecessor, so the time CHARGED to launch i is its
    exclusive part  end_i - max(start_i, end_{i-1})  — the charges add up to the union of the kernel's intervals, which is
    <= the step time by construction.  achieved = sum(algorithmic bytes of those launches) / sum(charged time)."""
    dev = args[0].device
    step, _, ctas, offs, buf = _traced_step(model, args, options)
    charged = [0.0] * len(ctas)
    first_last = []
    for r in range(reps):
        buf.zero_()
        if flush is not None:
            flush.fill_(r)
        torch.cuda.synchronize(dev)
        step.replay()
        torch.cuda.synchronize(dev)
        host = buf.cpu()
        iv = []
        for i, f in enumerate(step.fused):
            if ctas[i] == 0:
                continue
            t = host[offs[i]:offs[i] + ctas[i] * 16].view(ctas[i], 16)
            # slot 3 = this CTA's dependency has resolved (griddepcontrol.wait returned) and its gather loads are issued: the
            # prologue before it (barrier init, weight prefetch) overlaps the PREDECESSOR under PDL and is not
            # charged; slot 11 = CTA exit
            st, en = t[:, 3][t[:, 3] > 0], t[:, 11][t[:, 11] > 0]
            if st.numel() and en.numel():
                iv.append((int(st.min()), int(en.max()), i))
        iv.sort()
        prev_end = 0
        for st, en, i in iv:
            charged[i] += max(0, en - max(st, prev_end)) / 1e3 / reps          # us
            prev_end = max(prev_end, en)
        if iv:
            first_last.append((iv[-1][1] - iv[0][0]) / 1e3)
    traced = [i for i in range(len(ctas)) if ctas[i] > 0 and charged[i] > 0]
    if not traced:
        raise RuntimeError("in-graph roofline: none of the %d wgmma launches of the step left an entry (slot 3) and exit (slot 11) "
                           "stamp in the trace buffer" % sum(1 for c in ctas if c > 0))
    tot_us = sum(charged[i] for i in traced)
    tot_bytes = float(sum(step.fused[i].bytes for i in traced))
    tot_flops = float(sum(step.fused[i].flops for i in traced))
    pk = peaks()
    achieved = tot_bytes / (tot_us * 1e-6) / 1e9
    slow = sorted(traced, key=lambda i: -charged[i])[:5]
    return {
        "bound": "hbm", "achieved": achieved, "peak": pk["hbm_gbs"], "unit": "GB/s", "frac": achieved / pk["hbm_gbs"],
        "traffic": None,
        "kernel": "sige::tc5::tile_conv_tc5_kernel (%d of the %d fused gather-conv-scatter launches of one step%s)" % (
            len(traced), len(ctas), "" if len(traced) == len(ctas) else "; the rest run on mma.sync"),
        "launches": len(traced), "avg_launch_us": tot_us / max(1, len(traced)), "sum_in_graph_us": tot_us,
        "first_start_to_last_end_us": sorted(first_last)[len(first_last) // 2] if first_last else None,
        "algorithmic_bytes_per_launch": tot_bytes / max(1, len(traced)), "algorithmic_bytes_per_step": float(step.algorithmic_bytes()),
        "peak_source": pk["source"],
        "tensor": {"achieved_tflops": tot_flops / (tot_us * 1e-6) / 1e12 if tot_us else 0.0, "peak_tflops": pk["bf16_tflops"],
                   "frac": (tot_flops / (tot_us * 1e-6) / 1e12 / pk["bf16_tflops"]) if tot_us else 0.0},
        "slowest": [{"layer": step.fused[i].name, "us": charged[i], "tiles": step.fused[i].tiles,
                     "GBps": step.fused[i].bytes / (charged[i] * 1e-6) / 1e9} for i in slow],
        "method": "in-graph %%globaltimer stamps (first CTA past its dependency .. last CTA exit per launch), L2 flushed before the replay, "
                  "overlap with the predecessor (PDL prologue) charged once; median-free mean of %d replays" % reps,
    }


STAGES = (("dep_to_first_halo", 3, 5), ("mainloop", 5, 6), ("exchange", 6, 9), ("epilogue", 9, 11))


def stage_breakdown(model, args, options, flush, reps: int = 5):
    """Where the time of each wgmma launch of the traced step goes, from the per-CTA %globaltimer stamps of the kernel:
    for every fused launch the median over CTAs and replays (L2 flushed before each) of
      dep_to_first_halo  slot 3 -> 5   dependency resolved, gather issued -> first halo buffer full
      mainloop           slot 5 -> 6   first halo full -> last MMA retired
      exchange           slot 6 -> 9   split-K partial rows pushed and received (un-split: accumulator staging)
      epilogue           slot 9 -> 11  bias / residual / stores -> CTA exit
    in microseconds, with the layer name, the launch plan and the halo fills of each K rank (slot 12: the most
    fills any CTA of that rank consumed; None when the library does not record it)."""
    step, plans, ctas, offs, buf = _traced_step(model, args, options)
    dev = args[0].device
    samples = [{name: [] for name, _, _ in STAGES} for _ in ctas]
    fills = [None] * len(ctas)
    for r in range(reps):
        buf.zero_()
        if flush is not None:
            flush.fill_(r)
        torch.cuda.synchronize(dev)
        step.replay()
        torch.cuda.synchronize(dev)
        host = buf.cpu()
        for i, n in enumerate(ctas):
            if n == 0:
                continue
            t = host[offs[i]:offs[i] + n * 16].view(n, 16)
            live = (t[:, 3] > 0) & (t[:, 11] > 0)          # padding CTAs exit before their first stamp
            for name, a, b in STAGES:
                samples[i][name] += ((t[live, b] - t[live, a]).double() / 1e3).tolist()
            f = t[:, 12].view(plans[i].grid_z, -1).max(dim=1).values
            if int(f.max()) > 0:
                fills[i] = [int(v) for v in f]
    out = []
    for i, f in enumerate(step.fused):
        if ctas[i] == 0:
            continue
        pl = plans[i]
        med = {name: (float(torch.tensor(v).median()) if v else None) for name, v in samples[i].items()}
        out.append({"layer": f.name, "tiles": f.tiles, "bn": pl.bn, "ksplit": pl.ksplit, "deep_ring": pl.deep_ring,
                    "grid": [pl.grid_x, pl.grid_y, pl.grid_z], "halo_fills_per_rank": fills[i], "us": med})
    return out
