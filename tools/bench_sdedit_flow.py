"""The reference samplers' per-step flow at DDPM-256: a dense pass on the original and a sparse pass on the edit at every
denoising step (diffusion/samplers/ddim_ddpm_sampler.py `model_step`), three arms alternated step by step in one process:

    eager      the eager operator modules
    recompile  fused, every compiled step dropped before each sparse call (what a new dense pass cost before refresh)
    refresh    fused, the compiled step takes each dense pass in place (FusedStep.refresh)

    python tools/bench_sdedit_flow.py [--steps 20] [--ratio 0.012] [--model reference|intree] [--out DIR]

Per arm and step: synchronised wall time of the whole model_step; device time (CUDA events) of the dense pass, of the refresh
(refresh arm) and of the sparse call; the host time of enqueueing the dense pass, the cudaMalloc calls it caused and the Python
garbage collections during the step; the refresh's algorithmic bytes (every cache read once, every raw copy and view written
for each edit) over its device time, against the H100 SXM data-sheet 3.35 TB/s.  Prints one JSON line; writes each arm's
final eps to DIR/eps_<arm>.pt.  The card name, power limit and SM clock are read in the same run.
"""
import argparse
import gc
import json
import os
import subprocess
import sys
import tempfile
import time
import warnings

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "baseline"))
HBM_BYTES_PER_S = 3.35e12


def _card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]))
    except (OSError, IndexError, subprocess.TimeoutExpired):
        return {"name": torch.cuda.get_device_name(0)}


def _model(kind, cfg):
    import loader
    from sige_b200.workloads.ddpm import SIGEDDPMUNet, init_deterministic

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if kind == "reference":
            if not loader.available():
                raise SystemExit("baseline/_ref absent: python baseline/build_ref.py")
            m = loader.reference_ddpm_on_this_repo(cfg)
        else:
            m = SIGEDDPMUNet(cfg)
        return init_deterministic(m, seed=0).eval().cuda()


def _refresh_bytes(step):
    """Bytes the refresh must move at least: each cache read once, each raw copy and view written."""
    n = 0
    for b in step.low.cached_bufs:
        c = b.cached_init
        n += c.numel() * c.element_size()
        per = b.shape[0] * b.shape[1] * b.shape[2] * b.shape[3] * torch.finfo(step.dtype).bits // 8
        n += per * ((1 if b.has_raw else 0) + len(b.view_inits))
    return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ratio", type=float, default=0.012)
    ap.add_argument("--model", default="reference", choices=["reference", "intree"])
    ap.add_argument("--out", default=None)
    ap.add_argument("--arms", default="eager,recompile,refresh",
                    help="comma-separated subset; the recompile arm's graph captures empty the caching allocator, which the others then refill")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sdedit_flow: needs a GPU")
    from sige.utils import downsample_mask
    from sige_b200.workloads.ddpm import DDPMConfig, synthetic_inputs

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = DDPMConfig()
    x0, x1, mask, t0 = synthetic_inputs(cfg, a.ratio, seed=0)
    arms = {k: _model(a.model, cfg) for k in a.arms.split(",")}
    for k, m in arms.items():
        m.set_fused(k != "eager", dtype=torch.float16)
    for m in arms.values():
        with torch.no_grad():
            m.set_mode("full")
            m(x0.cuda(), t0.cuda())
            m.set_masks(downsample_mask(mask.cuda(), min_res=8))
    rec = {k: {"wall_ms": [], "dense_ms": [], "dense_host_ms": [], "refresh_ms": [], "sparse_ms": [], "dense_device_allocs": [],
               "gc_collections": []} for k in arms}
    refresh_bytes = None
    eps = {}
    for s in range(a.warmup + a.steps):
        g = torch.Generator().manual_seed(s)
        xt = (torch.cat([x0, x1], 0) * (1.0 - 0.02 * s) + 0.05 * torch.randn((2, *x0.shape[1:]), generator=g)).cuda()
        t = (t0 + 40 * s).cuda()
        names = list(arms)
        for k in names[s % len(names):] + names[:s % len(names)]:          # the order rotates every step: no arm always follows the same one
            m = arms[k]
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            torch.cuda.synchronize()
            allocs0, gcs0 = torch.cuda.memory_stats().get("num_device_alloc", 0), sum(st["collections"] for st in gc.get_stats())
            w0 = time.perf_counter()
            with torch.no_grad():
                ev[0].record()
                m.set_mode("full")
                m(xt[:1], t)
                m.set_mode("sparse")
                ev[1].record()
                dense_host = (time.perf_counter() - w0) * 1e3
                allocs = torch.cuda.memory_stats().get("num_device_alloc", 0) - allocs0
                if k == "recompile":
                    m._fused_steps.clear()
                elif k == "refresh":
                    m._fused_lookup((xt[1:], t))
                ev[2].record()
                eps[k] = m(xt[1:], t)
                ev[3].record()
            torch.cuda.synchronize()
            wall = (time.perf_counter() - w0) * 1e3
            if k == "refresh" and refresh_bytes is None and s > 0:
                refresh_bytes = _refresh_bytes(m.fused_step)
            if s >= a.warmup:
                r = rec[k]
                r["wall_ms"].append(wall)
                r["dense_host_ms"].append(dense_host)
                r["dense_device_allocs"].append(allocs)
                r["gc_collections"].append(sum(st["collections"] for st in gc.get_stats()) - gcs0)
                r["dense_ms"].append(ev[0].elapsed_time(ev[1]))
                r["refresh_ms"].append(ev[1].elapsed_time(ev[2]))
                r["sparse_ms"].append(ev[2].elapsed_time(ev[3]))
    assert "refresh" not in arms or arms["refresh"].fused_step.refresh_reason is None

    def med(v):
        v = sorted(v)
        return v[len(v) // 2]

    res = {"card": _card(), "model": a.model, "ratio": a.ratio, "steps": a.steps}
    for k, r in rec.items():
        res[k] = {n: round(med(v), 4) for n, v in r.items()}
    rt = med(rec["refresh"]["refresh_ms"]) / 1e3 if "refresh" in rec else 0
    res["refresh_bytes"] = refresh_bytes
    res["refresh_tb_per_s"] = round(refresh_bytes / rt / 1e12, 3) if refresh_bytes and rt > 0 else None
    res["refresh_share_of_3.35TB/s"] = round(refresh_bytes / rt / HBM_BYTES_PER_S, 3) if refresh_bytes and rt > 0 else None
    if "eager" in eps:
        ref = eps["eager"].float()
        for k in [k for k in eps if k != "eager"]:
            res["max_err_vs_eager_" + k] = float((eps[k].float() - ref).abs().max() / ref.abs().max())
    if "refresh" in eps and "recompile" in eps:
        res["refresh_equals_recompile"] = bool(torch.equal(eps["refresh"], eps["recompile"]))
    out = a.out or tempfile.mkdtemp(prefix="sdedit_flow_")
    os.makedirs(out, exist_ok=True)
    for k, v in eps.items():
        torch.save(v.cpu(), os.path.join(out, "eps_%s.pt" % k))
    res["eps_dir"] = out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
