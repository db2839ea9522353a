"""Time the apply step of an incremental edit (the reference's editing demo) on one GPU: eager operator modules against the fused
step with its sparse_update epilogue.

    python tools/bench_incremental_edit.py [--cache-ids 10] [--ratio 0.012] [--repeats 5] [--warmup 2] [--headroom 1.0]
                                           [--json PATH]

The demo's flow at full size (reference diffusion_demo/runner.py:134-141, samplers/dpm_solver_sampler.py:116-120): DDPM-256 (the
reference's model file through baseline/loader.py when its install is present, else the in-tree restatement), an fp32 model, one
dense pass per cache id along a DPM-solver-like t sequence ending at 750, then edits previewed and applied with sparse_update=True.
Two edits: the 1.2 % centred square, then a second edit shifted by 24 pixels applied on top of the first.  Two models with the same
weights and dense passes run side by side: `eager` (set_fused(False): the operator modules, cuDNN, fp32) and `fused`
(set_fused(True, dtype=torch.float16)).

Per edit it reports, over all cache ids (host wall time to a synchronised end, median of --repeats after --warmup, the paths
alternated within each repeat): `eager_apply_ms`, `fused_apply_ms`, `fused_preview_ms` (sparse_update off); per cache id the
epilogue's device time (CUDA events around `FusedStep.sparse_update()`, median) and the fused step's main-program device time
(CUDA events around a replay); `compile_s` (the first fused preview of every id, compilation included) separately; and the
parity of the final outputs and caches, fused against eager (max-normalised).  Applying the same edit again is idempotent, so the
repeated applies time the same work.  The GPU's name, power limit and SM clock are read in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import warnings

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


def make_model(cfg):
    from sige_b200.workloads.ddpm import SIGEDDPMUNet, init_deterministic

    sys.path.insert(0, os.path.join(REPO, "baseline"))
    import loader

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model = loader.reference_ddpm_on_this_repo(cfg) if loader.available() else SIGEDDPMUNet(cfg)
        return init_deterministic(model, seed=0).eval(), type(model).__module__


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--cache-ids", type=int, default=10)
    ap.add_argument("--ratio", type=float, default=0.012)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--headroom", type=float, default=1.0, help="tile-list capacity of the fused steps (the second edit is installed in place)")
    ap.add_argument("--json", default=None, help="also write the result line to this file")
    args = ap.parse_args()

    import torch

    from sige_b200.masks import downsample_mask
    from sige_b200.parallel import cache_tensors
    from sige_b200.workloads.ddpm import DDPMConfig, synthetic_inputs

    if not torch.cuda.is_available():
        raise SystemExit("bench_incremental_edit: needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    info = gpu_info()
    cfg = DDPMConfig()
    ids = list(range(args.cache_ids))
    ts = [round(999 - (999 - 750) * i / max(1, len(ids) - 1)) for i in ids]          # DPM-solver-like, ending at 750
    x0, xa, mask_a, _ = synthetic_inputs(cfg, args.ratio, seed=0, edit_seed=1)
    _, xn, _, _ = synthetic_inputs(cfg, args.ratio, seed=0, edit_seed=2)
    mask_s = torch.roll(mask_a, shifts=(24, 24), dims=(0, 1))
    xb = xa + (xn - x0) * mask_s[None, None].float()                                  # the shifted edit, on top of the first
    edits = [("edit_1", xa, mask_a), ("edit_2_on_top", xb, mask_a | mask_s)]

    models = {}
    for name in ("eager", "fused"):
        m, src = make_model(cfg)
        m = m.to(dev)
        with torch.no_grad():
            m.set_mode("full")
            for i in ids:
                m.set_cache_id(i)
                m((x0 * (1.0 + 0.01 * i)).to(dev), torch.tensor([ts[i]], device=dev))
            m.set_mode("sparse")
        if name == "eager":
            m.set_fused(False)
        else:
            m.set_fused(True, dtype=torch.float16, headroom=args.headroom)
        models[name] = m

    def inputs(x, i):
        return (x * (1.0 + 0.01 * i)).to(dev), torch.tensor([ts[i]], device=dev)

    def run_all(m, x, update):
        m.set_sparse_update(update)
        outs = []
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in ids:
            m.set_cache_id(i)
            outs.append(m(*inputs(x, i)))
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, outs

    def device_ms(fn, n=5):
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
        for a, b in ev:
            a.record()
            fn()
            b.record()
        torch.cuda.synchronize()
        return statistics.median(a.elapsed_time(b) for a, b in ev)

    line = {"workload": "DDPM-256 incremental edit, %d cache ids, t %d..%d" % (len(ids), ts[0], ts[-1]), "model": src, "gpu": info, "edits": []}
    with torch.no_grad():
        for label, x, mask in edits:
            pyr = downsample_mask(mask.to(dev), min_res=8)
            for m in models.values():
                m.set_masks(pyr)
            fused, eager = models["fused"], models["eager"]
            t0 = time.time()
            run_all(fused, x, False)                       # the first preview of every id compiles (or re-binds) its step
            compile_s = time.time() - t0
            rec = {"edit": label, "tiles_at_256": int(fused.fused_step.fused[0].spec.slot.n) if fused.fused_step.fused[0].spec.slot else None,
                   "compile_s": round(compile_s, 3)}
            times = {"eager_apply": [], "fused_apply": [], "fused_preview": []}
            for r in range(args.warmup + args.repeats):
                te, out_e = run_all(eager, x, True)
                tf, out_f = run_all(fused, x, True)
                tp, _ = run_all(fused, x, False)
                if r >= args.warmup:
                    times["eager_apply"].append(te)
                    times["fused_apply"].append(tf)
                    times["fused_preview"].append(tp)
            for k, v in times.items():
                rec[k + "_ms"] = round(statistics.median(v), 3)
                rec[k + "_ms_spread"] = [round(min(v), 3), round(max(v), 3)]
            per_id = []
            fused.set_sparse_update(False)
            for i in ids:
                fused.set_cache_id(i)
                fused(*inputs(x, i))
                st = fused.fused_step
                assert st.sparse_update_supported and st.eager_nodes == [], st.sparse_update_reason
                per_id.append({"id": i, "main_ms": round(device_ms(st.replay), 4), "epilogue_ms": round(device_ms(st.sparse_update), 4),
                               "epilogue_launches": len(st.low.epilogue)})
            rec["per_cache_id"] = per_id
            rec["epilogue_ms_mean"] = round(statistics.mean(p["epilogue_ms"] for p in per_id), 4)
            rec["main_ms_mean"] = round(statistics.mean(p["main_ms"] for p in per_id), 4)
            rec["epilogue_share_of_apply_step"] = round(rec["epilogue_ms_mean"] / (rec["epilogue_ms_mean"] + rec["main_ms_mean"]), 4)
            out_err = max(float((a.float() - b.float()).abs().max() / b.float().abs().max()) for a, b in zip(out_f, out_e))
            ce = dict(cache_tensors(eager))
            cache_err = max(float((v.float() - ce[n].float()).abs().max() / max(float(ce[n].float().abs().max()), 1e-12))
                            for n, v in cache_tensors(fused))
            rec["parity_outputs_max_norm"] = out_err
            rec["parity_caches_max_norm"] = cache_err
            line["edits"].append(rec)
            print("[%s] eager apply %.1f ms, fused apply %.1f ms, fused preview %.1f ms over %d ids; epilogue %.3f ms / main %.3f ms per id; "
                  "compile %.1f s; parity out %.2e caches %.2e" % (label, rec["eager_apply_ms"], rec["fused_apply_ms"], rec["fused_preview_ms"],
                                                                  len(ids), rec["epilogue_ms_mean"], rec["main_ms_mean"], compile_s, out_err, cache_err),
                  file=sys.stderr, flush=True)
    text = json.dumps(line)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            fh.write(text + "\n")
    print(text, flush=True)


if __name__ == "__main__":
    main()
