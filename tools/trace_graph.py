"""In-graph timeline of the fused DDPM step: every wgmma fused launch stamps globaltimer into its own trace
buffer (pointer captured with the kernel parameters), the CUDA graph is replayed, and the start/end of each kernel
plus the gaps between consecutive kernels are printed.  Development aid, GPU only."""
import ctypes, os, sys, warnings
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO); sys.path.insert(0, os.path.join(REPO, "baseline"))
import torch
import loader
from sige_b200 import _cabi
from sige_b200.fused import FusedConv, FusedStep
from sige_b200.masks import downsample_mask
from sige_b200.workloads.ddpm import DDPMConfig, SIGEDDPMUNet, init_deterministic, synthetic_inputs

dev = torch.device("cuda", 0)
cfg = DDPMConfig()
with warnings.catch_warnings():
    warnings.simplefilter("ignore")
    net = loader.reference_ddpm_on_this_repo(cfg) if loader.available() else SIGEDDPMUNet(cfg)
    model = init_deterministic(net, seed=0).eval().to(dev)       # fp32 model + fp32 dense pass, fp16 fused sparse step (bench.py's flow)
ratio = 0.012
for a in sys.argv[1:]:
    if a.startswith("--ratio="):
        ratio = float(a.split("=")[1])
n_edits = 1
for a in sys.argv[1:]:
    if a.startswith("--edits="):
        n_edits = int(a.split("=")[1])
edit_x, edit_masks = [], []
for e in range(n_edits):            # the batch of bench.py --edits N
    x0, x1e, mask_e, t = synthetic_inputs(cfg, ratio, seed=0, edit_seed=e)
    if e > 0:
        g = torch.Generator().manual_seed(1000 + e)
        shift = tuple(int(v) for v in torch.randint(-96, 97, (2,), generator=g))
        mask_e = torch.roll(mask_e, shift, (0, 1))
        x1e = x0 + torch.roll(x1e - x0, shift, (2, 3))
    edit_x.append(x1e)
    edit_masks.append(mask_e)
x1 = torch.cat(edit_x, 0)
cl = lambda a: a.to(dev)
with torch.no_grad():
    model.set_mode("full"); model(cl(x0), t.to(dev))
    if n_edits == 1:
        model.set_masks(downsample_mask(edit_masks[0].to(dev), min_res=8))
    else:
        from sige_b200.masks import stack_mask_pyramids
        model.set_masks(stack_mask_pyramids([downsample_mask(m.to(dev), min_res=8) for m in edit_masks]))
    model.set_mode("sparse")
lib = _cabi.lib()
SLOT = 1024 * 16
buf = torch.zeros(200 * SLOT, dtype=torch.int64, device=dev)
order = {}
def hook(fc):
    i = order.setdefault(id(fc), len(order))
    lib.sige_debug_set_trace(buf.data_ptr() + i * SLOT * 8)
FusedConv.trace_hook = hook
eng = FusedStep(model, cl(x1), t.to(dev), use_graph=True, dtype=torch.float16, tc5=True, pdl="--no-pdl" not in sys.argv, fused_attention="--no-fused-attention" not in sys.argv)
FusedConv.trace_hook = None
lib.sige_debug_set_trace(None)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
for _ in range(3):
    flush.fill_(1); eng.replay()
buf.zero_(); flush.fill_(2); torch.cuda.synchronize()
eng.replay(); torch.cuda.synchronize()
names = {order[id(f)]: f.name for f in eng.fused if id(f) in order}
tt = buf.view(200, 1024, 16).cpu()
rows = []
for i in sorted(names):
    t_ = tt[i]; t_ = t_[t_[:, 0] > 0]
    if t_.shape[0] == 0:
        continue
    st, en = int(t_[:, 0].min()), int(t_[:, 11][t_[:, 11] > 0].max()) if (t_[:, 11] > 0).any() else int(t_.max())
    gather_done = float(torch.median(t_[:, 4][t_[:, 4] > 0].float())) if (t_[:, 4] > 0).any() else 0
    rows.append((st, en, names[i], t_.shape[0], gather_done))
rows.sort()
t0 = rows[0][0]
prev_end = t0
busy = 0
for st, en, name, n, gd in rows:
    print("%-28s ctas %3d start %8.2f dur %6.2f gap-from-prev-end %6.2f" % (name, n, (st - t0) / 1e3, (en - st) / 1e3, (st - prev_end) / 1e3))
    busy += en - st
    prev_end = max(prev_end, en)
stage_names = ["start", "setup", "idx", "ldg", "store", "mmaA", "mmaEnd", "accOut", "rowsIn", "reduce", "stored", "end"]
print("--- in-graph stage medians (us after the kernel's own first CTA start) for selected layers")
for i in sorted(names):
    nm = names[i]
    if not any(k in nm for k in ("down.0.block.1", "mid.block_1", "up.4.block.1", "up.0.block.1", "up.4.attn.1")):
        continue
    t_ = tt[i]; t_ = t_[t_[:, 0] > 0]
    if t_.shape[0] == 0:
        continue
    rel = (t_ - t_[:, 0].min()).float(); rel[t_ == 0] = float("nan")
    med = [float(torch.nanmedian(rel[:, k])) / 1e3 for k in range(12)]
    print("%-28s " % nm + " ".join("%s %.1f" % (a, b) for a, b in zip(stage_names[1:], med[1:])))
if "--detail" in sys.argv:
    print("--- absolute in-graph stamps (us after the first kernel start): start(min) | wait released+loads issued | halo stored | MMA issued | acc ready | cluster sync | stored(max) | end(max)")
    det = []
    for i in sorted(names):
        t_ = tt[i]; t_ = t_[t_[:, 0] > 0]
        if t_.shape[0] == 0:
            continue
        def med(k):
            v = t_[:, k][t_[:, k] > 0]
            return (float(torch.median((v - t0).double())) / 1e3) if v.numel() else float("nan")
        def mx(k):
            v = t_[:, k][t_[:, k] > 0]
            return (float((v - t0).double().max()) / 1e3) if v.numel() else float("nan")
        det.append((int(t_[:, 0].min()), "%-28s n%3d | %8.2f | %8.2f %8.2f %8.2f %8.2f %8.2f | %8.2f %8.2f" %
                    (names[i], t_.shape[0], (int(t_[:, 0].min()) - t0) / 1e3, med(3), med(4), med(6), med(7), med(8), mx(10), mx(11))))
    for _, line in sorted(det):
        print(line)
if "--spread" in sys.argv:
    print("--- per-launch spread over CTAs (us after the first kernel start): released min/med/max | acc ready min/med/max | exchange done min/med/max | stored min/med/max")
    for i in sorted(names):
        t_ = tt[i]; t_ = t_[t_[:, 0] > 0]
        if t_.shape[0] == 0:
            continue
        def mmm(k):
            v = t_[:, k][t_[:, k] > 0]
            if not v.numel():
                return "   nan    nan    nan"
            v = (v - t0).double() / 1e3
            return "%7.2f %7.2f %7.2f" % (float(v.min()), float(v.median()), float(v.max()))
        print("%-28s n%3d | %s | %s | %s | %s" % (names[i], t_.shape[0], mmm(3), mmm(7), mmm(8), mmm(10)))
print("first start -> last end: %.1f us; sum of kernel durations %.1f us over %d traced launches" % ((prev_end - t0) / 1e3, busy / 1e3, len(rows)))
