"""Which launches of a compiled fused step may run at the same time, and what each reads before it waits for its predecessor: a
model of programmatic dependent launch (PDL) restated from the kernel sources, checked on a program without running it.

A launch made with the PDL attribute may start before its predecessor has finished.  Until its `griddepcontrol.wait` it reads
only what the lowering promises is already final; after the wait every earlier launch of the stream has completed.  For every
entry of a program the model states:

  * `kernel`: the kernel that runs it ("wgmma" / "mma.sync" tile conv, decided by `sige_tile_conv_plan` as
    `CudaExecutor.takes_wgmma` does; "separable", "attention", "conv_in", the tail's "gn_partial", "gn_finalize" and "conv_out",
    "sparse_attention", "spade", "writeback", "cache_load"; "eager" for a recorded torch call or copy);
  * `pdl`: launched with the attribute (conv_in and the tail always, dense_glue.cu:504-505,536-537,577-578,605; sparse
    attention, SPADE, write-back, cache load and torch calls never);
  * `releases_first`: it releases its dependents before it waits itself (every PDL kernel but the wgmma tile conv);
  * `reads`: the operand views it reads before its wait;
  * `writes`: the views of its record's destinations.

The window W(L) of a PDL launch L is its predecessor P (when P is a kernel of this project: a recorded torch call triggers its
dependents only when it has completed), plus W(P) when P releases first.  A launch without the attribute starts after its
predecessor has completed: its window is empty.  The check: no pre-wait read of L shares a 128-byte line with a write of a
launch of W(L).  Lines rather than bytes because the early reads go through `ld.global.nc`, whose lines the wait is not known to
drop.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import torch

LINE = 128


# ----------------------------------------------------------------------------------------------------------------------
# a simulator with the product executor's descriptors: the lowering then asks sige_tile_conv_plan which kernel each conv takes
# ----------------------------------------------------------------------------------------------------------------------
def _describer(dtype):
    from sige_b200.fused import CudaExecutor

    class Describer(CudaExecutor):
        """CudaExecutor.prepare_conv without a device: the descriptor of every launch, its packed weights left unpacked."""

        def __init__(self):
            from sige_b200 import ops

            self.ops, self.device, self.dtype = ops, torch.device("cpu"), dtype

        def _pack(self, w, key, pad_cin=0):
            return torch.empty((w.shape[2] * w.shape[3], w.shape[0], max(pad_cin, w.shape[1])), dtype=self.dtype)

    return Describer()


class PlannedMixin:
    """Put in front of a simulator class: every prepared conv also gets the descriptor the product executor would launch, and
    `takes_wgmma` answers from the host plan of that descriptor (an H100's plan without a device), so `Lowering._post` drops
    the early marks after an mma.sync launch here as it does on the GPU."""

    plan_dtype = torch.float16

    @property
    def ops(self):
        from sige_b200 import ops

        return ops

    def prepare_conv(self, fc):
        super().prepare_conv(fc)
        run = fc.launch_fn
        _describer(self.plan_dtype).prepare_conv(fc)
        fc.launch_fn = run

    def takes_wgmma(self, fc) -> bool:
        return plan_path(fc) == 1


def planned(base: type) -> type:
    return type("Planned" + base.__name__, (PlannedMixin, base), {})


def plan_path(fc) -> int:
    """1: the wgmma kernel runs the launch, 0: the mma.sync kernel (sige_tile_conv_plan of its descriptor)."""
    from sige_b200 import _cabi

    pl = _cabi.TileConvPlan()
    _cabi.check(_cabi.lib().sige_tile_conv_plan(ctypes.byref(fc.desc), ctypes.byref(pl)), "sige_tile_conv_plan")
    return int(pl.path)


# ----------------------------------------------------------------------------------------------------------------------
# the entries of a program
# ----------------------------------------------------------------------------------------------------------------------
Views = List[Tuple[str, torch.Tensor]]


@dataclass
class Entry:
    program: str
    pos: int
    name: str
    kernel: str
    pdl: bool
    releases_first: bool
    reads: Views = field(default_factory=list)
    writes: Views = field(default_factory=list)
    early: int = 0

    @property
    def label(self) -> str:
        return "%s launch %d (%s, %s)" % (self.program, self.pos, self.name, self.kernel)


def _views(pairs) -> Views:
    return [(n, t) for n, t in pairs if isinstance(t, torch.Tensor)]


def early_groups(s) -> List[Views]:
    """The reads of each source group of a tile conv's K loop (bit g of `early`): src[0] and src[1] with the gather's pre-op
    (scale, shift, SPADE's gamma and beta), the fused shortcut's sources."""
    pre = [("scale", s.scale), ("shift", s.shift)]
    if s.modulation is not None:
        pre += [("gamma", s.modulation[0]), ("beta", s.modulation[1])]
    groups = [_views([("src%d" % i, t)] + pre) for i, (t, _) in enumerate(s.srcs[:2])]
    groups += [[] for _ in range(2 - len(groups))]
    groups.append(_views(("shortcut src%d" % i, t) for i, t in enumerate(s.shortcut[0])) if s.shortcut is not None else [])
    return groups


def conv_writes(s, writes_raw: bool) -> Views:
    out = _views([("dst_stack", s.dst_stack)])
    if s.dst is not None and writes_raw:
        out += [("dst", s.dst.raw)]
    out += [("aux%d" % i, a[0]) for i, a in enumerate(s.aux)]
    return out


def conv_entry(program: str, pos: int, fc, writes_raw: bool) -> Entry:
    from sige_b200._cabi import CONV_PADDED

    s = fc.spec
    wgmma = plan_path(fc) == 1
    sc = s.shortcut
    if wgmma:
        # tile_conv_tc5.cu:439 (the padding exit) and 476-490: the tile list and the shortcut flags; 491-497: bias, the aux
        # destinations' scale / shift, bias2; the packed weights' TMA stream, started before the wait; then the early groups'
        # chunks (KOrder) up to the wait at 642-650
        reads = _views([("idx", s.idx), ("sc_flags", None if sc is None else sc[3]), ("bias", s.bias), ("bias2", None if sc is None else sc[2])])
        for i, (_, a_sc, a_sh, _) in enumerate(s.aux):
            reads += _views([("aux%d scale" % i, a_sc), ("aux%d shift" % i, a_sh)])
        reads += _views([("weight", s.weight), ("shortcut weight", None if sc is None else sc[1])])
        for g, views in enumerate(early_groups(s)):
            if (s.early >> g) & 1:
                reads += [("early group %d %s" % (g, n), t) for n, t in views]
    else:
        # tile_conv_mma.cu:130 (the padding exit reads the first list row) and 280-284 (the weight stages before the wait at 286)
        reads = _views([("weight", s.weight)] + ([("idx", s.idx)] if fc.desc.flags & CONV_PADDED else []))
    return Entry(program, pos, fc.name, "wgmma" if wgmma else "mma.sync", bool(s.pdl), bool(s.pdl) and not wgmma, reads,
                 conv_writes(s, writes_raw), int(s.early))


def entries(step, program=None, name: str = "main") -> List[Entry]:
    """The model of every entry of `program` (default: the step's main program).  The step's executor must be a recording one
    (fused_step_contract.recording) whose conv launches carry descriptors (`planned`, or the product executor)."""
    program = step.steps if program is None else program
    ex = step.ex
    out: List[Entry] = []
    for pos, (kind, fn) in enumerate(program):
        if kind == "eager":
            out.append(Entry(name, pos, "eager", "eager", False, False))
            continue
        rec = ex.record_of(kind, fn)
        if kind == "conv":
            fc = fn.__self__
            out.append(conv_entry(name, pos, fc, ex.writes_raw(fc)))
        elif kind == "separable":
            # separable_conv.cu:73-89: the 1x1 weights, the depthwise weights and bias before the wait at 90-91
            reads = []
            for b, (dwc, w1, _b1, _buf) in enumerate(rec.branches):
                reads += _views([("branch%d depthwise weight" % b, dwc.weight), ("branch%d depthwise bias" % b, dwc.bias), ("branch%d weight" % b, w1)])
            out.append(Entry(name, pos, rec.name, "separable", bool(rec.pdl), bool(rec.pdl), reads if rec.pdl else [],
                             [("branch%d dst" % b, br[3].raw) for b, br in enumerate(rec.branches)]))
        elif kind == "attention":
            # attention.cu:78-85: barrier set-up only before the wait
            out.append(Entry(name, pos, "attention", "attention", bool(rec["pdl"]), bool(rec["pdl"]), [], [("out", rec["out"])]))
        elif kind == "conv_in":
            # dense_glue.cu:49,60 (conv_in) / 151,162 (conv_in on tiles): the weights and bias before the wait at 63 / 165
            writes = ([("out", rec.out.raw)] if rec.out.has_raw else []) + [("aux%d" % i, a[0]) for i, a in enumerate(rec.aux)]
            out.append(Entry(name, pos, "conv_in", "conv_in", True, True, _views([("weight", rec.weight), ("bias", rec.bias)]), writes))
        elif kind == "tail":
            # dense_glue.cu:232-233, 281-282: GroupNorm's partial sums and fold read nothing before their wait and write the
            # launch's own workspace and (scale, shift), which nothing else reads; 354, 367-368: conv_out stages its weights first
            out.append(Entry(name, pos, "tail", "gn_partial", True, True))
            out.append(Entry(name, pos, "tail", "gn_finalize", True, True))
            out.append(Entry(name, pos, "tail", "conv_out", True, True, _views([("weight", rec["weight"])]), [("out", rec["out"])]))
        elif kind == "sparse_attention":
            out.append(Entry(name, pos, "sparse_attention", "sparse_attention", False, False, [], [("out", rec["out"])]))
        elif kind == "spade":
            out.append(Entry(name, pos, "spade", "spade", False, False, [], [("out", rec["out"])]))
        elif kind == "writeback":
            out.append(Entry(name, pos, "writeback", "writeback", False, False, [], [("cache%d" % i, e[1]) for i, e in enumerate(rec)]))
        elif kind == "cache_load":
            ws: Views = []
            for i, (_src, raw, views) in enumerate(rec):
                ws += _views([("raw%d" % i, raw)]) + [("view%d.%d" % (i, j), v[0]) for j, v in enumerate(views)]
            out.append(Entry(name, pos, "cache_load", "cache_load", False, False, [], ws))
        else:
            raise AssertionError("%s entry %d: no model for launch kind %r" % (name, pos, kind))
    return out


def load_entries(step) -> List[Entry]:
    """The cache load of a new edit (`Lowering.load_caches`): the prepared `sige_cache_load`, then the torch restores."""
    run, rest = step.low.prepared_loader()
    program = ([("cache_load", run)] if run is not None else []) + [("eager", None) for _ in rest]
    return entries(step, program, "loads")


# ----------------------------------------------------------------------------------------------------------------------
# windows and the check
# ----------------------------------------------------------------------------------------------------------------------
def windows(seq: Sequence[Entry]) -> List[List[int]]:
    out: List[List[int]] = []
    for i, e in enumerate(seq):
        if i == 0 or not e.pdl:
            out.append([])
            continue
        p = seq[i - 1]
        out.append(([] if p.kernel == "eager" else [i - 1]) + (out[i - 1] if p.releases_first else []))
    return out


def _key(t: torch.Tensor):
    return (t.device.type, t.untyped_storage().data_ptr())


class _Lines:
    """Per view: bool over the 128-byte lines of its storage, True where the view has a byte."""

    def __init__(self):
        self.cache: Dict[tuple, torch.Tensor] = {}

    def __call__(self, t: torch.Tensor) -> torch.Tensor:
        k = (_key(t), t.storage_offset(), tuple(t.shape), tuple(t.stride()), t.element_size())
        hit = self.cache.get(k)
        if hit is None:
            nb = t.untyped_storage().nbytes()
            es = t.element_size()
            n_lines = -(-nb // LINE)
            elem = torch.zeros(n_lines * LINE // es, dtype=torch.bool, device=t.device)
            if t.numel():
                elem.as_strided(t.shape, t.stride(), t.storage_offset()).fill_(True)
            hit = elem.view(n_lines, LINE // es).any(1)
            self.cache[k] = hit
        return hit


def hazards(seq: Sequence[Entry], names: Optional[Dict[tuple, str]] = None, first: bool = False) -> List[str]:
    """Every (L, operand, M, line) where a pre-wait read of L shares a 128-byte line with a write of M in W(L)."""
    lines = _Lines()
    names = names or {}
    found: List[str] = []
    for i, (e, w) in enumerate(zip(seq, windows(seq))):
        for op, view in e.reads:
            for j in w:
                m = seq[j]
                for wn, wv in m.writes:
                    if _key(wv) != _key(view):
                        continue
                    both = lines(view) & lines(wv)
                    if bool(both.any()):
                        at = int(both.nonzero()[0]) * LINE
                        found.append("%s reads %s before its wait, which %s may still be writing (%s): %s, line at byte %d (%d shared lines)"
                                     % (e.label, op, m.label, wn, names.get(_key(view), "storage %#x" % _key(view)[1]), at, int(both.sum())))
                        if first:
                            return found
    return found


def check(seq: Sequence[Entry], names: Optional[Dict[tuple, str]] = None) -> None:
    bad = hazards(seq, names)
    if bad:
        raise AssertionError("%d PDL hazards; the first: %s" % (len(bad), bad[0]))


def storage_names(step, model=None) -> Dict[tuple, str]:
    import fused_step_contract as fsc

    return {k: s.name for k, s in fsc.State(step, model).storages.items()}


@dataclass
class Stats:
    launches: int
    pdl: int
    releases_first: int
    deepest: int
    deepest_at: str
    early: int
    early_groups: int

    def __str__(self) -> str:
        return ("%d launches, %d PDL, %d release first, deepest window %d (at %s), %d launches with early groups (%d groups)"
                % (self.launches, self.pdl, self.releases_first, self.deepest, self.deepest_at, self.early, self.early_groups))


def stats(seq: Sequence[Entry]) -> Stats:
    ws = windows(seq)
    deep = max(range(len(seq)), key=lambda i: len(ws[i])) if seq else 0
    return Stats(sum(1 for e in seq if e.kernel != "eager"), sum(1 for e in seq if e.pdl), sum(1 for e in seq if e.releases_first),
                 len(ws[deep]) if seq else 0, seq[deep].label if seq else "-", sum(1 for e in seq if e.early),
                 sum(bin(e.early).count("1") for e in seq))


def sequences(step) -> Dict[str, List[Entry]]:
    """The sequences a step's programs form on a stream without a graph boundary: the main program after itself (`run_eager`
    twice), the main program then the sparse_update epilogue's first (eager) run, the cache load of a new edit then the main
    program."""
    main = entries(step)
    again = entries(step, name="main, next call")
    out = {"main then main": main + again}
    if getattr(step, "sparse_update_supported", False):
        out["main then sparse_update"] = main + entries(step, step.low.epilogue, "sparse_update")
    if step.low.cached_bufs:
        out["loads then main"] = load_entries(step) + main
    return out


def verify(step, tag: str, model=None) -> Dict[str, Stats]:
    """Check every sequence of the step; print its statistics; return them per sequence."""
    names = storage_names(step, model)
    res = {}
    for what, seq in sequences(step).items():
        check(seq, names)
        res[what] = stats(seq)
        print("[pdl hazards] %s, %s: %s" % (tag, what, res[what]))
    return res
