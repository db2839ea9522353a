"""A compiled fused step (sige_b200.fused), checked launch by launch against float64 restatements of its launch records.

Imported by tests/test_fused_step_contract.py (CPU: the descriptor simulator) and tests/test_gpu_fused_step_contract.py (GPU:
the product executor).  The kernel contracts (tile_conv_contract, kernel_contracts, step_kernel_contracts) check one kernel on
synthetic cases; this checks the PROGRAM a step is made of — what each record means, how the executor turned it into a launch,
and what the launches leave for each other:

  * `recording(Executor)` is the executor with every `prepare_*` remembering the record it was given, keyed by the callable it
    returns (a `conv` step is `FusedConv.launch`: its record is the FusedConv's spec).
  * `state(step)` is every storage the program can touch: buffers and their producer-written views, stacks, static inputs,
    outputs, attention and tail buffers, tile lists, shortcut flags and the module caches, deduplicated by storage.
  * `walk(step, program)` runs the program one entry at a time: the expectation of the entry's record in float64 from the live
    tensors, a snapshot of the whole state, the launch, a synchronise; every element the record writes within its bound and
    every other byte of the whole state bitwise unchanged.  Recorded torch calls and copies (`eager`) run unchecked.  Before
    it, every padding row of a fixed-capacity stack (`poison_padding`) is NaN: a launch that reads one shows NaN in a live
    element, one that writes one a stray byte.
  * `walk_loads(step)` checks the cache load of a new edit (`sige_cache_load`) the same way.

The restatements read the records (ConvSpec, ConvInRec, the tail / attention / SPADE arguments, write-back entries), never the C
descriptors, so a translation error of the executor shows as a wrong element or a stray write of the launch that made it.
"""
from __future__ import annotations

import time
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

import kernel_contracts as kc
import step_kernel_contracts as skc
from tile_conv_contract import ABS, ACC, PRE_ULPS, SWISH_LIP, UNIT_ROUNDOFF, _gather

NONE_BELOW = -20000            # tile origins at or below this are SIGE_TILE_NONE padding of a fixed-capacity list


# ----------------------------------------------------------------------------------------------------------------------
# the recording executor
# ----------------------------------------------------------------------------------------------------------------------
class RecordingMixin:
    """Put in front of an executor class: every prepared launch keeps the record it was made from."""

    def _records(self) -> Dict[int, tuple]:
        return self.__dict__.setdefault("records", {})

    def _keep(self, kind: str, fn, rec):
        self._records()[id(fn)] = (kind, rec, fn)
        return fn

    def prepare_conv(self, fc):
        # whether the launch writes its destination's raw tensor is decided here (a raw tensor exists, or nothing else receives the
        # result): a buffer that only has producer-written views now may get a raw tensor later (the sparse_update epilogue writes
        # it), which this launch then leaves alone
        s = fc.spec
        self._records()[id(fc)] = ("conv", s.dst is not None and (s.dst.has_raw or not s.aux), fc)
        return super().prepare_conv(fc)

    def writes_raw(self, fc) -> bool:
        hit = self._records().get(id(fc))
        assert hit is not None and hit[2] is fc, "conv launch %s was not prepared by the recording executor" % fc.name
        return hit[1]

    def prepare_conv_in(self, rec):
        return self._keep("conv_in", super().prepare_conv_in(rec), rec)

    def prepare_tail(self, x, groups, eps, gamma, beta, act, weight, bias, out):
        return self._keep("tail", super().prepare_tail(x, groups, eps, gamma, beta, act, weight, bias, out),
                          dict(x=x, groups=groups, eps=eps, gamma=gamma, beta=beta, act=act, weight=weight, bias=bias, out=out))

    def prepare_attention(self, qkv_tokens, out_tokens, pdl):
        return self._keep("attention", super().prepare_attention(qkv_tokens, out_tokens, pdl), dict(qkv=qkv_tokens, out=out_tokens, pdl=pdl))

    def prepare_sparse_attention(self, q, k, v, scale, out):
        return self._keep("sparse_attention", super().prepare_sparse_attention(q, k, v, scale, out), dict(q=q, k=k, v=v, scale=scale, out=out))

    def prepare_separable(self, rec):
        return self._keep("separable", super().prepare_separable(rec), rec)

    def prepare_spade(self, x, gamma, beta, slope, out):
        return self._keep("spade", super().prepare_spade(x, gamma, beta, slope, out), dict(x=x, gamma=gamma, beta=beta, slope=slope, out=out))

    def prepare_writeback(self, entries):
        return self._keep("writeback", super().prepare_writeback(entries), list(entries))

    def prepare_cache_load(self, entries):
        return self._keep("cache_load", super().prepare_cache_load(entries), [(src, raw, list(views)) for (src, raw, views) in entries])

    def record_of(self, kind: str, fn):
        if kind == "conv":
            return fn.__self__.spec
        hit = self._records().get(id(fn))
        assert hit is not None and hit[2] is fn and hit[0] == kind, "a %s step was not prepared by the recording executor" % kind
        return hit[1]


def recording(base: type) -> type:
    return type("Recording" + base.__name__, (RecordingMixin, base), {})


# ----------------------------------------------------------------------------------------------------------------------
# the whole state of a step
# ----------------------------------------------------------------------------------------------------------------------
def _tensors(obj, out: List[torch.Tensor], depth: int = 0) -> None:
    if isinstance(obj, torch.Tensor):
        out.append(obj)
    elif isinstance(obj, (list, tuple)) and depth < 4:
        for o in obj:
            _tensors(o, out, depth + 1)
    elif isinstance(obj, dict) and depth < 4:
        for o in obj.values():
            _tensors(o, out, depth + 1)


def _buf_tensors(b, out: List[torch.Tensor]) -> None:
    if b is None:
        return
    if b.has_raw:
        out.append(b.raw)
    out += [v[0] for v in b.views.values()] + [v[0] for v in b.view_inits]
    if b.cached_init is not None:
        out.append(b.cached_init)


def _spec_tensors(s, out: List[torch.Tensor]) -> None:
    out += [t for t, _ in s.srcs] + [s.idx, s.tile_img, s.residual, s.dst_stack, s.scale, s.shift, s.weight, s.bias]
    _buf_tensors(s.dst, out)
    out += [a[0] for a in s.aux]
    if s.shortcut is not None:
        _tensors(s.shortcut, out)
    if s.modulation is not None:
        out += [s.modulation[0], s.modulation[1]]


@dataclass
class Storage:
    name: str
    bytes: torch.Tensor         # uint8 view of the whole storage


class State:
    """Every storage a step's program can touch, as uint8 views; `snapshot()` / `restore()` / `diff()` over all of them."""

    def __init__(self, step, model=None):
        from sige_b200.fused import Buf, Full

        low = step.low
        found: List[Tuple[str, torch.Tensor]] = []

        def add(name, ts):
            found.extend((name, t) for t in ts if isinstance(t, torch.Tensor))

        for v in low.env.values():
            if isinstance(v, Full):
                for b, _ in v.segs:
                    ts: List[torch.Tensor] = []
                    _buf_tensors(b, ts)
                    add("buffer %s" % (b.shape,), ts)
        for b in low.cached_bufs:
            ts = []
            _buf_tensors(b, ts)
            add("cached buffer %s" % (b.shape,), ts)
        for fc in list(low.fused) + list(low.epilogue_fused):
            ts = []
            _spec_tensors(fc.spec, ts)
            add(fc.name, ts)
        for rec in low.conv_ins:
            ts = [rec.x, rec.weight, rec.bias, rec.tiles, rec.tile_img] + [a[0] for a in rec.aux]
            _buf_tensors(rec.out, ts)
            add("conv_in", ts)
        for rec in low.separable:
            ts = [rec.src, rec.idx, rec.tile_img]
            for br in rec.branches:
                _buf_tensors(br[3], ts)
            add(rec.name, ts)
        add("stack", list(low._nhwc_stacks.values()))
        add("static input", step.static_inputs)
        outs: List[torch.Tensor] = []
        _tensors(step.outputs, outs)
        add("output", outs)
        add("tile list", [sl.buf for sl in low.slots.values()] + [sl.tile_img for sl in low.slots.values()])
        add("shortcut flags", [r[0] for r in low.flag_recipes])
        for kind, rec, _fn in getattr(step.ex, "records", {}).values():
            ts = []
            _tensors(rec if not hasattr(rec, "out") else [rec.x, rec.weight, rec.bias, rec.tiles, rec.tile_img] + [a[0] for a in rec.aux], ts)
            if hasattr(rec, "out") and isinstance(rec.out, Buf):
                _buf_tensors(rec.out, ts)
            add(kind, ts)
        if model is not None:
            from sige_b200.parallel import cache_tensors

            for n, t in cache_tensors(model):
                found.append(("cache " + n, t))
        self.storages: Dict[Tuple[str, int], Storage] = {}
        for name, t in found:
            st = t.untyped_storage()
            key = (t.device.type, st.data_ptr())
            if key in self.storages or st.nbytes() == 0:
                continue
            b = torch.empty(0, dtype=torch.uint8, device=t.device).set_(st, 0, (st.nbytes(),), (1,))
            self.storages[key] = Storage(name, b)

    def holds(self, t: torch.Tensor) -> bool:
        return _key(t) in self.storages

    def assert_complete(self, step) -> None:
        """Every per-edit tensor a launch could wrongly write is part of the state: the tile lists and their image indices, the
        separable launches' image indices, the stacks of the attention chain (the q and o stacks of a sparse attention)."""
        low = step.low
        want = [("tile list", sl.buf) for sl in low.slots.values()]
        want += [("tile_img of a tile list", sl.tile_img) for sl in low.slots.values() if sl.tile_img is not None]
        want += [("tile_img of %s" % r.name, r.tile_img) for r in low.separable if r.tile_img is not None]
        for kind, rec, _fn in getattr(step.ex, "records", {}).values():
            if kind == "sparse_attention":
                want += [("sparse attention q", rec["q"]), ("sparse attention out", rec["out"])]
        for what, t in want:
            assert self.holds(t), "the step's state misses the %s" % what

    @property
    def nbytes(self) -> int:
        return sum(s.bytes.numel() for s in self.storages.values())

    def snapshot(self) -> Dict[Tuple[str, int], torch.Tensor]:
        return {k: s.bytes.clone() for k, s in self.storages.items()}

    def restore(self, snap) -> None:
        for k, s in self.storages.items():
            s.bytes.copy_(snap[k])

    def differs(self, snap) -> Optional[str]:
        for k, s in self.storages.items():
            if not torch.equal(s.bytes, snap[k]):
                return "%s (%d bytes differ)" % (s.name, int((s.bytes != snap[k]).sum()))
        return None


def _key(t: torch.Tensor):
    return (t.device.type, t.untyped_storage().data_ptr())


def padded_stacks(step) -> Dict[Tuple[str, int], Tuple[torch.Tensor, torch.Tensor]]:
    """Per storage: (stack [cap, C, h, w], its fixed-capacity list [cap, 2]) of every stack a launch writes or reads row for row
    through a one-edit list (row r is the tile of list entry r): the rows of SIGE_TILE_NONE entries belong to no tile."""
    out = {}
    for fc in list(step.low.fused) + list(step.low.epilogue_fused):
        s = fc.spec
        if s.idx is None or s.tile_img is not None or s.B != 1:
            continue
        for t in ([s.dst_stack] if s.dst_stack is not None else []) + ([s.srcs[0][0]] if s.src_is_stack else []):
            if t.shape[0] == s.idx.shape[0]:
                out[_key(t)] = (t, s.idx)
    return out


def poison_padding(step) -> int:
    """NaN into every row of a padded stack whose list entry is SIGE_TILE_NONE, so that a launch that reads one shows as NaN in a
    live element, or writes one as a stray byte.  Returns the number of rows poisoned."""
    n = 0
    with torch.no_grad():
        for t, idx in padded_stacks(step).values():
            pad = (idx[:, 0] <= NONE_BELOW).to(t.device)
            t[pad] = float("nan")
            n += int(pad.sum())
    return n


def live_tokens(step, t: torch.Tensor) -> Optional[torch.Tensor]:
    """bool [tokens] of a token view of a padded stack (row r: tokens r*h*w ..): the tokens of real tiles; None for another tensor."""
    hit = padded_stacks(step).get(_key(t))
    if hit is None:
        return None
    stack, idx = hit
    per = int(stack.shape[2] * stack.shape[3])
    assert t.data_ptr() == stack.data_ptr() and t.shape[-2] == stack.shape[0] * per
    return (idx[:, 0] > NONE_BELOW).to(t.device).repeat_interleave(per)


# ----------------------------------------------------------------------------------------------------------------------
# expectations
# ----------------------------------------------------------------------------------------------------------------------
@dataclass
class Want:
    """What a launch must leave in the elements of `tensor` (a live view) it writes: float64 values, the written mask, the
    per-element bound and the part of it that is the element's own rounding."""
    name: str
    tensor: torch.Tensor
    want: torch.Tensor
    written: torch.Tensor
    bound: torch.Tensor
    rounding: torch.Tensor
    free: Optional[torch.Tensor] = None      # elements the launch may leave with any value (rows of no tile)
    exact: Optional[torch.Tensor] = None     # the written tensor's exact contents in its dtype: compared bit for bit


def _from_expects(expects: List[kc.Expect]) -> List[Want]:
    out = []
    for e in expects:
        assert e.scratch is None, e.name
        out.append(Want(e.name, e.g.flat, e.want, e.written, e.bound, e.rounding))
    return out


def _live(t: torch.Tensor, layout: str) -> kc.Guarded:
    """A live buffer as a kc.Guarded with no guard band (the whole-state check stands in for it)."""
    assert t.is_contiguous(), "a %s buffer that is not contiguous in its layout" % layout
    return kc.Guarded(t.reshape(-1), t, 0, layout)


def _nhwc(t: torch.Tensor) -> torch.Tensor:
    return t.permute(0, 2, 3, 1)


def _u(dtype) -> float:
    return UNIT_ROUNDOFF[dtype]


def _act(x, name: str):
    return x * torch.sigmoid(x) if name == "swish" else x


def conv_expect(s, dtype, writes_raw: Optional[bool] = None) -> List[Want]:
    """float64 restatement of a ConvSpec (the launch contract of sige_tile_conv, as the lowering means it): gather halo tiles of the
    (virtually concatenated / up-sampled) sources, the pre-op or SPADE's modulation staged in `dtype`, zero outside the image, conv
    with the weight (rows scaled by `out_row_scale`) rounded once to `dtype` and the fp32 bias, the fresh 1x1 shortcut on flagged
    tiles and the residual elsewhere, the ReLU epilogue, the in-place scatter at (off + origin) / stride and the aux views.
    SIGE_TILE_NONE rows gather and write nothing."""
    dev = s.weight.device
    u = _u(dtype)
    w32, b32 = s.weight.clone(), None if s.bias is None else s.bias.clone()
    if s.out_row_scale is not None:
        rows, f = s.out_row_scale
        w32[:rows] *= f
        if b32 is not None:
            b32[:rows] *= f
    w = w32.to(dtype).double()
    R, k, st = s.block, s.k, s.stride
    Ro = (R - k) // st + 1
    if s.tile_img is not None:
        NT = s.N
        t = torch.arange(NT, device=dev)
        img, row = s.tile_img.long().to(dev), t
    else:
        NT = s.B * s.N
        t = torch.arange(NT, device=dev)
        img, row = t // s.N, t % s.N
    org = None if s.idx is None else s.idx.long().to(dev)[row]
    none = torch.zeros(NT, dtype=torch.bool, device=dev) if org is None else org[:, 0] <= NONE_BELOW
    pre_term = torch.zeros(s.Cout, dtype=torch.float64, device=dev)
    if s.src_is_stack:
        X = _nhwc(s.srcs[0][0])
        assert X.shape[0] == NT and X.shape[1] == R, (s.name, tuple(X.shape), NT)
        a = X.double()
    else:
        assert sum(int(t_.shape[1]) for t_, _ in s.srcs) == s.Cin, s.name
        safe = torch.where(none[:, None], torch.zeros_like(org), org)
        a, valid = _gather([(_nhwc(t_), up) for t_, up in s.srcs], safe, img, R, s.H, s.W)
        staged = s.scale is not None or s.shift is not None or s.act != "identity" or s.modulation is not None
        if staged:
            def per(v):
                v = v.double().to(dev)
                return (v[img] if v.dim() == 2 else v.expand(NT, -1))[:, None, None, :]
            if s.scale is not None:
                a = a * per(s.scale)
            if s.shift is not None:
                a = a + per(s.shift)
            a = _act(a, s.act)
            if s.modulation is not None:
                gamma, beta, slope = s.modulation
                g, _ = _gather([(_nhwc(gamma), 0)], safe, img, R, s.H, s.W)
                bt, _ = _gather([(_nhwc(beta), 0)], safe, img, R, s.H, s.W)
                m = a * (1 + g) + bt
                a = torch.where(m > 0, m, m * float(slope))
            a = a.to(dtype).double()
        a = torch.where((valid & ~none[:, None, None])[..., None], a, torch.zeros((), dtype=a.dtype, device=dev))
        if staged:
            pre_term = PRE_ULPS * u * w.abs().amax(dim=(1, 2, 3)) * a.abs().max()
    nchw = a.permute(0, 3, 1, 2)
    v = F.conv2d(nchw, w, stride=st).permute(0, 2, 3, 1)                                  # [NT, Ro, Ro, Cout]
    mag = F.conv2d(nchw.abs(), w.abs(), stride=st).permute(0, 2, 3, 1)
    if b32 is not None:
        v, mag = v + b32.double(), mag + b32.double().abs()
    zero = torch.zeros((), dtype=torch.float64, device=dev)
    fresh = torch.zeros(NT, dtype=torch.bool, device=dev)
    if s.shortcut is not None:
        sc_tensors, sc_w, sc_b, sc_flags = s.shortcut
        assert k == 3 and R == 6 and st == 1, s.name
        fresh = torch.ones(NT, dtype=torch.bool, device=dev) if sc_flags is None else sc_flags.to(dev)[row] != 0
        fresh = fresh & ~none
        x2, ok2 = _gather([(_nhwc(t_), 0) for t_ in sc_tensors], torch.where(none[:, None], torch.zeros_like(org), org) + 1, img, 4, s.H, s.W)
        x2 = torch.where(ok2[..., None], x2, zero)
        w2 = sc_w.to(dtype).double()[:, :, 0, 0]
        b2 = torch.zeros(s.Cout, dtype=torch.float64, device=dev) if sc_b is None else sc_b.double()
        f = fresh[:, None, None, None]
        v = v + torch.where(f, x2 @ w2.t() + b2, zero)
        mag = mag + torch.where(f, x2.abs() @ w2.abs().t() + b2.abs(), zero)
    out: List[Want] = []

    def put(name, tensor, val, bd, rows_ok, pix=None):
        """tensor: NHWC view; rows_ok [NT] tiles that write; pix (OB, OH, OW, ok [NT, Ro, Ro]) or None for a stack."""
        want = tensor.double().clone()
        written = torch.zeros(tensor.shape, dtype=torch.bool, device=dev)
        bound = torch.zeros(tensor.shape, dtype=torch.float64, device=dev)
        rnd = torch.zeros(tensor.shape, dtype=torch.float64, device=dev)
        sl = slice(0, s.Cout)
        if pix is None:
            tt = torch.arange(NT, device=dev)[rows_ok]
            want[tt, :, :, sl], written[tt, :, :, sl] = val[rows_ok], True
            bound[tt, :, :, sl], rnd[tt, :, :, sl] = bd[rows_ok], u * val[rows_ok].abs()
        else:
            OB, OH, OW, ok = pix
            want[OB[ok], OH[ok], OW[ok], sl] = val[ok]
            written[OB[ok], OH[ok], OW[ok], sl] = True
            bound[OB[ok], OH[ok], OW[ok], sl] = bd[ok]
            rnd[OB[ok], OH[ok], OW[ok], sl] = u * val[ok].abs()
        out.append(Want(name, tensor, want, written, bound, rnd))

    if s.dst_stack is not None:
        assert s.residual is None and not s.aux, s.name
        if s.epilogue_act == "relu":
            v = v.clamp(min=0)
        put("dst_stack", _nhwc(s.dst_stack), v, u * v.abs() + ACC * mag + pre_term + ABS, ~none)
        return out
    Hd, Wd = s.dst.shape[2], s.dst.shape[3]
    base = s.off + org
    base = torch.div(base, st, rounding_mode="trunc") if st != 1 else base
    d = torch.arange(Ro, device=dev)
    oh, ow = base[:, :1] + d, base[:, 1:] + d
    ok = ((oh >= 0) & (oh < Hd))[:, :, None] & ((ow >= 0) & (ow < Wd))[:, None, :] & ~none[:, None, None]
    OB = img[:, None, None].expand(NT, Ro, Ro)
    OH, OW = oh[:, :, None].expand(NT, Ro, Ro).clamp(0, Hd - 1), ow[:, None, :].expand(NT, Ro, Ro).clamp(0, Wd - 1)
    if s.residual is not None:
        r = _nhwc(s.residual)[OB, OH, OW][..., :s.Cout].double()
        use = (~fresh)[:, None, None, None]
        v = v + torch.where(use, r, zero)
        mag = mag + torch.where(use, r.abs(), zero)
    if s.epilogue_act == "relu":
        assert not s.aux, s.name
        v = v.clamp(min=0)
    bound = u * v.abs() + ACC * mag + pre_term + ABS
    pix = (OB, OH, OW, ok)
    if s.dst.has_raw if writes_raw is None else writes_raw:
        put("dst", _nhwc(s.dst.raw), v, bound, None, pix)
    for i, (view, sc, sh, act) in enumerate(s.aux):
        scv = torch.ones(s.Cout, dtype=torch.float64, device=dev) if sc is None else sc.double()
        shv = torch.zeros(s.Cout, dtype=torch.float64, device=dev) if sh is None else sh.double()
        av = _act(v * scv + shv, act)
        put("aux%d" % i, _nhwc(view), av, SWISH_LIP * scv.abs() * bound + u * av.abs(), None, pix)
    return out


def conv_in_expect(rec, dtype) -> List[Want]:
    """The stem's record as a kernel_contracts conv_in case on the live tensors (tiles: per-image rows when the lists are a batch)."""
    x = _nhwc(rec.x)
    B, H, W, Cin = x.shape
    Cout = int(rec.weight.shape[0])
    tiles, n_tiles = None, 0
    if rec.tiles is not None:
        idx = rec.tiles.to(torch.int32)
        if rec.tile_img is None:
            tiles, n_tiles = (False, (int(idx.shape[0]),), rec.tile_size, 0), int(idx.shape[0])
        else:                                         # tile i of image tile_img[i]: row tile_img[i] * n + i of B lists of n rows
            n = int(idx.shape[0])
            rows = torch.full((B * n, 2), kc.TILE_NONE, dtype=torch.int32, device=idx.device)
            ii = torch.arange(n, device=idx.device)
            rows[rec.tile_img.long() * n + ii] = idx
            idx, tiles, n_tiles = rows, (True, (n,) * B, rec.tile_size, 0), n
        rec_idx = idx
    else:
        rec_idx = None
    aux_spec = tuple((sc is not None or sh is not None, 1 if act == "swish" else 0, False) for (_, sc, sh, act) in rec.aux)
    spec = kc.ConvInSpec("conv_in", B=B, H=H, W=W, Cin=Cin, Cout=Cout, aux=aux_spec, tiles=tiles, bias=rec.bias is not None)
    if rec.out.has_raw:
        out_g = _live(_nhwc(rec.out.raw), "nhwc")
    else:                                             # only the aux views are written: a stand-in for the raw output
        dummy = torch.zeros(B, H, W, Cout, dtype=dtype, device=x.device)
        out_g = kc.Guarded(dummy.reshape(-1), dummy, 0, "nhwc")
    case = kc.ConvInCase(spec, dtype, x, rec.weight.detach().to(dtype), None if rec.bias is None else rec.bias.detach().to(dtype), rec_idx, n_tiles,
                         out_g, [_live(_nhwc(a[0]), "nhwc") for a in rec.aux],
                         [None if a[1] is None and a[2] is None else (torch.ones(Cout, device=x.device) if a[1] is None else a[1]) for a in rec.aux],
                         [None if a[1] is None and a[2] is None else (torch.zeros(Cout, device=x.device) if a[2] is None else a[2]) for a in rec.aux])
    wants = _from_expects(kc.conv_in_reference(case))
    return wants if rec.out.has_raw else wants[1:]


def tail_expect(r, dtype) -> List[Want]:
    """GroupNorm folded into (scale, shift) (kernel_contracts.gn_reference) and conv_out on act(x*scale + shift)
    (kernel_contracts.conv_out_reference), with the fold's bound carried through the conv."""
    x = _nhwc(r["x"])
    B, H, W, C = x.shape
    dev = x.device
    gamma = None if r["gamma"] is None else r["gamma"].detach().to(dtype)
    beta = None if r["beta"] is None else r["beta"].detach().to(dtype)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count if dev.type == "cuda" else kc.H100_SMS
    def spare():
        flat = torch.zeros(B * C, device=dev)
        return kc.Guarded(flat, flat.view(B, C), 0, "bc")

    gn = kc.GNCase(kc.GNSpec("tail", B, H, W, C, int(r["groups"]), affine=gamma is not None, eps=float(r["eps"])), dtype, x, gamma, beta,
                   spare(), spare(), spare(), sms)
    expects, (b_scale, b_shift) = kc.gn_reference(gn)
    scale = expects[0].want.view(B, C).float()
    shift = expects[1].want.view(B, C).float()
    out = r["out"]
    Cout = int(r["weight"].shape[0])
    act = 1 if r["act"] == "swish" else 0
    case = kc.ConvOutCase(kc.ConvOutSpec("tail", B, H, W, C, Cout, act=act, pre="both", bias=r["bias"] is not None), dtype, x, scale, shift,
                          r["weight"].detach().to(dtype), None if r["bias"] is None else r["bias"].detach().to(dtype), _live(out, "nchw"))
    (e,) = kc.conv_out_reference(case)
    # the kernel's (scale, shift) is within (b_scale, b_shift) of the float64 fold, which is fp32-rounded here: twice that, through
    # the activation (<= SWISH_LIP) and the conv's |w|
    dz = 2 * (x.double().abs() * b_scale.view(B, 1, 1, C) + b_shift.view(B, 1, 1, C)) * SWISH_LIP
    prop = F.conv2d(dz.permute(0, 3, 1, 2), case.w.double().abs(), padding=1)
    e.bound = e.bound + prop.reshape(-1)
    return _from_expects([e])


def attention_expect(r, dtype) -> List[Want]:
    qkv, out = r["qkv"], r["out"]
    B, N, C3 = qkv.shape
    case = kc.AttnCase(kc.AttnSpec("attention", B, N, C3 // 3, "random"), dtype, qkv, _live(out, "bnc"))
    return _from_expects(kc.attn_reference(case))


def sparse_attention_expect(r, dtype, live: Optional[torch.Tensor] = None) -> List[Want]:
    """live: bool [Nq], the queries of real tiles (None: all).  Every live query within its bound; the others (rows of padding
    tiles) may be left with any value."""
    q, k, v, out = r["q"], r["k"], r["v"], r["out"]
    if q.dim() == 3:
        q, k, v, out = q.unsqueeze(1), k.unsqueeze(1), v.unsqueeze(1), out.unsqueeze(1)
    B, Hh, Nq, D = q.shape
    spec = skc.SAttnSpec("sparse_attention", B, Hh, Nq, int(k.shape[2]), D, scale=float(r["scale"]))
    case = skc.SAttnCase(spec, dtype, q, k, v, {}, _live(out, "bhnd"), out)
    sms = torch.cuda.get_device_properties(q.device).multi_processor_count if q.device.type == "cuda" else kc.H100_SMS
    (w,) = _from_expects(skc.wide_sattn_reference(case, sms=sms) if D == skc.WIDE_D else skc.sattn_reference(case))
    if live is not None:
        dead = (~live.to(q.device)).view(1, 1, Nq, 1).expand(B, Hh, Nq, D).reshape(-1)
        w.free = dead & w.written
        w.written = w.written & ~dead
    return [w]


class _LiveSpade(skc.SpadeCase):
    """A SpadeCase on live [pixels, C] operands."""

    def __init__(self, spec, dtype, x, gamma, beta, out):
        super().__init__(spec, dtype, x, gamma, out)
        self._x, self._g, self._b = x, gamma, beta

    @property
    def C(self):
        return int(self._x.shape[1])

    @property
    def x(self):
        return self._x

    @property
    def gamma(self):
        return self._g

    @property
    def beta(self):
        return self._b


def spade_expect(r, dtype) -> List[Want]:
    def pc(t):
        return _nhwc(t).reshape(-1, t.shape[1]) if t.dim() == 4 else t.reshape(-1, t.shape[-1])

    out = r["out"]
    o = _nhwc(out) if out.dim() == 4 else out
    x = pc(r["x"])
    case = _LiveSpade(skc.SpadeSpec("spade", int(x.shape[1]), int(x.shape[0]), float(r["slope"])), dtype, x, pc(r["gamma"]), pc(r["beta"]),
                      _live(o.reshape(-1, o.shape[-1]), "pc"))
    return _from_expects(skc.spade_reference(case))


def separable_expect(rec, dtype) -> List[Want]:
    """A SepLaunch as a kernel_contracts separable case on the live tensors: the depthwise weight and bias with the record's
    per-channel affine folded in fp32 (scale * w, scale * b + shift), the 1x1 weight in `dtype`, its fp32 bias.  A batch of
    edits (`tile_img`): row m of the list is a tile of image tile_img[m] only, the per-image form of the restatement."""
    src = _nhwc(rec.src)
    idx = rec.idx
    per_image = rec.tile_img is not None
    n = int(idx.shape[0]) // (rec.batch if per_image else 1)
    Cin, Cout = rec.Cin, rec.Cout
    dw_w, dw_b, pw_w, pw_b, dst = [], [], [], [], []
    for (dwc, w1, b1, buf) in rec.branches:
        w = dwc.weight.detach().float().reshape(Cin, 9)
        b = None if dwc.bias is None else dwc.bias.detach().float()
        if dwc.scale is not None:
            sc = dwc.scale.float().reshape(-1).to(w.device)
            w = w * sc[:, None]
            b = None if b is None else b * sc
        if dwc.shift is not None:
            sh = dwc.shift.float().reshape(-1).to(w.device)
            b = sh if b is None else b + sh
        dw_w.append(w.contiguous())
        dw_b.append(b)
        pw_w.append(w1.detach().to(dtype).reshape(Cout, -1))
        pw_b.append(None if b1 is None else b1.detach().float())
        dst.append(_live(_nhwc(buf.raw), "nhwc"))
    dH, dW = int(rec.branches[0][3].shape[2]), int(rec.branches[0][3].shape[3])
    spec = kc.SepSpec(rec.name, B=rec.batch, Cin=Cin, Cout=Cout, H=6 if rec.src_stack else int(src.shape[1]), W=6 if rec.src_stack else int(src.shape[2]),
                      real=n, lead=n, pre=rec.c0, post=int(src.shape[3]) - rec.c0 - Cin, src_stack=rec.src_stack, offH=rec.off, offW=rec.off,
                      dH=dH, dW=dW, dsts=tuple(("buf", int(b_.shape[1]) - Cout, 0) for (_, _, _, b_) in rec.branches), per_image=per_image)
    case = kc.SepCase(spec, dtype, src, idx, dw_w, dw_b, pw_w, pw_b, dst, rec.tile_img)
    return _from_expects(kc.sep_reference(case))


def _cdiv(a: torch.Tensor, b: int) -> torch.Tensor:
    return torch.div(a, b, rounding_mode="trunc")


def writeback_expect(entries, dtype) -> List[Want]:
    """sige_tile_writeback: the output tiles of each tile list copied exactly into the cache (f32 or the source's dtype)."""
    out = []
    for i, (src, dst, idx, off, stride, ro) in enumerate(entries):
        dev = src.device
        B, C, H, W = src.shape
        org = idx.long().to(dev)
        org = org[org[:, 0] > NONE_BELOW]
        y, x = _cdiv(off + org[:, 0], stride), _cdiv(off + org[:, 1], stride)
        d = torch.arange(ro, device=dev)
        hh, ww = y[:, None] + d, x[:, None] + d
        mask = torch.zeros(H, W, dtype=torch.bool, device=dev)
        ok = ((hh >= 0) & (hh < H))[:, :, None] & ((ww >= 0) & (ww < W))[:, None, :]
        mask[hh[:, :, None].expand(-1, ro, ro)[ok], ww[:, None, :].expand(-1, ro, ro)[ok]] = True
        m4 = mask.view(1, 1, H, W).expand(B, C, H, W)
        want = torch.where(m4, src.to(dst.dtype).double(), dst.double())
        z = torch.zeros(dst.shape, dtype=torch.float64, device=dev)
        out.append(Want("cache%d" % i, dst, want, m4.clone(), z, z))
    return out


def cached_view(c: torch.Tensor, sc, sh, act: str, dtype) -> Tuple[torch.Tensor, torch.Tensor]:
    """float64 act(cache * scale + shift) of a producer-written view of a cached buffer, and its bound: the fp32 affine and
    activation (4 fp32 roundings of |cache * scale| + |shift| through the activation), the rounding to `dtype`."""
    z = c.double()
    if sc is not None:
        z = z * sc.double().view(1, -1, 1, 1)
    if sh is not None:
        z = z + sh.double().view(1, -1, 1, 1)
    want = _act(z, act)
    lin = c.double().abs() * (1 if sc is None else sc.double().abs().view(1, -1, 1, 1)) + (0 if sh is None else sh.double().abs().view(1, -1, 1, 1))
    return want, _u(dtype) * want.abs() + SWISH_LIP * 4 * 2.0 ** -24 * lin + ABS


def cache_load_expect(entries, dtype) -> List[Want]:
    """sige_cache_load: each raw buffer the cache in `dtype` broadcast over the buffer's images, bitwise; each view
    act(cache * scale + shift) within cached_view's bound."""
    out = []
    for i, (src, raw, views) in enumerate(entries):
        if raw is not None:
            exact = src.to(raw.device).to(dtype).expand(raw.shape)
            z = torch.zeros(raw.shape, dtype=torch.float64, device=raw.device)
            out.append(Want("raw%d" % i, raw, exact.double(), torch.ones(raw.shape, dtype=torch.bool, device=raw.device), z, z, exact=exact))
        for j, (v, sc, sh, act) in enumerate(views):
            want, bound = cached_view(src.to(v.device), sc, sh, act, dtype)
            want, bound = want.expand(v.shape), bound.expand(v.shape)
            out.append(Want("view%d.%d" % (i, j), v, want, torch.ones(v.shape, dtype=torch.bool, device=v.device), bound, _u(dtype) * want.abs()))
    return out


EXPECT = {"conv": conv_expect, "conv_in": conv_in_expect, "tail": tail_expect, "attention": attention_expect,
          "sparse_attention": sparse_attention_expect, "spade": spade_expect, "separable": separable_expect, "writeback": writeback_expect,
          "cache_load": cache_load_expect}


# ----------------------------------------------------------------------------------------------------------------------
# the walk
# ----------------------------------------------------------------------------------------------------------------------
Masks = Dict[Tuple[str, int], torch.Tensor]


def _allowed(state: State, wants: List[Want], free_only: bool = False) -> Masks:
    """Per storage: bool over its bytes, True where the launch may write (free_only: only the elements it may leave with any
    value)."""
    out: Masks = {}
    for w in wants:
        t = w.tensor
        key = _key(t)
        assert key in state.storages, "%s: written tensor outside the step's state" % w.name
        if free_only and w.free is None:
            continue
        nb = state.storages[key].bytes.numel()
        es = t.element_size()
        elem = torch.zeros(nb // es, dtype=torch.bool, device=t.device)
        elem.as_strided(t.shape, t.stride(), t.storage_offset())[w.free if free_only else (w.written if w.free is None else (w.written | w.free))] = True
        byte = elem.view(-1, 1).expand(-1, es).reshape(-1)
        out[key] = byte if key not in out else (out[key] | byte)
    return out


def _union(into: Masks, more: Masks) -> None:
    for k, m in more.items():
        into[k] = m.clone() if k not in into else (into[k] | m)


@dataclass
class KindStats:
    launches: int = 0
    worst: float = 0.0
    worst_at: str = ""
    excess: float = 0.0
    excess_at: str = ""


def _check_values(label: str, wants: List[Want]) -> Tuple[float, float]:
    worst = excess = 0.0
    for w in wants:
        if w.exact is not None:
            same = kc.bits(w.tensor.contiguous()) == kc.bits(w.exact.contiguous())
            if not bool(same.all()):
                pos = tuple(int(z) for z in (~same).nonzero()[0])
                raise AssertionError("%s: %s at %s of %s: got %r, want %r bit for bit; %d elements differ"
                                     % (label, w.name, pos, tuple(w.tensor.shape), float(w.tensor[pos]), float(w.exact[pos]), int((~same).sum())))
        m = w.written
        if not bool(m.any()):
            continue
        got = w.tensor.double()[m]
        err = (got - w.want[m]).abs()
        bd = w.bound[m]
        ratio = torch.nan_to_num(torch.where(err == 0, torch.zeros_like(err), err / bd), nan=float("inf"))
        r = float(ratio.max())
        if r > 1.0:
            j = int(ratio.argmax())
            pos = tuple(int(z) for z in m.nonzero()[j])
            raise AssertionError("%s: %s at %s of %s: got %r, want %r, |err| %.3g > bound %.3g; %d elements over"
                                 % (label, w.name, pos, tuple(w.tensor.shape), float(got[j]), float(w.want[m][j]), float(err[j]), float(bd[j]),
                                    int((ratio > 1).sum())))
        worst = max(worst, r)
        rest = (bd - w.rounding[m]).clamp(min=1e-300)
        excess = max(excess, float(((err - w.rounding[m]).clamp(min=0) / rest).max()))
    return worst, excess


def _sync(dev) -> None:
    if dev.type == "cuda":
        torch.cuda.synchronize(dev)


def _check_launch(state: State, kinds: Dict[str, KindStats], kind: str, label: str, wants: List[Want], fn, stream, dev,
                  footprint: Masks, free: Masks) -> None:
    """Snapshot the whole state, launch, synchronise: nothing outside the wanted elements changed, every wanted one in bound.
    The bytes the launch may write join `footprint`, those it may leave with any value `free`."""
    allowed = _allowed(state, wants)
    _union(footprint, allowed)
    _union(free, _allowed(state, wants, free_only=True))
    snap = state.snapshot()
    fn(stream)
    _sync(dev)
    for key, s in state.storages.items():
        changed = s.bytes != snap[key]
        if key in allowed:
            changed &= ~allowed[key]
        if bool(changed.any()):
            i = int(changed.nonzero()[0])
            raise AssertionError("%s: wrote outside its record into %s at byte %d of %d (%d stray bytes)"
                                 % (label, s.name, i, s.bytes.numel(), int(changed.sum())))
    r, x = _check_values(label, wants)
    ks = kinds.setdefault(kind, KindStats())
    ks.launches += 1
    if r >= ks.worst:
        ks.worst, ks.worst_at = r, label
    if x >= ks.excess:
        ks.excess, ks.excess_at = x, label


def walk(step, program=None, model=None, state: Optional[State] = None) -> Dict[str, object]:
    """Run `program` (default: the step's main program) entry by entry, checking each against its record, after poisoning the
    padding rows of the step's stacks (poison_padding).  Returns {"kinds": {kind: KindStats}, "eager": count, "seconds": wall
    time, "state_bytes": size of the whole state, "poisoned": padding rows poisoned}."""
    program = step.steps if program is None else program
    ex = step.ex
    state = state or State(step, model)
    state.assert_complete(step)
    poisoned = poison_padding(step)
    dev = step.dev
    stream = torch.cuda.current_stream(dev).cuda_stream if dev.type == "cuda" else 0
    kinds: Dict[str, KindStats] = {}
    footprint: Masks = {}
    free: Masks = {}
    eager = 0
    t0 = time.perf_counter()
    with torch.no_grad():
        for pos, (kind, fn) in enumerate(program):
            if kind == "eager":
                fn(stream)
                _sync(dev)
                eager += 1
                continue
            if kind not in EXPECT:
                raise AssertionError("step %d: no restatement for launch kind %r" % (pos, kind))
            rec = ex.record_of(kind, fn)
            label = "%s launch %d (%s)" % (kind, pos, rec.name if kind in ("conv", "separable") else kind)
            if kind == "conv":
                wants = conv_expect(rec, step.dtype, ex.writes_raw(fn.__self__))
            elif kind == "sparse_attention":
                wants = sparse_attention_expect(rec, step.dtype, live_tokens(step, rec["q"]))
            else:
                wants = EXPECT[kind](rec, step.dtype)
            _check_launch(state, kinds, kind, label, wants, fn, stream, dev, footprint, free)
    return {"kinds": kinds, "eager": eager, "seconds": time.perf_counter() - t0, "state_bytes": state.nbytes, "poisoned": poisoned,
            "footprint": footprint, "free": free}


def walk_loads(step, model=None, state: Optional[State] = None) -> Dict[str, object]:
    """The cache load of a new edit (`Lowering.load_caches`) as a program of its own: the prepared `sige_cache_load`, checked as
    `walk` checks a launch, then the torch restores of the cached buffers it does not take, unchecked and counted as `eager`."""
    run, rest = step.low.prepared_loader()
    state = state or State(step, model)
    dev = step.dev
    stream = torch.cuda.current_stream(dev).cuda_stream if dev.type == "cuda" else 0
    kinds: Dict[str, KindStats] = {}
    footprint: Masks = {}
    free: Masks = {}
    t0 = time.perf_counter()
    with torch.no_grad():
        if run is not None:
            rec = step.ex.record_of("cache_load", run)
            _check_launch(state, kinds, "cache_load", "cache_load launch 0 (cache_load)", cache_load_expect(rec, step.dtype), run, stream, dev,
                          footprint, free)
        for b in rest:
            b.restore()
        _sync(dev)
    return {"kinds": kinds, "eager": len(rest), "seconds": time.perf_counter() - t0, "state_bytes": state.nbytes,
            "entries": 0 if run is None else len(step.ex.record_of("cache_load", run)), "footprint": footprint, "free": free}


POISON = 0xFF                  # every byte: NaN in f16, bf16 and f32


def poison(state: State, footprint: Masks) -> int:
    """POISON into every byte of a program's write footprint (the union of its launches' `_allowed` masks, as `walk` returns
    it).  A launch that reads a byte its program writes before the program has written it then reads NaN.  Returns the bytes
    poisoned."""
    n = 0
    with torch.no_grad():
        for key, m in footprint.items():
            state.storages[key].bytes[m] = POISON
            n += int(m.sum())
    return n


def differs_outside(state: State, snap, free: Masks) -> Optional[str]:
    """Like State.differs, ignoring the bytes a launch may leave with any value (`free`: rows of padding tiles)."""
    for k, s in state.storages.items():
        d = s.bytes != snap[k]
        if k in free:
            d &= ~free[k]
        if bool(d.any()):
            return "%s (%d bytes differ, the first at byte %d)" % (s.name, int(d.sum()), int(d.nonzero()[0]))
    return None


def poisoned_walk(step, res, start, walked, program=None, model=None, state: Optional[State] = None, loads: bool = False):
    """From `start`, the footprint of the first walk `res` poisoned (and, before a walk, the padding rows, as `walk` does): the
    walk again (walk or walk_loads), which must meet every record and leave every byte outside the padding rows as the first walk left them
    (`walked`).  Returns (the second walk's result, the poisoned state it started from, the state it ended in, bytes
    poisoned)."""
    state = state or State(step, model)
    state.restore(start)
    n = poison(state, res["footprint"])
    if not loads:
        poison_padding(step)
    from_ = state.snapshot()
    res2 = walk_loads(step, model=model, state=state) if loads else walk(step, program, model=model, state=state)
    diff = differs_outside(state, walked, res["free"])
    assert diff is None, "after its write footprint was poisoned (%d bytes), the walk ends differently: %s" % (n, diff)
    return res2, from_, state.snapshot(), n


def summary(tag: str, res) -> str:
    parts = ["%s x%d worst %.3f (%s) excess %.3f" % (k, s.launches, s.worst, s.worst_at, s.excess) for k, s in sorted(res["kinds"].items())]
    return "[fused step contract] %s: %s; eager %d; %d padding rows poisoned; %.2f s; state %.1f MB" % (
        tag, "; ".join(parts), res["eager"], res.get("poisoned", 0), res["seconds"], res["state_bytes"] / 2 ** 20)


def checked_all(step, res, program=None) -> None:
    """Every non-eager entry of the program was checked, and nothing else."""
    program = step.steps if program is None else program
    want: Dict[str, int] = {}
    for kind, _ in program:
        if kind != "eager":
            want[kind] = want.get(kind, 0) + 1
    got = {k: s.launches for k, s in res["kinds"].items()}
    assert got == want, (got, want)
    assert res["eager"] == sum(1 for k, _ in program if k == "eager")


def cached_state_after_rebind(step) -> float:
    """After `rebind()`: every cached buffer's raw equals its cache in the step dtype, bitwise, and every producer-written view
    of it is within the aux bound of act(cache*scale + shift).  Returns the worst view error / bound ratio."""
    dt = step.dtype
    worst = 0.0
    for b in step.low.cached_bufs:
        c = b.cached_init.to(b.raw.device if b.has_raw else step.dev)
        if b.has_raw:
            want = c.to(dt).expand(b.shape)
            assert torch.equal(kc.bits(b.raw.contiguous()), kc.bits(want.contiguous())), "cached buffer %s differs from its cache" % (b.shape,)
        for (v, sc, sh, act) in b.view_inits:
            want, bound = cached_view(c, sc, sh, act, dt)
            r = float(((v.double() - want.expand(v.shape)).abs() / bound.expand(v.shape)).max())
            assert r <= 1.0, "view of cached buffer %s: error / bound %.3g" % (b.shape, r)
            worst = max(worst, r)
    return worst




