"""Mode / mask / cache state machine of the SIGE operator surface.

Mirrors the control-plane half of reference sige/nn/base.py (SIGEModule :10-72,
SIGEModuleWrapper :75-77, SIGEModel :95-129): three inference modes —

    full     dense pass on the ORIGINAL image; modules record shapes and fill their caches
    sparse   tile-sparse pass on the EDITED image, using the caches and the active-tile lists
    profile  shape-only dummies so that a MAC profiler can trace the sparse graph

— plus ``set_masks`` (difference-mask pyramid -> per-module active indices, memoised per
geometry inside one call), ``set_cache_id`` / ``set_sparse_update`` (the multi-step cached flow
of reference diffusion_demo/) and ``clear_cache``.

What differs from the reference: there is one backend.  ``load_runtime`` does not import
``sige.cpu|cuda|mps`` (reference base.py:35-50); the kernels live in libsige_b200.so and are
reached through ``sige_b200.ops``; a non-CUDA tensor in sparse mode raises.  fp16 / bf16 are
accepted next to fp32 (the reference rejects them, base.py:15,55-63).
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Tuple

import torch
from torch import nn

MODES = ("full", "sparse", "profile")
SUPPORTED_DTYPES = [torch.float32, torch.float16, torch.bfloat16]

# Bumped whenever a Scatter* / ScatterGather module (re)fills a cache in `full` mode: compiled fused steps that were
# built from older caches are stale.
_cache_generation = [0]


def bump_cache_generation() -> None:
    _cache_generation[0] += 1


class SIGEModule(nn.Module):
    """Base of every mode-aware module.  ``call_super=False`` lets a class that also derives from
    another nn.Module (e.g. ``SIGEConv2d(nn.Conv2d, SIGEModule)``) initialise nn.Module once."""

    def __init__(self, call_super: bool = True):
        if call_super:
            super().__init__()
        self.devices: List[str] = ["cuda"]
        self.supported_dtypes = list(SUPPORTED_DTYPES)
        self.mode: str = "full"
        self.runtime: Dict = {}
        self.mask: Optional[torch.Tensor] = None
        self.timestamp = None
        self.cache_id = 0
        self.sparse_update = False

    # ---- state setters walked by SIGEModel ----
    def set_mask(self, masks: Dict, cache: Dict, timestamp: int):
        self.timestamp = timestamp

    def set_mode(self, mode: str):
        self.mode = mode

    def set_cache_id(self, cache_id: int):
        self.cache_id = cache_id

    def set_sparse_update(self, sparse_update: bool):
        self.sparse_update = sparse_update

    def clear_cache(self):
        pass

    # ---- backend lookup (API-compatible; single backend) ----
    def load_runtime(self, function_name: str, runtime_dict: Dict = None) -> Dict:
        """Reference base.py:35-50 probes sige.cpu / sige.cuda / sige.mps.  Here the only runtime is
        the sm_90a library; the dict keeps the reference's shape ({device: callable})."""
        from .. import ops

        if runtime_dict is None:
            runtime_dict = self.runtime
        runtime_dict["cuda"] = getattr(ops, function_name, None)
        return runtime_dict

    # ---- argument checks (reference base.py:55-72) ----
    def check_dtype(self, *tensors):
        for t in tensors:
            if t is None:
                continue
            assert isinstance(t, torch.Tensor)
            if t.dtype not in self.supported_dtypes:
                raise NotImplementedError(
                    "[%s] does not support dtype [%s]!!! Currently supported dtype %s."
                    % (self.__class__.__name__, t.dtype, str(self.supported_dtypes))
                )

    def check_dim(self, *tensors):
        for t in tensors:
            if t is None:
                continue
            assert isinstance(t, torch.Tensor)
            if t.dim() != 4:
                raise NotImplementedError("[%s] does not support input with dim [%d]!!!" % (self.__class__.__name__, t.dim()))

    def _unknown_mode(self):
        return NotImplementedError("Unknown mode: [%s]!!!" % self.mode)


class SIGEModuleWrapper:
    """Holds a module WITHOUT registering it as a child (a Scatter refers to its paired Gather,
    which is already owned by the block; reference base.py:75-77)."""

    def __init__(self, module: SIGEModule):
        self.module = module


class SIGEModel(nn.Module):
    """Top-level wrapper: broadcasts mode / masks / cache controls to every SIGEModule below it
    (reference base.py:95-129).

    Beyond the reference: in ``sparse`` mode on a CUDA fp16/bf16 input the forward is run as a FUSED STEP
    (``sige_b200.fused``): traced once on lazy handles, lowered to one fused sm_90a launch per wrapped layer,
    captured in a CUDA graph and replayed on every later call — the model file itself is unchanged.  The compiled step
    is keyed on (set_masks call, cache generation, cache_id, argument shapes) and rebuilt when any of them changes;
    ``set_fused(False)`` (or SIGE_FUSED=0) keeps the eager operator modules, which is also what a forward that cannot
    be traced falls back to.  An fp32 model (the reference's own precision) keeps its dense pass exactly as the reference
    computes it and runs its sparse steps on the tensor cores after ``set_fused(True, dtype=torch.float16)``; without that
    opt-in fp32 inputs always run through the eager fp32 operator modules."""

    def __init__(self, call_super: bool = True):
        if call_super:
            super().__init__()
        self.mode = "full"
        self.timestamp = 0
        self._sige_cache_id = 0
        self._sige_sparse_update = False
        self._fused_enabled = os.environ.get("SIGE_FUSED", "1") != "0"
        self._fused_options: Dict = {}
        self._fused_steps: Dict = {}
        self.fused_step = None          # the step object that served the last fused call (for introspection / benchmarks)

    def _sige_modules(self):
        for m in self.modules():
            if isinstance(m, SIGEModule):
                yield m

    def set_masks(self, masks: Dict[Tuple[int, int], torch.Tensor]):
        """Difference-mask pyramid -> active tile lists of every module (reference base.py:102-108).

        Beyond the reference: (i) calling it again with the SAME mask tensors (Stable Diffusion's sampler does, every step:
        stable-diffusion/ldm/models/diffusion/ddim.py:203-204) is a no-op — no kernel, no host sync, compiled fused steps stay
        valid; (ii) a new pyramid costs ONE host synchronisation for all geometries together (the reference pays one
        ``torch.nonzero`` sync per geometry)."""
        sig = tuple(sorted((tuple(res), t.data_ptr(), t._version, tuple(t.shape), str(t.dtype), str(t.device)) for res, t in masks.items()))
        d = self.__dict__
        d.pop("_async_masks", None)          # a synchronous call supersedes lists installed by set_masks_async
        if d.get("_mask_sig") == sig and d.get("_mask_modules") == sum(1 for _ in self._sige_modules()):
            return
        self.timestamp += 1
        shared: Dict = {}  # geometry-keyed memo shared by all modules during this call
        from .modules import prefill_active_indices

        mods = list(self._sige_modules())
        prefill_active_indices(mods, masks, shared)
        for m in mods:
            m.set_mask(masks, shared, self.timestamp)
        d["_mask_sig"], d["_mask_keep"], d["_mask_modules"] = sig, list(masks.values()), len(mods)     # (the tensors are kept alive: their addresses are part of the key)

    def set_masks_async(self, masks: Dict[Tuple[int, int], torch.Tensor]) -> bool:
        """`set_masks` for the NEXT edit without a host synchronisation (an extension; SURVEY section 8f-4): when a compiled fused
        step exists whose tile lists are fixed-capacity device buffers (`set_fused(headroom=...)` sizes them), the new pyramid is
        reduced on the device straight into those buffers (`FusedStep.rebind_device`) — the host never learns the tile counts, no
        re-trace, no re-capture, only enqueued work.  A batch of edits ([E, H, W] masks, the same E as the compiled step) takes
        one `sige_reduce_mask_batched` launch per geometry.  Returns True when that happened; `masks_async_ok()` tells (with a
        sync, whenever the caller can afford one) whether every list fit.  Otherwise — no compiled step yet, a batch of another
        size, eager operator-module fallbacks in the step, CPU masks — falls back to the synchronous `set_masks` and returns False.
        The operator modules' own `active_indices` are brought up to date lazily (by a synchronous `set_masks`) if a later call
        cannot use the compiled step."""
        d = self.__dict__
        steps = d.get("_fused_steps", {})
        live = [(k, st) for k, st in steps.items() if st is not None and k[1] == _cache_generation[0] and k[2] == d.get("_sige_cache_id", 0)]
        if d.get("_fused_enabled", False) and d.get("mode") == "sparse" and len(live) == 1 and live[0][1].rebind_device(masks):
            key, st = live[0]
            steps.clear()
            self.timestamp += 1
            steps[(self.timestamp, *key[1:])] = st
            d["_async_masks"] = dict(masks)
            d["_mask_sig"] = None
            return True
        self.set_masks(masks)
        return False

    def masks_async_ok(self) -> bool:
        """Did every tile list of the last `set_masks_async` fit its capacity?  (Synchronises.)"""
        st = self.__dict__.get("fused_step")
        return st is None or st.async_ok()

    def _sync_async_masks(self) -> None:
        """The operator modules' tile lists are stale after `set_masks_async`; bring them up to date (one host sync)."""
        pending = self.__dict__.pop("_async_masks", None)
        if pending is not None:
            self.__dict__.get("_fused_steps", {}).clear()
            self.set_masks(pending)

    def set_mode(self, mode: str):
        self.mode = mode
        for m in self._sige_modules():
            m.set_mode(mode)

    def clear_cache(self):
        bump_cache_generation()
        self.__dict__.get("_fused_steps", {}).clear()
        for m in self._sige_modules():
            m.clear_cache()

    def set_cache_id(self, cache_id: int):
        self.__dict__["_sige_cache_id"] = cache_id
        for m in self._sige_modules():
            m.set_cache_id(cache_id)

    def set_sparse_update(self, sparse_update: bool):
        self.__dict__["_sige_sparse_update"] = sparse_update
        for m in self._sige_modules():
            m.set_sparse_update(sparse_update)

    # ---- fused step -------------------------------------------------------------------------------------------------
    def set_fused(self, enabled: bool = True, **options):
        """Enable / disable the fused step and set its options (see sige_b200.fused.Lowering)."""
        self.__dict__["_fused_enabled"] = bool(enabled)
        self.__dict__["_fused_options"] = dict(options)
        self.__dict__.setdefault("_fused_steps", {}).clear()
        return self

    def _fused_lookup(self, args, kwargs=None):
        d = self.__dict__
        if not d.get("_fused_enabled", False) or d.get("mode") != "sparse" or torch.is_grad_enabled():
            return None
        x = args[0] if args else None
        compute = d.get("_fused_options", {}).get("dtype")
        if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dim() == 4 and (compute or x.dtype) in (torch.float16, torch.bfloat16)):
            return None
        from .. import lazy

        if isinstance(x, lazy.LazyTensor):
            return None
        kwargs = kwargs or {}
        flat = list(args) + [("kw", k) for k in sorted(kwargs)] + [kwargs[k] for k in sorted(kwargs)]
        sig = tuple((tuple(a.shape), a.dtype, str(a.device)) if isinstance(a, torch.Tensor) else ("v", a) for a in flat)
        try:
            hash(sig)
        except TypeError:
            return None
        key = (d.get("timestamp", 0), _cache_generation[0], d.get("_sige_cache_id", 0), sig)
        steps = d.setdefault("_fused_steps", {})
        if key not in steps and d.get("_async_masks") is not None:
            self._sync_async_masks()          # lists installed on the device only: a different call signature needs the modules' lists
            key = (d.get("timestamp", 0), _cache_generation[0], d.get("_sige_cache_id", 0), sig)
        if key not in steps:
            # same cache id, same arguments, a NEW dense pass (new caches and statistics) and / or NEW masks: take them into the
            # compiled step in place (FusedStep.refresh, then FusedStep.rebind)
            for k in [k for k in steps if k[2:] == key[2:] and k[:2] != key[:2]]:
                st = steps.pop(k)
                # (a rebind reloads the cached buffers itself: the refresh before it leaves them)
                if st is None or (k[1] != key[1] and not st.refresh(load=k[0] == key[0])) or (k[0] != key[0] and not st.rebind()):
                    continue
                steps[key] = st
                break
        if key not in steps:
            for k in [k for k in steps if k[0] != key[0] or k[1] != key[1]]:
                del steps[k]           # older masks / older caches: their buffers are garbage now
            from ..fused import FusedStep

            update = d.get("_sige_sparse_update", False)
            try:
                # built with sparse_update off: an eager operator-module node of the step must never write a cache from inside the
                # captured graph (the write-back is the step's own epilogue, `FusedStep.sparse_update`)
                if update:
                    self.set_sparse_update(False)
                steps[key] = FusedStep(self, *args, call_kwargs=kwargs, **d.get("_fused_options", {}))
            except Exception as e:  # noqa: BLE001
                # TraceUnsupported = the forward needs tensor VALUES at trace time; anything else = a pattern the lowering
                # mishandled.  Either way the model must keep working: loud warning, eager operator modules from here on
                # (SIGE_FUSED_STRICT=1 re-raises: the test-suite runs that way).
                if os.environ.get("SIGE_FUSED_STRICT", "0") == "1" and not isinstance(e, lazy.TraceUnsupported):
                    raise
                import warnings

                warnings.warn("sige: this forward does not run as a fused step (%s: %s); using the eager operator modules" % (type(e).__name__, e))
                steps[key] = None
            finally:
                if update:
                    self.set_sparse_update(True)
        return steps[key]

    def _drop_stale_steps(self, keep=None) -> None:
        """A write-back changed the caches of the current cache id without a new cache generation: every other compiled step of that
        id holds buffers cloned from the old contents."""
        steps = self.__dict__.get("_fused_steps", {})
        cid = self.__dict__.get("_sige_cache_id", 0)
        for k in [k for k, st in steps.items() if k[2] == cid and st is not None and st is not keep]:
            del steps[k]

    def __call__(self, *args, **kwargs):
        step = self._fused_lookup(args, kwargs)
        update = self.__dict__.get("_sige_sparse_update", False)
        if step is not None and update and not step.sparse_update_supported:
            step = None                       # this step cannot write back: the operator modules apply the edit
        if step is None:
            self._sync_async_masks()
            if update and self.__dict__.get("mode") == "sparse":
                self._drop_stale_steps()
            return super().__call__(*args, **kwargs)
        self.__dict__["fused_step"] = step
        out = step(*args, **kwargs)
        if update:
            step.sparse_update()
            self._drop_stale_steps(keep=step)
        like = args[0].dtype      # results are fresh tensors in the caller's dtype (the static buffers are reused by the next call)

        def fresh(o):
            return o.to(like, copy=True) if (isinstance(o, torch.Tensor) and o.dtype.is_floating_point) else (o.clone() if isinstance(o, torch.Tensor) else o)

        return fresh(out) if isinstance(out, torch.Tensor) else type(out)(fresh(o) for o in out)
