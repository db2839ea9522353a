"""Deferred execution for the operator surface: a tape of one sparse forward.

The reference's model files call ``Gather`` -> ``SIGEConv2d`` -> ``Scatter`` as three separate modules
(reference diffusion/models/ddpm_arch/sige_fused_unet.py:100-131) with plain torch glue in between
(``torch.cat`` :423, ``F.interpolate`` :223, dense low-resolution blocks :112-123, the attention core
:185-199, ``norm_out``/``conv_out`` :431-433).  To run such an UNMODIFIED forward as one fused launch per
layer, the forward is executed once on ``LazyTensor`` handles (SURVEY.md §7.2): every torch function and
every operator-module call that sees a handle is RECORDED instead of executed, with output shapes
inferred on the meta device.  ``sige_b200.fused`` then lowers the tape to fused sm_90a launches and
replays them (CUDA graph); nothing on the tape is ever executed by this module.

A handle is a real ``torch.Tensor`` subclass (wrapper subclass: shape / dtype / device are genuine, there
is no storage), so model code that asserts on shapes, unpacks ``x.shape`` or checks ``isinstance(x,
torch.Tensor)`` runs unchanged.  Anything that needs VALUES at trace time (``.item()``, ``bool(t)``,
``.cpu()``, in-place writes) raises ``TraceUnsupported`` and the caller falls back to the eager
operator modules.
"""
from __future__ import annotations

from typing import Any, List, Optional, Sequence, Tuple

import torch


class TraceUnsupported(RuntimeError):
    """The forward did something a tape cannot represent; run it through the eager operator modules."""


class Node:
    """One recorded call.  ``op`` is the torch callable, or a string for operator-module calls
    ("sige.gather", "sige.conv", "sige.scatter", "sige.scatter_block_residual", "sige.scatter_gather")."""

    __slots__ = ("index", "op", "args", "kwargs", "outs", "module", "uses", "multi")

    def __init__(self, index: int, op, args, kwargs, module=None):
        self.index, self.op, self.args, self.kwargs, self.module = index, op, args, kwargs, module
        self.outs: List["LazyTensor"] = []
        self.multi = False          # the call returned a tuple / list

    @property
    def name(self) -> str:
        if isinstance(self.op, str):
            return self.op
        return getattr(self.op, "__name__", None) or str(self.op)

    def __repr__(self) -> str:
        return "<%d %s -> %s>" % (self.index, self.name, [tuple(o.shape) for o in self.outs])


class Tape:
    def __init__(self):
        self.nodes: List[Node] = []
        self.inputs: List["LazyTensor"] = []

    def add(self, op, args, kwargs, module=None) -> Node:
        n = Node(len(self.nodes), op, args, kwargs, module)
        self.nodes.append(n)
        return n


_ACTIVE: Optional[Tape] = None

# metadata queries answered from the handle itself (never recorded)
_META_METHODS = {
    "size", "dim", "ndimension", "numel", "nelement", "stride", "is_contiguous", "is_floating_point", "is_complex",
    "element_size", "storage_offset", "get_device", "type", "data_ptr", "__len__", "__format__", "__repr__", "__str__",
    "is_cuda.__get__", "requires_grad_", "detach", "__hash__", "is_quantized.__get__",
}
_VALUE_METHODS = {"item", "tolist", "numpy", "cpu", "__bool__", "__int__", "__float__", "__index__", "__array__", "__contains__",
                  "__setitem__", "copy_", "nonzero", "unique", "any", "all", "backward"}


def _fname(func) -> str:
    n = getattr(func, "__name__", None)
    if n == "__get__":
        owner = getattr(func, "__self__", None)
        return "%s.__get__" % getattr(owner, "__name__", "?")
    return n or str(func)


def _tree_map(fn, obj):
    if isinstance(obj, (list, tuple)):
        return type(obj)(_tree_map(fn, o) for o in obj)
    if isinstance(obj, dict):
        return {k: _tree_map(fn, v) for k, v in obj.items()}
    return fn(obj)


def _to_meta(o):
    if isinstance(o, LazyTensor):
        return torch.empty_strided(o.shape, o.stride(), dtype=o.dtype, device="meta")
    if isinstance(o, torch.Tensor):
        with torch._C.DisableTorchFunctionSubclass():
            return torch.empty_strided(o.shape, o.stride(), dtype=o.dtype, device="meta")
    if isinstance(o, torch.device):
        return torch.device("meta")
    return o


class LazyTensor(torch.Tensor):
    """Handle of a value on the tape.  ``node``/``slot`` say which call produced it (inputs: node None)."""

    @staticmethod
    def __new__(cls, shape, dtype, device, strides=None, node: Optional[Node] = None, slot: int = 0, tape: Optional[Tape] = None):
        t = torch.Tensor._make_wrapper_subclass(cls, tuple(shape), strides=strides, dtype=dtype, device=device, requires_grad=False)
        t.node, t.slot, t.tape = node, slot, tape
        return t

    @classmethod
    def __torch_dispatch__(cls, func, types, args=(), kwargs=None):
        # every op is caught one level up, in __torch_function__; reaching the dispatcher means a code path ran with
        # torch-function handling disabled, which a tape cannot see
        raise TraceUnsupported("%s reached the dispatcher on a lazy tensor" % (func,))

    def __repr__(self):  # never touches data
        return "LazyTensor(shape=%s, dtype=%s, from=%s)" % (tuple(self.shape), self.dtype, self.node)

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        name = _fname(func)
        if name.endswith(".__get__"):
            attr = name[:-8]
            if attr in ("shape", "dtype", "device", "ndim", "is_cuda", "layout", "requires_grad", "is_meta", "is_sparse", "is_quantized",
                        "names", "grad", "grad_fn", "is_leaf", "is_cpu", "itemsize", "nbytes", "is_mps", "is_xpu", "is_nested", "is_mkldnn"):
                with torch._C.DisableTorchFunctionSubclass():
                    return func(*args, **kwargs)
            if attr in ("T", "mT", "H", "mH", "real"):
                return _record(func, args, kwargs)
            raise TraceUnsupported("attribute %s of a lazy tensor" % attr)
        if name == "type" and (len(args) > 1 or kwargs):
            return _record(func, args, kwargs)          # x.type(dtype) is a cast, x.type() a query
        if name in _META_METHODS:
            if name in ("data_ptr",):
                raise TraceUnsupported("data_ptr() of a lazy tensor")
            if name == "detach":
                return args[0]
            if name in ("__repr__", "__str__", "__format__"):
                return LazyTensor.__repr__(args[0])
            if name == "__hash__":
                return id(args[0])
            with torch._C.DisableTorchFunctionSubclass():
                return func(*args, **kwargs)
        if name in _VALUE_METHODS:
            raise TraceUnsupported("%s needs tensor values at trace time" % name)
        if name.endswith("_") and not name.endswith("__") and name not in ("requires_grad_",):
            raise TraceUnsupported("in-place op %s on a lazy tensor" % name)
        if name.startswith("__i") and name.endswith("__") and name not in ("__invert__", "__index__", "__int__"):
            raise TraceUnsupported("in-place op %s on a lazy tensor" % name)
        if kwargs.get("out") is not None:
            raise TraceUnsupported("out= on a lazy tensor op")
        return _record(func, args, kwargs)


def _record(func, args, kwargs, module=None):
    tape = _ACTIVE
    if tape is None:
        raise TraceUnsupported("lazy tensor used outside its trace (%s)" % _fname(func))
    with torch._C.DisableTorchFunctionSubclass():
        margs, mkwargs = _tree_map(_to_meta, args), _tree_map(_to_meta, kwargs)
        try:
            mout = func(*margs, **mkwargs)
        except Exception as e:  # noqa: BLE001
            raise TraceUnsupported("shape inference failed for %s: %r" % (_fname(func), e)) from e
    node = tape.add(func, args, kwargs, module)
    return wrap_outputs(node, mout, _device_of(args, kwargs))


def _device_of(args, kwargs):
    found = []

    def visit(o):
        if isinstance(o, LazyTensor) and not found:
            found.append(o.device)
        return o

    _tree_map(visit, args)
    _tree_map(visit, kwargs)
    return found[0] if found else torch.device("cpu")


def wrap_outputs(node: Node, mout, device):
    tape = _ACTIVE

    def wrap(m):
        if isinstance(m, torch.Tensor):
            lt = LazyTensor(m.shape, m.dtype, device, strides=m.stride(), node=node, slot=len(node.outs), tape=tape)
            node.outs.append(lt)
            return lt
        return m

    if isinstance(mout, (tuple, list)):
        node.multi = True
        return type(mout)(wrap(m) for m in mout) if not hasattr(mout, "_fields") else type(mout)(*[wrap(m) for m in mout])
    return wrap(mout)


def record_module_call(kind: str, module, args: Sequence[Any], out_shape: Tuple[int, ...], like: "LazyTensor") -> "LazyTensor":
    """Record an operator-module call (Gather / SIGEConv2d / Scatter* / ScatterGather in sparse mode) as ONE node."""
    tape = _ACTIVE
    if tape is None:
        raise TraceUnsupported("lazy tensor used outside its trace (%s)" % kind)
    node = tape.add(kind, tuple(args), {}, module)
    lt = LazyTensor(out_shape, like.dtype, like.device, node=node, slot=0, tape=tape)
    node.outs.append(lt)
    return lt


def is_lazy(*ts) -> bool:
    return any(isinstance(t, LazyTensor) for t in ts)


class tracing:
    """Context manager: ``with tracing() as tape:`` — LazyTensor ops are recorded on ``tape``."""

    def __enter__(self) -> Tape:
        global _ACTIVE
        if _ACTIVE is not None:
            raise RuntimeError("nested lazy traces are not supported")
        _ACTIVE = Tape()
        return _ACTIVE

    def __exit__(self, *exc):
        global _ACTIVE
        _ACTIVE = None
        return False


def make_input(t: torch.Tensor, tape: Tape, dtype: Optional[torch.dtype] = None) -> LazyTensor:
    lt = LazyTensor(t.shape, dtype or t.dtype, t.device, strides=None, node=None, slot=len(tape.inputs), tape=tape)
    tape.inputs.append(lt)
    return lt
