"""The sparse-query attention, SPADE modulation and the tile ops against the float64 restatements of their C-ABI contracts
(tests/step_kernel_contracts.py).

Every launch must be within the per-element bound on every element it writes, leave every other element of every buffer (guard
bands included) and every input bitwise unchanged, and be bitwise equal on a repeat.  The arithmetic must not depend on the
operands' layout (attention) or on the kernel variant the pointers select (the tile ops' scalar and vector NHWC paths), and a
launch replayed from a CUDA graph must equal the stream launch.  The worst error / bound ratio of each launch is printed
(pytest -s).
"""
from dataclasses import replace

import pytest
import torch

import kernel_contracts as kc
import step_kernel_contracts as sk
from kernel_contracts import _launch, _run_and_check

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NAME = {torch.float32: "f32", torch.float16: "f16", torch.bfloat16: "bf16"}
DT16 = pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=["f32", "f16", "bf16"])


def _lib():
    from sige_b200 import _cabi

    return _cabi.lib()


def _window(g: kc.Guarded, flat: torch.Tensor) -> torch.Tensor:
    return flat[g.off:g.off + g.view.numel()].view(*g.view.shape)


# ---------------------------------------------------------------------------------------------------------------- attention
@DT16
@pytest.mark.parametrize("spec", sk.SATTN_CASES, ids=lambda s: s.name)
def test_sparse_attention_matches_the_float64_contract(spec, dtype):
    case = sk.make_sattn(spec, dtype, DEV)
    expects = sk.sattn_reference(case)
    d = sk.sattn_descriptor(case)
    lib = _lib()
    _run_and_check("sparse_att", "%s %s" % (spec.name, NAME[dtype]), case, expects, lambda flags: sk.sattn_call(case, lib, d))


@DT16
@pytest.mark.parametrize("spec", [s for s in sk.SATTN_CASES if s.layout != "bhnd" and s.Nk <= 1024], ids=lambda s: s.name)
def test_sparse_attention_layout_does_not_change_the_bits(spec, dtype):
    """The same values addressed in place ("b n (h d)", kv pairs) and contiguous: bitwise the same output."""
    lib = _lib()
    outs = []
    for lay in (spec.layout, "bhnd"):
        case = sk.make_sattn(spec, dtype, DEV, layout=lay)
        d = sk.sattn_descriptor(case)
        got = _launch(case, kc.snapshot(case.buffers()), lambda: sk.sattn_call(case, lib, d))
        w = _window(case.out, got["out"])
        outs.append(w if lay == "bhnd" else w[..., :spec.D].permute(0, 2, 1, 3))
    assert torch.equal(kc.bits(outs[0]), kc.bits(outs[1])), "%s: the %s layout changed the result" % (spec.name, spec.layout)


# ---------------------------------------------------------------------------------------------------------------- SPADE
@pytest.mark.parametrize("spec", sk.SPADE_CASES, ids=lambda s: s.name)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=["f32", "f16", "bf16"])
def test_spade_modulate_matches_the_float64_contract(spec, dtype):
    case = sk.make_spade(spec, dtype, DEV)
    expects = sk.spade_reference(case)
    lib = _lib()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    trips = sk.spade_iterations(spec.pixels * case.C // case.vec, sms)
    got = _run_and_check("spade", "%s %s (%d grid-stride trips)" % (spec.name, NAME[dtype], trips), case, expects,
                         lambda flags: sk.spade_call(case, lib))
    if spec.identity:
        assert torch.equal(kc.bits(_window(case.out, got["out"])[:, :case.C]), kc.bits(case.x)), "%s: x * (1 + 0) + 0 is not x" % spec.name


# ---------------------------------------------------------------------------------------------------------------- tile ops
def _device_map(case: sk.TileCase) -> torch.Tensor:
    s = case.spec
    m = torch.empty(s.H, s.W, 3, dtype=torch.int32, device=DEV)
    idx = case.idx["idx"]
    rc = _lib().sige_get_scatter_map(s.H, s.W, 6, 6, 3, 3, 1, 1, 1, 1, idx.data_ptr(), idx.shape[0], m.data_ptr(), sk._stream())
    torch.cuda.synchronize()
    assert rc == 0
    return m


@DTYPES
@pytest.mark.parametrize("spec", sk.TILE_CASES, ids=lambda s: s.name)
def test_tile_op_matches_the_float64_contract(spec, dtype):
    case = sk.make_tile(spec, dtype, DEV)
    path = sk.tile_path(spec, dtype)
    ptrs = [case.out.view.data_ptr()] + [case.t[k].data_ptr() for k in ("x", "y") if k in case.t]
    vec = 16 // case.out.flat.element_size()
    assert (path == "vec") == (spec.layout == "nhwc" and spec.C % vec == 0 and all(p % 16 == 0 for p in ptrs)), spec.name
    if spec.op == "scatter_gather":
        m = _device_map(case)
        assert torch.equal(m, case.idx["map"]), "%s: get_scatter_map differs from its restatement" % spec.name
        case.idx["map"] = m                                                                # the kernel's own map
    expects = sk.tile_reference(case)
    lib = _lib()
    keep = []
    _run_and_check("tile_ops", "%s %s (%s)" % (spec.name, NAME[dtype], path), case, expects, lambda flags: sk.tile_call(case, lib, keep))


@DTYPES
@pytest.mark.parametrize("spec", [s for s in sk.TILE_CASES if sk.tile_path(s, torch.float16) == "vec"], ids=lambda s: s.name)
def test_tile_op_scalar_path_matches_the_vector_path(spec, dtype):
    """The same inputs through the 16-byte-vector NHWC kernel and, with the destination one element off alignment, the scalar
    one: bitwise the same written elements."""
    lib = _lib()
    res = []
    for mis in (False, True):
        case = sk.make_tile(replace(spec, misalign=mis), dtype, DEV)
        assert sk.tile_path(case.spec, dtype) == ("scalar" if mis else "vec")
        (e,) = sk.tile_reference(case)
        keep = []
        got = _launch(case, kc.snapshot(case.buffers()), lambda: sk.tile_call(case, lib, keep))
        res.append(_window(case.out, got["out"])[_window(case.out, e.written)])
    assert torch.equal(kc.bits(res[0]), kc.bits(res[1])), "%s: the scalar NHWC path differs from the vector path" % spec.name


# ---------------------------------------------------------------------------------------------------------------- CUDA graphs
def test_graph_replay_matches_the_stream_launch():
    lib = _lib()
    spec = next(s for s in sk.SATTN_CASES if s.name == "d40_q65_k130_random_bnhd")
    case = sk.make_sattn(spec, torch.float16, DEV)
    d = sk.sattn_descriptor(case)
    kc.graph_equals_stream(case, lambda: sk.sattn_call(case, lib, d))
    spec = next(s for s in sk.TILE_CASES if s.name.startswith("g_nhwc_1111_afff32"))
    for dt in (torch.bfloat16, torch.float32):
        case = sk.make_tile(spec, dt, DEV)
        keep = []
        kc.graph_equals_stream(case, lambda: sk.tile_call(case, lib, keep))
