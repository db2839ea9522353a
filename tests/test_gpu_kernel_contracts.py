"""The separable SPADE conv, the dense glue kernels and the attention core against the float64 restatements of their C-ABI
contracts (tests/kernel_contracts.py), in fp16 and bf16.

Every launch must be within the per-element bound on every element it writes, leave every other element of every buffer (guard
bands included) and every input bitwise unchanged, and be bitwise equal on a repeat; where the entry point takes SIGE_CONV_PDL,
the launch with programmatic dependent launch must be bitwise equal to the one without.  The worst error / bound ratio of each
launch is printed (pytest -s), so the headroom measured on the device is on record.
"""
from ctypes import byref

import pytest
import torch

import kernel_contracts as kc
from kernel_contracts import _launch, _run_and_check
from tile_conv_contract import DTYPE_NAME

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])


def _lib():
    from sige_b200 import _cabi

    return _cabi.lib()


# ---------------------------------------------------------------------------------------------------------------- separable
@DTYPES
@pytest.mark.parametrize("spec", kc.SEP_CASES, ids=lambda s: s.name)
def test_separable_conv_matches_the_float64_contract(spec, dtype):
    case = kc.make_sep(spec, dtype, DEV)
    expects = kc.sep_reference(case)
    d = kc.sep_descriptor(case)
    lib = _lib()

    def call(flags):
        d.flags = flags
        return lib.sige_separable_conv(byref(d), torch.cuda.current_stream().cuda_stream)

    _run_and_check("separable", "%s %s" % (spec.name, DTYPE_NAME[dtype]), case, expects, call, (0, kc.PDL))


@DTYPES
def test_separable_stack_destination_keeps_padding_rows(dtype):
    """The padding rule, pinned: with a tile list, the stack rows of SIGE_TILE_NONE entries are left as they were (bitwise),
    for a stack source and for a buffer source."""
    for name in ("mixed_stack_buf", "mixed_buf_stack_stacksrc"):
        spec = next(s for s in kc.SEP_CASES if s.name == name)
        case = kc.make_sep(spec, dtype, DEV)
        d = kc.sep_descriptor(case)
        init = kc.snapshot(case.buffers())
        got = _launch(case, init, lambda: _lib().sige_separable_conv(byref(d), torch.cuda.current_stream().cuda_stream))
        pad = (case.idx[:, 0] == kc.TILE_NONE).repeat(spec.B)
        assert bool(pad.any())
        for i, (kind, _, _) in enumerate(spec.dsts):
            if kind != "stack":
                continue
            g = case.dst[i]
            now = got["dst%d" % i][g.off:g.off + g.view.numel()].view(*g.view.shape)
            was = init["dst%d" % i][g.off:g.off + g.view.numel()].view(*g.view.shape)
            assert torch.equal(kc.bits(now[pad]), kc.bits(was[pad])), "%s: a padding row of the stack destination was written" % name
            assert not torch.equal(kc.bits(now[~pad]), kc.bits(was[~pad]))


# ---------------------------------------------------------------------------------------------------------------- conv_in
@DTYPES
@pytest.mark.parametrize("spec", kc.CONV_IN_CASES, ids=lambda s: s.name)
def test_conv_in_matches_the_float64_contract(spec, dtype):
    case = kc.make_conv_in(spec, dtype, DEV)
    expects = kc.conv_in_reference(case)
    lib = _lib()
    _run_and_check("conv_in", "%s %s" % (spec.name, DTYPE_NAME[dtype]), case, expects, lambda flags: kc.conv_in_call(case, lib))


# ---------------------------------------------------------------------------------------------------------------- GroupNorm fold
@DTYPES
@pytest.mark.parametrize("spec", kc.GN_CASES, ids=lambda s: s.name)
def test_group_norm_fold_matches_the_float64_contract(spec, dtype):
    case = kc.make_gn(spec, dtype, DEV)
    expects, bounds = kc.gn_reference(case)
    lib = _lib()
    label = "%s %s" % (spec.name, DTYPE_NAME[dtype])
    got = _run_and_check("gn_fold", label, case, expects, lambda flags: kc.gn_call(case, lib))
    for k, g in case.buffers().items():
        g.flat.copy_(got[k])
    r = kc.gn_folded_check(label, case, bounds)
    print("[kernel contract] %-10s %-52s x*scale + shift vs group_norm: worst |err| / bound %.3f" % ("gn_fold", label, r))
    # a workspace one float short: refused, nothing launched
    init = kc.snapshot(case.buffers())
    rc = kc.gn_call(case, lib, workspace_floats=case.ws.view.numel() - 1)
    torch.cuda.synchronize()
    assert rc != 0 and "workspace too small" in _lib().sige_last_error().decode()
    assert all(torch.equal(kc.bits(g.flat), kc.bits(init[k])) for k, g in case.buffers().items())


# ---------------------------------------------------------------------------------------------------------------- conv_out
@DTYPES
@pytest.mark.parametrize("spec", kc.CONV_OUT_CASES, ids=lambda s: s.name)
def test_conv_out_matches_the_float64_contract(spec, dtype):
    case = kc.make_conv_out(spec, dtype, DEV)
    expects = kc.conv_out_reference(case)
    lib = _lib()
    path = "per-element" if kc.conv_out_per_element(spec.C) else "octet"
    _run_and_check("conv_out", "%s %s (%s)" % (spec.name, DTYPE_NAME[dtype], path), case, expects, lambda flags: kc.conv_out_call(case, lib))


# ---------------------------------------------------------------------------------------------------------------- attention
@DTYPES
@pytest.mark.parametrize("spec", kc.ATTN_CASES, ids=lambda s: s.name)
def test_attention_tokens_matches_the_float64_contract(spec, dtype):
    case = kc.make_attn(spec, dtype, DEV)
    expects = kc.attn_reference(case)
    lib = _lib()
    _run_and_check("attention", "%s %s" % (spec.name, DTYPE_NAME[dtype]), case, expects, lambda flags: kc.attn_call(case, lib, flags),
                   (0, kc.PDL))
