"""ctypes binding of the C-ABI (include/sige_b200.h) — the only way Python reaches the kernels.

There is NO fallback: if ``sige_b200/lib/libsige_b200.so`` is missing this module raises
``SigeLibraryMissing`` the first time an op is needed (build it with
``python -m sige_b200.build`` or ``__graft_entry__.build()``).

The reference binds its kernels through pybind11 + libtorch
(reference sige/cuda/pybind_cuda.cpp:5-12, loaded by sige/nn/base.py:35-50); here the
boundary is plain C so that any host language can bind it (see INTEGRATION.md).
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_int, c_int32, c_int64, c_void_p

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libsige_b200.so")

F32, F16, BF16 = 0, 1, 2
NCHW, NHWC = 0, 1
ACT_IDENTITY, ACT_SWISH, ACT_RELU = 0, 1, 2
CONV_PDL = 1
CONV_TC5 = 2
CONV_PADDED = 4
CONV_EARLY_RELEASE = 8
CONV_EARLY_SRC0, CONV_EARLY_SRC1, CONV_EARLY_SHORTCUT = 16, 32, 64      # early source groups: (mask & 7) << 4
CONV_PER_IMAGE_OPERANDS = 128       # a batch of independent edits: per-image tile lists over B-image operands
TILE_NONE = -30000


class SigeLibraryMissing(ImportError):
    pass


class SigeError(RuntimeError):
    """A C-ABI call returned non-zero; the message is sige_last_error()."""


class Bcast(Structure):
    _fields_ = [("ptr", c_void_p), ("dims", c_int * 4), ("stride", c_int64 * 4), ("dtype", c_int)]


class ConvSrc(Structure):
    _fields_ = [("ptr", c_void_p), ("C", c_int), ("up", c_int)]


class ConvAux(Structure):
    _fields_ = [("ptr", c_void_p), ("C", c_int), ("c0", c_int), ("scale", c_void_p), ("shift", c_void_p), ("act", c_int)]


class ConvModulation(Structure):
    _fields_ = [("gamma", c_void_p), ("gamma_C", c_int), ("gamma_c0", c_int), ("beta", c_void_p), ("beta_C", c_int), ("beta_c0", c_int),
                ("negative_slope", ctypes.c_float)]


class TileConvPlan(ctypes.Structure):
    _fields_ = [("path", ctypes.c_int), ("bn", ctypes.c_int), ("ksplit", ctypes.c_int), ("deep_ring", ctypes.c_int),
                ("grid_x", ctypes.c_int), ("grid_y", ctypes.c_int), ("grid_z", ctypes.c_int)]


class SparseAttention(Structure):
    _fields_ = [("q", c_void_p), ("k", c_void_p), ("v", c_void_p), ("out", c_void_p),
                ("B", c_int), ("heads", c_int), ("Nq", c_int), ("Nk", c_int), ("D", c_int),
                ("q_stride", c_int64 * 3), ("k_stride", c_int64 * 3), ("v_stride", c_int64 * 3), ("out_stride", c_int64 * 3),
                ("scale", ctypes.c_float), ("dtype", c_int), ("flags", c_int)]


class SeparableBranch(Structure):
    _fields_ = [("dw_weight", c_void_p), ("dw_bias", c_void_p), ("pw_weight", c_void_p), ("pw_bias", c_void_p), ("dst", c_void_p),
                ("dst_is_stack", c_int), ("dH", c_int), ("dW", c_int), ("dst_C", c_int), ("dst_c0", c_int)]


class SeparableConv(Structure):
    _fields_ = [("dtype", c_int), ("src", c_void_p), ("src_is_stack", c_int), ("src_C", c_int), ("src_c0", c_int),
                ("B", c_int), ("H", c_int), ("W", c_int), ("idx", c_void_p), ("N", c_int), ("Cin", c_int), ("Cout", c_int),
                ("offH", c_int), ("offW", c_int), ("nbranch", c_int), ("branch", SeparableBranch * 2), ("flags", c_int)]


class WritebackEntry(Structure):
    _fields_ = [("src", c_void_p), ("dst", c_void_p), ("idx", c_void_p), ("N", c_int), ("B", c_int), ("C", c_int), ("H", c_int), ("W", c_int),
                ("src_dtype", c_int), ("dst_dtype", c_int), ("dst_layout", c_int), ("offH", c_int), ("offW", c_int),
                ("strideH", c_int), ("strideW", c_int), ("Ro", c_int), ("So", c_int)]


WRITEBACK_MAX_ENTRIES = 64


class CacheView(Structure):
    _fields_ = [("dst", c_void_p), ("scale", c_void_p), ("shift", c_void_p), ("act", c_int)]


class CacheLoadEntry(Structure):
    _fields_ = [("src", c_void_p), ("src_dtype", c_int), ("src_layout", c_int), ("src_batch", c_int), ("C", c_int), ("H", c_int), ("W", c_int),
                ("E", c_int), ("raw", c_void_p), ("n_views", c_int), ("view", CacheView * 2)]


CACHE_LOAD_MAX_ENTRIES = 64


class TileConv(Structure):
    _fields_ = [
        ("dtype", c_int),
        ("n_src", c_int),
        ("src", ConvSrc * 2),
        ("B", c_int), ("H", c_int), ("W", c_int),
        ("src_is_stack", c_int),
        ("idx", c_void_p),
        ("N", c_int),
        ("R", c_int), ("S", c_int),
        ("scale", c_void_p), ("shift", c_void_p),
        ("affine_bstride", c_int),
        ("act", c_int),
        ("w_packed", c_void_p), ("bias", c_void_p),
        ("Cin", c_int), ("Cout", c_int), ("kH", c_int), ("kW", c_int), ("stride", c_int),
        ("dst", c_void_p),
        ("dst_is_stack", c_int),
        ("dH", c_int), ("dW", c_int), ("dC", c_int), ("dst_c0", c_int),
        ("offH", c_int), ("offW", c_int),
        ("residual", c_void_p),
        ("rC", c_int), ("res_c0", c_int),
        ("ksplit", c_int), ("flags", c_int),
        ("n_aux", c_int), ("aux", ConvAux * 2),
        ("n_src2", c_int), ("src2", ConvSrc * 2), ("Cin2", c_int), ("w2_packed", c_void_p), ("bias2", c_void_p), ("sc_flags", c_void_p),
        ("idx_per_image", c_int),
        ("src_pixel_stride", c_int),
        ("modulation", POINTER(ConvModulation)),
    ]


# name -> (restype, argtypes); the list is also what tests/test_cabi_symbols.py checks
# against include/sige_b200.h.
_I = c_int
_P = c_void_p
_BP = POINTER(Bcast)
PROTOTYPES = {
    "sige_last_error": (c_char_p, []),
    "sige_abi_version": (_I, []),
    "sige_built_arch": (c_char_p, []),
    "sige_activation_from_name": (_I, [c_char_p]),
    "sige_reduce_mask": (_I, [_P, _I, _I, _I, _I, _I, _I, _I, _I, _P, _I, _P, _P]),
    "sige_reduce_mask_batched": (_I, [_P] + [_I] * 9 + [_P, _I, _P, _P, _P]),
    "sige_reduce_mask_capacity": (_I, [_I] * 8),
    "sige_gather": (_I, [_P, _I, _I, _I, _I, _I, _I, _I, _I, _P, _I, _BP, _BP, _I, _I, _P, _P]),
    "sige_gather_upsampled": (_I, [_P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P, _I, _BP, _BP, _I, _I, _P, _P]),
    "sige_scatter": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P, _I, _BP, _P]),
    "sige_scatter_with_block_residual": (_I, [_P, _P, _P, _P, _P] + [_I] * 14 + [_P, _I, _P, _I, _P]),
    "sige_get_scatter_map": (_I, [_I] * 10 + [_P, _I, _P, _P]),
    "sige_scatter_gather": (_I, [_P, _P] + [_I] * 10 + [_P, _I, _P, _BP, _BP, _I, _I, _P, _P]),
    "sige_pack_conv_weight": (_I, [_P, _I, _I, _I, _I, _I, _P, _I, _P]),
    "sige_tile_conv": (_I, [POINTER(TileConv), _P]),
    "sige_resblock": (_I, [POINTER(TileConv), POINTER(TileConv), _P]),
    "sige_tile_conv_generic": (_I, [_P, _P, _P, _P] + [_I] * 14 + [_P]),
    "sige_tile_conv_plan": (_I, [_P, _P]),
    "sige_conv_in_nhwc": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _P]),
    "sige_conv_in_nhwc_tiles": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _I, _I, _I, _I, _I, _P, _P]),
    "sige_group_norm_fold_workspace": (_I, [_I, _I]),
    "sige_group_norm_fold": (_I, [_P, _I, _I, _I, _I, _I, _I, ctypes.c_float, _P, _P, _P, _P, _P, _I, _P]),
    "sige_conv_out_nhwc": (_I, [_P, _P, _P, _I, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "sige_attention_tokens_supported": (_I, [_I, _I, _I]),
    "sige_attention_tokens": (_I, [_P, _P, _I, _I, _I, _I, _I, _P]),
    "sige_sparse_attention_supported": (_I, [_I, _I]),
    "sige_sparse_attention": (_I, [POINTER(SparseAttention), _P]),
    "sige_spade_modulate": (_I, [_P, c_int64, _P, c_int64, _P, c_int64, _P, c_int64, c_int64, _I, ctypes.c_float, _I, _P]),
    "sige_separable_conv_supported": (_I, [_I, _I, _I, _I]),
    "sige_separable_conv": (_I, [POINTER(SeparableConv), _P]),
    "sige_tile_writeback": (_I, [POINTER(WritebackEntry), _I, _P]),
    "sige_cache_load": (_I, [POINTER(CacheLoadEntry), _I, _I, _P]),
    "sige_debug_set_trace": (_I, [_P]),
    "sige_debug_set_split_halo_buffers": (_I, [_I]),
}

_lib = None


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not os.path.isfile(LIB_PATH):
            raise SigeLibraryMissing(
                "sige_b200: %s not found. Build it with `python -m sige_b200.build` "
                "(needs nvcc; targets sm_90a). There is no CPU or PyTorch fallback." % LIB_PATH
            )
        handle = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in PROTOTYPES.items():
            fn = getattr(handle, name)  # AttributeError if the symbol is missing: loud by design
            fn.restype = res
            fn.argtypes = args
        if handle.sige_abi_version() != 3:
            raise SigeLibraryMissing("sige_b200: ABI version mismatch, rebuild the library")
        _lib = handle
    return _lib


def last_error() -> str:
    return lib().sige_last_error().decode("utf-8", "replace")


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise SigeError("%s failed (rc=%d): %s" % (what, rc, last_error()))
