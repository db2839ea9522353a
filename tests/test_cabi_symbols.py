"""The C-ABI shared library loads without a GPU and exports every function include/*.h declares;
the ctypes prototype table covers exactly that set.  No compute call is made here."""
import ctypes
import os
import re

from conftest import REPO


def _declared():
    names = set()
    inc = os.path.join(REPO, "include")
    for f in os.listdir(inc):
        if f.endswith(".h"):
            src = open(os.path.join(inc, f)).read()
            src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
            names |= set(re.findall(r"\b(sige_[a-z0-9_]+)\s*\(", src))
    return names


def test_library_exports_every_declared_symbol(cabi_lib):
    lib = ctypes.CDLL(cabi_lib)
    declared = _declared()
    assert len(declared) >= 14
    for name in sorted(declared):
        assert hasattr(lib, name), "libsige_b200.so does not export %s" % name


def test_prototype_table_matches_the_abi_3_header(cabi_lib):
    from sige_b200 import _cabi

    assert set(_cabi.PROTOTYPES) == _declared()
    lib = _cabi.lib()
    assert lib.sige_abi_version() == 3
    assert lib.sige_built_arch() == b"sm_90a"
    assert lib.sige_activation_from_name(b"identity") == 0
    assert lib.sige_activation_from_name(b"swish") == 1
    assert lib.sige_activation_from_name(b"gelu") == -1     # the reference has UB here (common.cpp:22)
    assert lib.sige_reduce_mask_capacity(256, 256, 6, 6, 4, 4, 1, 1) == 65 * 65


def test_argument_errors_are_reported_not_crashes(cabi_lib):
    """Bad arguments return non-zero with a message before any CUDA call (safe without a GPU)."""
    from sige_b200 import _cabi

    lib = _cabi.lib()
    rc = lib.sige_gather(None, 0, 7, 1, 1, 4, 4, 2, 2, None, 1, None, None, 0, 0, None, None)
    assert rc != 0 and b"layout" in lib.sige_last_error()
    assert lib.sige_gather(None, 0, 0, 1, 1, 4, 4, 2, 2, None, 0, None, None, 0, 0, None, None) == 0   # N == 0: no-op
    rc = lib.sige_tile_conv(None, None)
    assert rc != 0 and b"null" in lib.sige_last_error()


def test_missing_library_is_loud(monkeypatch, tmp_path):
    from sige_b200 import _cabi

    monkeypatch.setattr(_cabi, "_lib", None)
    monkeypatch.setattr(_cabi, "LIB_PATH", str(tmp_path / "nope.so"))
    try:
        _cabi.lib()
    except _cabi.SigeLibraryMissing as e:
        assert "no CPU or PyTorch fallback" in str(e)
    else:
        raise AssertionError("expected SigeLibraryMissing")


def test_attention_shape_predicate_is_pure_host_logic(cabi_lib):
    """sige_attention_tokens_supported() never touches the device: the shapes the fused attention core takes
    (64 keys per CTA, clusters of 1 / 2 / 4 key slices; 256 or 512 channels; 16-bit storage)."""
    h = ctypes.CDLL(cabi_lib)
    f = h.sige_attention_tokens_supported
    f.restype, f.argtypes = ctypes.c_int, [ctypes.c_int] * 3
    F32, F16, BF16 = 0, 1, 2
    assert f(256, 512, F16) == 1 and f(64, 512, BF16) == 1 and f(128, 256, F16) == 1
    assert f(256, 512, F32) == 0      # fp32 goes through the library path
    assert f(100, 512, F16) == 0 and f(512, 512, F16) == 0 and f(256, 192, F16) == 0 and f(0, 512, F16) == 0


def test_sparse_attention_predicate_and_argument_checks_need_no_device(cabi_lib):
    """sige_sparse_attention_supported() is host logic; the entry point validates its descriptor before touching the device
    (null descriptor, unsupported head dim, a scale that is not positive and finite, misaligned strides) and treats Nq == 0
    as a no-op."""
    from sige_b200 import _cabi

    h = _cabi.lib()
    F32, F16, BF16 = 0, 1, 2
    for d in (32, 40, 64, 80, 128, 160):
        assert h.sige_sparse_attention_supported(d, F16) == 1 and h.sige_sparse_attention_supported(d, BF16) == 1
    assert h.sige_sparse_attention_supported(40, F32) == 0 and h.sige_sparse_attention_supported(48, F16) == 0 and h.sige_sparse_attention_supported(320, F16) == 0
    a = _cabi.SparseAttention()
    a.B, a.heads, a.Nq, a.Nk, a.D, a.dtype, a.scale = 1, 8, 0, 77, 40, F16, 0.158
    assert h.sige_sparse_attention(ctypes.byref(a), None) == 0            # no query: no-op, pointers not looked at
    a.D = 48
    assert h.sige_sparse_attention(ctypes.byref(a), None) != 0 and b"head dim" in h.sige_last_error()
    a.D, a.Nq = 40, 16
    assert h.sige_sparse_attention(ctypes.byref(a), None) != 0 and b"null buffer" in h.sige_last_error()
    assert h.sige_sparse_attention(None, None) != 0
    # scale = 0 would turn the masked keys of a partial last block into -inf * 0 = NaN, scale < 0 would take the running
    # maximum at the wrong end: refused, as are NaN and infinities, with or without queries (the pointers here are not device
    # memory, so a launch would fault)
    P = 0x10000
    a.q = a.k = a.v = a.out = P
    for nq in (0, 16):
        for bad in (0.0, -0.0, -0.158, float("nan"), float("inf"), float("-inf")):
            a.Nq, a.scale = nq, bad
            assert h.sige_sparse_attention(ctypes.byref(a), None) != 0, (nq, bad)
            assert b"scale" in h.sige_last_error() and b"positive and finite" in h.sige_last_error()
    a.Nq, a.scale = 0, 1e-30                                              # tiny but positive: accepted (a no-op here)
    assert h.sige_sparse_attention(ctypes.byref(a), None) == 0


def _conv_desc(n_tiles, cin, cout, k, *, stride=1, cin2=0, ksplit=0, res=64):
    from sige_b200 import _cabi

    d = _cabi.TileConv()
    d.dtype = _cabi.F16
    d.B, d.H, d.W = 1, res, res
    d.n_src = 1
    d.src[0].C, d.src[0].up = cin, 0
    d.src_is_stack = 0
    d.N = n_tiles
    d.R = d.S = {(3, 1): 6, (1, 1): 4, (3, 2): 5}[(k, stride)]
    d.Cin, d.Cout, d.kH, d.kW, d.stride = cin, cout, k, k, stride
    d.dst_is_stack, d.dH, d.dW, d.dC = 0, res // stride, res // stride, cout
    d.ksplit = ksplit
    d.flags = _cabi.CONV_PDL | _cabi.CONV_TC5
    if cin2:
        d.n_src2, d.Cin2 = 1, cin2
        d.src2[0].C = cin2
    return d


def test_tile_conv_launch_plan_heuristics(cabi_lib):
    """sige_tile_conv_plan: the host-side choice of tile width, split-K (= cluster size) and ring flavour of the wgmma
    kernel, on the layer shapes of a DDPM-256 step.  Invariants: one wave only (132 / 132 / 120 / 120 co-resident CTAs on an H100
    for cluster sizes 1 / 2 / 4 / 8), every K slice non-empty, deep ring exactly for split narrow 3x3 launches."""
    from sige_b200 import _cabi

    lib = _cabi.lib()
    cap = {1: 132, 2: 132, 4: 120, 8: 120}

    def plan(d):
        p = _cabi.TileConvPlan()
        assert lib.sige_tile_conv_plan(ctypes.byref(d), ctypes.byref(p)) == 0
        return p

    # known points (1.2 % edit: 64 tiles at 256^2 ... 4 tiles at 8^2)
    p = plan(_conv_desc(4, 512, 512, 3))
    assert (p.path, p.bn, p.ksplit, p.deep_ring, p.grid_x, p.grid_y, p.grid_z) == (1, 64, 8, 1, 1, 8, 8)
    p = plan(_conv_desc(16, 512, 512, 3))
    assert (p.bn, p.ksplit, p.deep_ring, p.grid_x * p.grid_y * p.grid_z) == (64, 4, 1, 64)
    p = plan(_conv_desc(64, 128, 128, 3, res=256))
    assert (p.bn, p.ksplit, p.deep_ring) == (64, 4, 1)
    p = plan(_conv_desc(1296, 128, 128, 3, res=256))        # 30 % edit: wide tiles, no split
    assert (p.bn, p.ksplit, p.deep_ring, p.grid_x) == (128, 1, 0, 162)
    p = plan(_conv_desc(16, 512, 1536, 1))                  # qkv of the 16x16 attention block
    assert p.path == 1 and p.bn == 64 and p.ksplit in (1, 2) and p.deep_ring == 0
    p = plan(_conv_desc(16, 512, 512, 3, stride=2))                    # stride-2 downsample (5x5 -> 2x2 tiles): wgmma kernel, 32 tiles per CTA
    assert (p.path, p.bn, p.deep_ring, p.grid_x, p.grid_y) == (1, 64, 0, 1, 8) and p.ksplit == 8
    assert plan(_conv_desc(64, 256, 256, 3, stride=2)).grid_x == 2
    d2 = _conv_desc(16, 256, 256, 3, stride=2)
    d2.act = 1                                                         # ... a pre-op in the gather stage of that geometry: mma.sync kernel
    assert plan(d2).path == 0
    assert plan(_conv_desc(16, 96, 128, 3)).path == 0                  # Cin not a multiple of 64
    assert plan(_conv_desc(4, 512, 512, 3, ksplit=2)).ksplit == 2      # an explicit request is honoured
    # sweep
    for n_tiles in (1, 4, 13, 16, 32, 64, 100, 256, 1296, 4096):
        for cin, cout in ((128, 128), (128, 256), (256, 256), (512, 512), (1024, 512), (768, 256)):
            for k in (1, 3):
                for cin2 in ((0, cin) if k == 3 else (0,)):
                    p = plan(_conv_desc(n_tiles, cin, cout, k, cin2=cin2, res=256))
                    assert p.path == 1 and p.bn in (64, 128) and p.ksplit in cap
                    ctas = p.grid_x * p.grid_y * p.grid_z
                    assert p.grid_x == (n_tiles + 7) // 8 and p.grid_y == cout // p.bn and p.grid_z == p.ksplit
                    if p.ksplit > 1:
                        assert ctas <= cap[p.ksplit] and p.bn == 64
                    steps = (cin // 64) * (k * k // (3 if (k == 3 and p.bn == 64) else 1)) + cin2 // 64
                    assert p.ksplit <= steps
                    assert p.deep_ring == int(p.bn == 64 and k == 3 and p.ksplit > 1)
