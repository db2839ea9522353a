"""`sige_cache_load` on the GPU against the torch chain it replaces (the restatement `Buf.restore` / `Lowering.init_view` keep):
raw copies and identity / swish views bitwise equal, guard bands around every destination untouched."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GUARD = 64          # elements of guard band on both sides of every destination (a multiple of 16 bytes)


def _guarded(shape, dtype, gen):
    E, C, H, W = shape
    n = E * C * H * W
    store = torch.randn(n + 2 * GUARD, generator=gen, device=DEV).to(dtype)
    keep = store.clone()
    t = store[GUARD:GUARD + n].view(E, H, W, C).permute(0, 3, 1, 2)        # channels-last [E, C, H, W]
    return t, store, keep


def _torch_chain(src, sc, sh, act, like):
    z = src.float()
    if sc is not None:
        z = z * sc.view(1, -1, 1, 1)
    if sh is not None:
        z = z + sh.view(1, -1, 1, 1)
    if act == "swish":
        z = z * torch.sigmoid(z)
    return torch.empty_like(like).copy_(z.expand(like.shape[0], *z.shape[1:]))


def _bits(t):
    return t.contiguous().view(torch.int16)


def _entries(seed, n):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    rng = torch.Generator().manual_seed(seed)

    def pick(xs):
        return xs[int(torch.randint(len(xs), (1,), generator=rng))]

    out = []
    for k in range(n):
        C = 8 * int(torch.randint(1, 129, (1,), generator=rng))
        H, W = 2 * int(torch.randint(1, 20, (1,), generator=rng)) + 1, 2 * int(torch.randint(1, 20, (1,), generator=rng)) + 1
        E = pick([1, 3, 8])
        B = pick([1, E])
        src_dt = pick([torch.float32, torch.float16, torch.bfloat16])
        src = torch.randn(B, C, H, W, generator=gen, device=DEV).mul(3).to(src_dt)
        if pick([0, 1]):
            src = src.contiguous(memory_format=torch.channels_last)
        nv = pick([0, 1, 2])
        raw = k % 5 != 0 or nv == 0
        out.append((src, E, raw, [(pick([None, "s"]), pick([None, "h"]), pick(["identity", "swish"])) for _ in range(nv)]))
    return out, gen


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_cache_load_matches_the_torch_chain(dtype, seed):
    from sige_b200 import ops

    specs, gen = _entries(seed, 70)             # more entries than one launch takes
    entries, checks, guards = [], [], []
    for (src, E, want_raw, views) in specs:
        B, C, H, W = src.shape
        raw = None
        if want_raw:
            raw, store, keep = _guarded((E, C, H, W), dtype, gen)
            guards.append((store, keep))
            checks.append((raw, _torch_chain(src, None, None, "identity", raw), "raw"))
        vs = []
        for (sc, sh, act) in views:
            v, store, keep = _guarded((E, C, H, W), dtype, gen)
            guards.append((store, keep))
            sc = None if sc is None else torch.rand(C, generator=gen, device=DEV) * 2 - 0.5
            sh = None if sh is None else torch.randn(C, generator=gen, device=DEV)
            vs.append((v, sc, sh, act))
            checks.append((v, _torch_chain(src, sc, sh, act, v), act))
        entries.append((src, raw, vs))
    ops.cache_load(entries, dtype)
    torch.cuda.synchronize()
    worst = 0
    for (got, want, kind) in checks:
        if kind == "swish" and not torch.equal(_bits(got), _bits(want)):
            worst = max(worst, int((_bits(got).int() - _bits(want).int()).abs().max()))
        assert torch.equal(_bits(got), _bits(want)), "%s view differs by %d ulp at most" % (kind, worst)
    for store, keep in guards:
        assert torch.equal(store[:GUARD], keep[:GUARD]) and torch.equal(store[-GUARD:], keep[-GUARD:]), "a guard band was written"


def test_cache_load_destination_beyond_two_gigabytes():
    from sige_b200 import ops

    E, C, H, W = 8, 1024, 363, 363          # 8 * 1024 * 363 * 363 * 2 bytes = 2.16 GB > 2^31
    gen = torch.Generator(device=DEV).manual_seed(7)
    src = torch.randn(1, C, H, W, generator=gen, device=DEV)
    raw, store, keep = _guarded((E, C, H, W), torch.float16, gen)
    assert raw.numel() * 2 > 2 ** 31
    ops.cache_load([(src, raw, [])], torch.float16)
    want = src.to(torch.float16)
    for e in (0, E - 1):
        assert torch.equal(raw[e], want[0]), "image %d" % e
    assert torch.equal(store[:GUARD], keep[:GUARD]) and torch.equal(store[-GUARD:], keep[-GUARD:])


def test_cache_load_rejects_bad_entries_and_does_nothing_for_none():
    from sige_b200 import _cabi, ops

    ops.cache_load([], torch.float16)
    src = torch.zeros(1, 12, 4, 4, device=DEV)
    raw = torch.empty(1, 12, 4, 4, device=DEV, dtype=torch.float16, memory_format=torch.channels_last)
    with pytest.raises(ValueError):
        ops.cache_load([(src, raw, [])], torch.float16)            # C not a multiple of 8
    e = _cabi.CacheLoadEntry()
    e.src, e.src_dtype, e.src_layout, e.src_batch, e.C, e.H, e.W, e.E, e.n_views = src.data_ptr(), 0, 0, 2, 16, 4, 4, 3, 0
    e.raw = raw.data_ptr()
    rc = _cabi.lib().sige_cache_load((_cabi.CacheLoadEntry * 1)(e), 1, 1, None)
    assert rc != 0 and b"destination images" in _cabi.lib().sige_last_error()
