// cache_load.cu — reload of a compiled step's cached buffers from the module caches, every buffer in one launch
// (include/sige_b200.h, sige_cache_load).
// A cached buffer of a fused step is an NHWC copy of a module cache in the step's dtype, plus up to two transformed views
// act(cache * scale + shift) that its producer keeps up to date.  They are (re)loaded when the step is built, when a new edit is
// bound to it and after every dense pass.  Each entry's source is read once: a CTA stages a 64-channel x 64-pixel tile in shared
// memory (an NCHW source is read along pixels, an NHWC one along channels, both coalesced) and writes every destination of
// every image in 16-byte channel vectors.  The arithmetic restates the torch chain it replaces, rounding each step:
// fp32 multiply, fp32 add, swish = z * (1 / (1 + expf(-z))), round-to-nearest into the step's dtype.
#include <cstring>

#include "common.cuh"

namespace sige {

namespace {

constexpr int kClThreads = 256;
constexpr int kClC = 64;     // channels per tile
constexpr int kClP = 64;     // pixels per tile

struct ClParams {
    sige_cache_load_entry_t e[SIGE_CACHE_LOAD_MAX_ENTRIES];
    long long start[SIGE_CACHE_LOAD_MAX_ENTRIES + 1];   // first CTA of entry k; start[n] = grid size
    int n;
};

template <typename S>
__device__ __forceinline__ float load_src(const void *p, long long off) {
    return DT<S>::to_f(reinterpret_cast<const S *>(p)[off]);
}

__device__ __forceinline__ float load_any(int dtype, const void *p, long long off) {
    if (dtype == SIGE_F32) return load_src<float>(p, off);
    if (dtype == SIGE_F16) return load_src<__half>(p, off);
    return load_src<__nv_bfloat16>(p, off);
}

__device__ __forceinline__ float view_value(float z, const sige_cache_view_t &v, int c) {
    if (v.scale) z = __fmul_rn(z, __ldg(v.scale + c));
    if (v.shift) z = __fadd_rn(z, __ldg(v.shift + c));
    if (v.act == SIGE_ACT_SWISH) z = __fmul_rn(z, __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-z))));
    return z;
}

template <typename T>
__device__ __forceinline__ void store8(void *base, long long off, const float f[8]) {
    Vec16<T> v;
#pragma unroll
    for (int z = 0; z < 8; ++z) v.v[z] = DT<T>::from_f(f[z]);
    *reinterpret_cast<Vec16<T> *>(reinterpret_cast<T *>(base) + off) = v;
}

template <typename T>
__device__ void load_tile(const sige_cache_load_entry_t &e, long long local, float (*s)[kClP + 1]) {
    const long long HW = (long long)e.H * e.W;
    const int nct = (e.C + kClC - 1) / kClC;
    const long long npt = (HW + kClP - 1) / kClP;
    const int ct = (int)(local % nct);
    const long long rest = local / nct;
    const long long pt = rest % npt;
    const int b = (int)(rest / npt);
    const int c0 = ct * kClC;
    const long long p0 = pt * kClP;
    const int cc = min(kClC, e.C - c0);
    const int pp = (int)min((long long)kClP, HW - p0);
    // stage: s[c][p] in fp32 (exact for every source dtype)
    if (e.src_layout == SIGE_NCHW) {
        for (int t = threadIdx.x; t < kClC * kClP; t += kClThreads) {
            const int c = t / kClP, p = t - c * kClP;
            if (c < cc && p < pp) s[c][p] = load_any(e.src_dtype, e.src, ((long long)b * e.C + c0 + c) * HW + p0 + p);
        }
    } else {
        for (int t = threadIdx.x; t < kClC * kClP; t += kClThreads) {
            const int p = t / kClC, c = t - p * kClC;
            if (c < cc && p < pp) s[c][p] = load_any(e.src_dtype, e.src, ((long long)b * HW + p0 + p) * e.C + c0 + c);
        }
    }
    __syncthreads();
    // write: one 16-byte channel vector of one pixel per item, to every image it belongs to
    const int ngrp = cc / 8;
    const int i0 = e.src_batch == 1 ? 0 : b, i1 = e.src_batch == 1 ? e.E : b + 1;
    for (int t = threadIdx.x; t < pp * ngrp; t += kClThreads) {
        const int p = t / ngrp, g = t - p * ngrp;
        float raw[8];
#pragma unroll
        for (int z = 0; z < 8; ++z) raw[z] = s[g * 8 + z][p];
        const int c = c0 + g * 8;
        float vw[2][8];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            if (k < e.n_views) {
#pragma unroll
                for (int z = 0; z < 8; ++z) vw[k][z] = view_value(raw[z], e.view[k], c + z);
            }
        }
        for (int img = i0; img < i1; ++img) {
            const long long off = ((long long)img * HW + p0 + p) * e.C + c;
            if (e.raw) store8<T>(e.raw, off, raw);
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                if (k < e.n_views) store8<T>(e.view[k].dst, off, vw[k]);
            }
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(kClThreads) cache_load_kernel(const __grid_constant__ ClParams p) {
    __shared__ float s[kClC][kClP + 1];
    const long long cta = blockIdx.x;
    int k = 0;
    while (k + 1 < p.n && p.start[k + 1] <= cta) ++k;
    load_tile<T>(p.e[k], cta - p.start[k], s);
}

long long entry_ctas(const sige_cache_load_entry_t &e) {
    const long long HW = (long long)e.H * e.W;
    return (long long)e.src_batch * ((HW + kClP - 1) / kClP) * ((e.C + kClC - 1) / kClC);
}

int check_entry(const sige_cache_load_entry_t &e, int k) {
    SIGE_REQUIRE(e.src != nullptr, "sige_cache_load: entry %d: null source", k);
    SIGE_REQUIRE(e.src_dtype == SIGE_F32 || e.src_dtype == SIGE_F16 || e.src_dtype == SIGE_BF16, "sige_cache_load: entry %d: source dtype %d", k,
                 e.src_dtype);
    SIGE_REQUIRE(e.src_layout == SIGE_NCHW || e.src_layout == SIGE_NHWC, "sige_cache_load: entry %d: unknown layout %d", k, e.src_layout);
    SIGE_REQUIRE(e.C > 0 && e.C % 8 == 0 && e.H > 0 && e.W > 0 && e.E > 0,
                 "sige_cache_load: entry %d: C = %d, H = %d, W = %d, E = %d (C a multiple of 8)", k, e.C, e.H, e.W, e.E);
    SIGE_REQUIRE(e.src_batch == 1 || e.src_batch == e.E, "sige_cache_load: entry %d: a source of %d images for %d destination images (1 or E)", k,
                 e.src_batch, e.E);
    SIGE_REQUIRE(e.n_views >= 0 && e.n_views <= 2, "sige_cache_load: entry %d: %d views (at most 2)", k, e.n_views);
    SIGE_REQUIRE(e.raw != nullptr || e.n_views > 0, "sige_cache_load: entry %d: no destination", k);
    SIGE_REQUIRE((uintptr_t)e.raw % 16 == 0, "sige_cache_load: entry %d: the raw destination must be 16-byte aligned", k);
    for (int v = 0; v < e.n_views; ++v) {
        SIGE_REQUIRE(e.view[v].dst != nullptr && (uintptr_t)e.view[v].dst % 16 == 0, "sige_cache_load: entry %d: view %d must be a 16-byte aligned buffer",
                     k, v);
        SIGE_REQUIRE(e.view[v].act == SIGE_ACT_IDENTITY || e.view[v].act == SIGE_ACT_SWISH, "sige_cache_load: entry %d: view %d: activation %d", k, v,
                     e.view[v].act);
    }
    return 0;
}

}  // namespace

}  // namespace sige

extern "C" int sige_cache_load(const sige_cache_load_entry_t *entries, int n_entries, int dtype, sige_stream_t stream) {
    using namespace sige;
    SIGE_REQUIRE(n_entries >= 0 && n_entries <= SIGE_CACHE_LOAD_MAX_ENTRIES, "sige_cache_load: %d entries (at most %d per call)", n_entries,
                 SIGE_CACHE_LOAD_MAX_ENTRIES);
    if (n_entries == 0) return 0;
    SIGE_REQUIRE(entries != nullptr, "sige_cache_load: null entry table");
    SIGE_REQUIRE(dtype == SIGE_F16 || dtype == SIGE_BF16, "sige_cache_load: destination dtype %d (f16 or bf16)", dtype);
    ClParams p;
    memset(&p, 0, sizeof(p));
    long long total = 0;
    for (int k = 0; k < n_entries; ++k) {
        if (check_entry(entries[k], k)) return 1;
        p.e[k] = entries[k];
        p.start[k] = total;
        total += entry_ctas(entries[k]);
    }
    p.n = n_entries;
    p.start[n_entries] = total;
    SIGE_REQUIRE(total < (1LL << 31), "sige_cache_load: %lld tiles in one call", total);
    if (dtype == SIGE_F16)
        cache_load_kernel<__half><<<(unsigned)total, kClThreads, 0, (cudaStream_t)stream>>>(p);
    else
        cache_load_kernel<__nv_bfloat16><<<(unsigned)total, kClThreads, 0, (cudaStream_t)stream>>>(p);
    return check_launch("sige_cache_load");
}
