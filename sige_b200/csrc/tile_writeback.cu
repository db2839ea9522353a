// tile_writeback.cu — sparse_update write-back: the output tiles of many NHWC buffers of a step copied into their module caches,
// one launch (include/sige_b200.h, sige_tile_writeback).
// The reference copies each sparse result back into its cache after the module call (sige/nn/scatter.py:59-60,114-129,
// sige/nn/scatter_gather.py:65-77): one full-tensor copy per module.  Here only the tiles the step rewrote are copied, for every
// cached buffer of the step together.  The entry table rides in the kernel parameters (__grid_constant__), so the launch reads the
// fixed-capacity tile lists of the step as they are at run time and stays valid across graph replays and in-place re-binds.
// One CTA per (entry, image, tile); the host's prefix sum over B*N maps the CTA to its entry.  Sources are read in 16-byte
// channel vectors; an NCHW destination is written through a shared-memory transpose, so each (channel, row) of a tile is one
// contiguous run of So elements.
#include <cstring>

#include "common.cuh"

namespace sige {

namespace {

constexpr int kWbThreads = 128;
constexpr int kWbChunk = 64;     // channels per shared-memory pass of an NCHW destination
constexpr int kWbMaxPix = 64;    // Ro * So <= 8 * 8

struct WbParams {
    sige_writeback_entry_t e[SIGE_WRITEBACK_MAX_ENTRIES];
    long long start[SIGE_WRITEBACK_MAX_ENTRIES + 1];   // first CTA of entry k; start[n] = grid size
    int n;
};

template <typename S>
__device__ __forceinline__ void load8(const S *p, float f[8]) {
    const Vec16<S> v = *reinterpret_cast<const Vec16<S> *>(p);
#pragma unroll
    for (int z = 0; z < 8; ++z) f[z] = DT<S>::to_f(v.v[z]);
}

template <typename S>
__device__ void writeback_tile(const sige_writeback_entry_t &e, long long local, float *smem) {
    const int b = (int)(local / e.N), i = (int)(local - (long long)b * e.N);
    const int ih = __ldg(e.idx + 2 * i), iw = __ldg(e.idx + 2 * i + 1);
    if (ih == SIGE_TILE_NONE) return;
    const int oy = (e.offH + ih) / e.strideH, ox = (e.offW + iw) / e.strideW;
    const int r0 = max(oy, 0), r1 = min(oy + e.Ro, e.H), s0 = max(ox, 0), s1 = min(ox + e.So, e.W);
    if (r0 >= r1 || s0 >= s1) return;
    const int rows = r1 - r0, cols = s1 - s0, pix = rows * cols;
    const int CV = e.C / 8;
    const S *src = reinterpret_cast<const S *>(e.src);
    const long long img = (long long)b * e.H * e.W;
    if (e.dst_layout == SIGE_NHWC) {
        for (int t = threadIdx.x; t < pix * CV; t += blockDim.x) {
            const int p = t / CV, cv = t - p * CV;
            const long long off = (img + (long long)(r0 + p / cols) * e.W + (s0 + p % cols)) * e.C + cv * 8;
            if (e.dst_dtype == SIGE_F32) {
                float f[8];
                load8(src + off, f);
                float4 *d = reinterpret_cast<float4 *>(reinterpret_cast<float *>(e.dst) + off);
                d[0] = make_float4(f[0], f[1], f[2], f[3]);
                d[1] = make_float4(f[4], f[5], f[6], f[7]);
            } else {
                *reinterpret_cast<Vec16<S> *>(reinterpret_cast<S *>(e.dst) + off) = *reinterpret_cast<const Vec16<S> *>(src + off);
            }
        }
        return;
    }
    // NCHW: 64 channels of the tile's pixels in shared memory (fp32, a padded row per pixel), then (channel, row) runs of So
    const long long plane = (long long)e.H * e.W;
    for (int c0 = 0; c0 < e.C; c0 += kWbChunk) {
        const int cc = min(kWbChunk, e.C - c0), ccv = cc / 8;
        for (int t = threadIdx.x; t < pix * ccv; t += blockDim.x) {
            const int p = t / ccv, cv = t - p * ccv;
            float f[8];
            load8(src + (img + (long long)(r0 + p / cols) * e.W + (s0 + p % cols)) * e.C + c0 + cv * 8, f);
#pragma unroll
            for (int z = 0; z < 8; ++z) smem[p * (kWbChunk + 1) + cv * 8 + z] = f[z];
        }
        __syncthreads();
        for (int t = threadIdx.x; t < cc * pix; t += blockDim.x) {
            const int c = t / pix, p = t - c * pix, r = p / cols, s = p - r * cols;
            const long long off = ((long long)b * e.C + c0 + c) * plane + (long long)(r0 + r) * e.W + s0 + s;
            const float v = smem[p * (kWbChunk + 1) + c];
            if (e.dst_dtype == SIGE_F32)
                reinterpret_cast<float *>(e.dst)[off] = v;
            else
                reinterpret_cast<S *>(e.dst)[off] = DT<S>::from_f(v);     // exact: v came from an S
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kWbThreads) tile_writeback_kernel(const __grid_constant__ WbParams p) {
    __shared__ float smem[kWbMaxPix * (kWbChunk + 1)];
    const long long cta = blockIdx.x;
    int k = 0;
    while (k + 1 < p.n && p.start[k + 1] <= cta) ++k;
    const sige_writeback_entry_t &e = p.e[k];
    if (e.src_dtype == SIGE_F16)
        writeback_tile<__half>(e, cta - p.start[k], smem);
    else
        writeback_tile<__nv_bfloat16>(e, cta - p.start[k], smem);
}

int check_entry(const sige_writeback_entry_t &e, int k) {
    SIGE_REQUIRE(e.N >= 0, "sige_tile_writeback: entry %d: N = %d", k, e.N);
    if (e.N == 0) return 0;
    SIGE_REQUIRE(e.src && e.dst && e.idx, "sige_tile_writeback: entry %d: null buffer", k);
    SIGE_REQUIRE(e.src_dtype == SIGE_F16 || e.src_dtype == SIGE_BF16, "sige_tile_writeback: entry %d: the source must be f16 or bf16 (got dtype %d)", k, e.src_dtype);
    SIGE_REQUIRE(e.dst_dtype == SIGE_F32 || e.dst_dtype == e.src_dtype,
                 "sige_tile_writeback: entry %d: dtype %d -> %d would round (the cache must be f32 or the source's dtype)", k, e.src_dtype, e.dst_dtype);
    SIGE_REQUIRE(e.dst_layout == SIGE_NCHW || e.dst_layout == SIGE_NHWC, "sige_tile_writeback: entry %d: unknown layout %d", k, e.dst_layout);
    SIGE_REQUIRE(e.B > 0 && e.H > 0 && e.W > 0 && e.C > 0 && e.C % 8 == 0,
                 "sige_tile_writeback: entry %d: B = %d, C = %d, H = %d, W = %d (C a multiple of 8)", k, e.B, e.C, e.H, e.W);
    SIGE_REQUIRE(e.strideH >= 1 && e.strideW >= 1 && e.Ro >= 1 && e.Ro <= 8 && e.So >= 1 && e.So <= 8,
                 "sige_tile_writeback: entry %d: strides %d x %d, output tile %d x %d (1..8)", k, e.strideH, e.strideW, e.Ro, e.So);
    SIGE_REQUIRE(((uintptr_t)e.src | (uintptr_t)e.dst) % 16 == 0, "sige_tile_writeback: entry %d: buffers must be 16-byte aligned", k);
    SIGE_REQUIRE((long long)e.B * e.N < (1LL << 31), "sige_tile_writeback: entry %d: too many tiles", k);
    return 0;
}

}  // namespace

}  // namespace sige

extern "C" int sige_tile_writeback(const sige_writeback_entry_t *entries, int n_entries, sige_stream_t stream) {
    using namespace sige;
    SIGE_REQUIRE(n_entries >= 0 && n_entries <= SIGE_WRITEBACK_MAX_ENTRIES, "sige_tile_writeback: %d entries (at most %d per call)", n_entries,
                 SIGE_WRITEBACK_MAX_ENTRIES);
    if (n_entries == 0) return 0;
    SIGE_REQUIRE(entries != nullptr, "sige_tile_writeback: null entry table");
    WbParams p;
    memset(&p, 0, sizeof(p));
    long long total = 0;
    for (int k = 0; k < n_entries; ++k) {
        if (check_entry(entries[k], k)) return 1;
        if (entries[k].N == 0) continue;
        p.e[p.n] = entries[k];
        p.start[p.n] = total;
        total += (long long)entries[k].B * entries[k].N;
        ++p.n;
    }
    p.start[p.n] = total;
    if (total == 0) return 0;
    SIGE_REQUIRE(total < (1LL << 31), "sige_tile_writeback: %lld tiles in one call", total);
    tile_writeback_kernel<<<(unsigned)total, kWbThreads, 0, (cudaStream_t)stream>>>(p);
    return check_launch("sige_tile_writeback");
}
