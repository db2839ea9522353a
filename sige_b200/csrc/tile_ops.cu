// tile_ops.cu — the five data-movement ops of the SIGE hot path + mask reduction,
// written for sm_90a.  HBM-bound byte movers: the design rules that matter are
// coalescing and 16-byte vector accesses, not tensor cores.
//
// Replaces reference sige/cuda/{gather,scatter,scatter_gather}_kernel.cu.  Unlike the
// reference (one thread per scalar element, fp32/NCHW only, legacy default stream,
// full-tensor clone inside scatter) every op here
//   * is templated on the storage type (fp32 / fp16 / bf16),
//   * has an NHWC (channels-last) variant in which a thread moves one 16-byte channel
//     vector, so that both the gather reads and the scatter writes are fully coalesced
//     (a 128-channel fp16 pixel is two 128-byte lines), next to the reference's NCHW,
//   * takes the stream from the caller, never allocates, never syncs,
//   * treats N == 0 as a no-op.
#include "common.cuh"

namespace sige {

constexpr int kThreads = 256;

struct TileGeom {
    int B, C, H, W;  // full tensor extent
    int N;           // tiles per batch element
    int R, S;        // tile extent (of the stack being read or written)
    int up;          // gather only: 1 = the source holds (H/2, W/2) pixels, read through nearest x2 up-sampling
};

// ----------------------------------------------------------------------------
// gather   (reference sige/cuda/gather_kernel.cu:7-67)
// ----------------------------------------------------------------------------
template <typename T, bool kFast>
__global__ void gather_nchw_kernel(long long total, TileGeom g, const T *__restrict__ x, T *__restrict__ out,
                                   const int32_t *__restrict__ idx, Bcast scale, Bcast shift, int act,
                                   bool act_first) {
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= total) return;
    long long t = i;
    const int s = t % g.S; t /= g.S;
    const int r = t % g.R; t /= g.R;
    const int c = t % g.C; t /= g.C;
    const int n = t % g.N, b = t / g.N;
    const int hh = __ldg(idx + 2 * n) + r, ww = __ldg(idx + 2 * n + 1) + s;
    float z = 0.f;
    if (hh >= 0 && hh < g.H && ww >= 0 && ww < g.W) {
        z = DT<T>::to_f(x[(((long long)b * g.C + c) * (g.H >> g.up) + (hh >> g.up)) * (g.W >> g.up) + (ww >> g.up)]);
        z = affine_act<kFast>(z, scale, shift, act, act_first, b, c, hh, ww);
    }
    out[i] = DT<T>::from_f(z);
}

// NHWC: one thread per (tile, r, s, channel-vector).  V = elements per thread.
template <typename T, int V, bool kFast>
__global__ void gather_nhwc_kernel(long long total, TileGeom g, const T *__restrict__ x, T *__restrict__ out,
                                   const int32_t *__restrict__ idx, Bcast scale, Bcast shift, int act,
                                   bool act_first) {
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int CV = g.C / V;
    long long t = i;
    const int cv = t % CV; t /= CV;
    const int s = t % g.S; t /= g.S;
    const int r = t % g.R; t /= g.R;
    const int n = t % g.N, b = t / g.N;
    const int hh = __ldg(idx + 2 * n) + r, ww = __ldg(idx + 2 * n + 1) + s;
    const int c0 = cv * V;
    T res[V];
    if (hh >= 0 && hh < g.H && ww >= 0 && ww < g.W) {
        const T *src = x + (((long long)b * (g.H >> g.up) + (hh >> g.up)) * (g.W >> g.up) + (ww >> g.up)) * g.C + c0;
        if (V == DT<T>::vec) {
            *reinterpret_cast<Vec16<T> *>(res) = *reinterpret_cast<const Vec16<T> *>(src);
        } else {
#pragma unroll
            for (int k = 0; k < V; ++k) res[k] = src[k];
        }
#pragma unroll
        for (int k = 0; k < V; ++k)
            res[k] = DT<T>::from_f(
                affine_act<kFast>(DT<T>::to_f(res[k]), scale, shift, act, act_first, b, c0 + k, hh, ww));
    } else {
#pragma unroll
        for (int k = 0; k < V; ++k) res[k] = DT<T>::from_f(0.f);
    }
    T *dst = out + i * V;
    if (V == DT<T>::vec) {
        *reinterpret_cast<Vec16<T> *>(dst) = *reinterpret_cast<const Vec16<T> *>(res);
    } else {
#pragma unroll
        for (int k = 0; k < V; ++k) dst[k] = res[k];
    }
}

// ----------------------------------------------------------------------------
// scatter  (reference sige/cuda/scatter_kernel.cu:8-44)
// g.R/g.S are the extent of the stack x (the conv's output tile).
// ----------------------------------------------------------------------------
template <typename T>
__global__ void scatter_nchw_kernel(long long total, TileGeom g, int offH, int offW, int strideH, int strideW,
                                    const T *__restrict__ x, T *__restrict__ out,
                                    const int32_t *__restrict__ idx, Bcast residual) {
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= total) return;
    long long t = i;
    const int s = t % g.S; t /= g.S;
    const int r = t % g.R; t /= g.R;
    const int c = t % g.C; t /= g.C;
    const int n = t % g.N, b = t / g.N;
    const int hh = (offH + __ldg(idx + 2 * n)) / strideH + r;
    const int ww = (offW + __ldg(idx + 2 * n + 1)) / strideW + s;
    if (hh < 0 || hh >= g.H || ww < 0 || ww >= g.W) return;
    float z = DT<T>::to_f(x[i]);
    if (residual.ptr) z = bcast_at(residual, b, c, hh, ww) + z;
    out[(((long long)b * g.C + c) * g.H + hh) * g.W + ww] = DT<T>::from_f(z);
}

template <typename T, int V>
__global__ void scatter_nhwc_kernel(long long total, TileGeom g, int offH, int offW, int strideH, int strideW,
                                    const T *__restrict__ x, T *__restrict__ out,
                                    const int32_t *__restrict__ idx, Bcast residual) {
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int CV = g.C / V;
    long long t = i;
    const int cv = t % CV; t /= CV;
    const int s = t % g.S; t /= g.S;
    const int r = t % g.R; t /= g.R;
    const int n = t % g.N, b = t / g.N;
    const int hh = (offH + __ldg(idx + 2 * n)) / strideH + r;
    const int ww = (offW + __ldg(idx + 2 * n + 1)) / strideW + s;
    if (hh < 0 || hh >= g.H || ww < 0 || ww >= g.W) return;
    const int c0 = cv * V;
    T val[V];
    const T *src = x + i * V;
    if (V == DT<T>::vec) {
        *reinterpret_cast<Vec16<T> *>(val) = *reinterpret_cast<const Vec16<T> *>(src);
    } else {
#pragma unroll
        for (int k = 0; k < V; ++k) val[k] = src[k];
    }
    if (residual.ptr) {
#pragma unroll
        for (int k = 0; k < V; ++k)
            val[k] = DT<T>::from_f(bcast_at(residual, b, c0 + k, hh, ww) + DT<T>::to_f(val[k]));
    }
    T *dst = out + (((long long)b * g.H + hh) * g.W + ww) * g.C + c0;
    if (V == DT<T>::vec) {
        *reinterpret_cast<Vec16<T> *>(dst) = *reinterpret_cast<const Vec16<T> *>(val);
    } else {
#pragma unroll
        for (int k = 0; k < V; ++k) dst[k] = val[k];
    }
}

// ----------------------------------------------------------------------------
// calibrate residual  (reference sige/cuda/scatter_kernel.cu:46-74)
// out[p] += x1[tile] - y1[p] on the shortcut tiles (raw origins).
// ----------------------------------------------------------------------------
template <typename T, bool kNHWC>
__global__ void calibrate_kernel(long long total, TileGeom g, const T *__restrict__ x1, const T *__restrict__ y1,
                                 T *__restrict__ out, const int32_t *__restrict__ idx) {
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= total) return;
    long long t = i;
    int s, r, c;
    if (kNHWC) {
        c = t % g.C; t /= g.C;
        s = t % g.S; t /= g.S;
        r = t % g.R; t /= g.R;
    } else {
        s = t % g.S; t /= g.S;
        r = t % g.R; t /= g.R;
        c = t % g.C; t /= g.C;
    }
    const int n = t % g.N, b = t / g.N;
    const int hh = __ldg(idx + 2 * n) + r, ww = __ldg(idx + 2 * n + 1) + s;
    if (hh < 0 || hh >= g.H || ww < 0 || ww >= g.W) return;
    const long long p = kNHWC ? ((((long long)b * g.H + hh) * g.W + ww) * g.C + c)
                              : ((((long long)b * g.C + c) * g.H + hh) * g.W + ww);
    out[p] = DT<T>::from_f(DT<T>::to_f(out[p]) + (DT<T>::to_f(x1[i]) - DT<T>::to_f(y1[p])));
}

// ----------------------------------------------------------------------------
// scatter map  (reference sige/cuda/scatter_gather_kernel.cu:69-98)
// ----------------------------------------------------------------------------
__global__ void scatter_map_kernel(long long total, int H, int W, int Ro, int So, int offH, int offW, int strideH,
                                   int strideW, int32_t *__restrict__ map, const int32_t *__restrict__ idx) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= total) return;
    long long t = i;
    const int s = t % So; t /= So;
    const int r = t % Ro; t /= Ro;
    const int n = (int)t;                       // < N
    const int hh = (offH + idx[2LL * n]) / strideH + r, ww = (offW + idx[2LL * n + 1]) / strideW + s;
    if (hh < 0 || hh >= H || ww < 0 || ww >= W) return;
    int32_t *m = map + 3 * ((long long)hh * W + ww);
    m[0] = n; m[1] = r; m[2] = s;
}

// ----------------------------------------------------------------------------
// scatter_gather  (reference sige/cuda/scatter_gather_kernel.cu:8-67)
// g.R/g.S = output (next conv's halo) tile; Rx/Sx = extent of stack x.
// ----------------------------------------------------------------------------
template <typename T, bool kFast>
__global__ void scatter_gather_nchw_kernel(long long total, TileGeom g, int Rx, int Sx, const T *__restrict__ x,
                                           const T *__restrict__ y, T *__restrict__ out,
                                           const int32_t *__restrict__ idx, const int32_t *__restrict__ map,
                                           Bcast scale, Bcast shift, int act, bool act_first) {
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= total) return;
    long long t = i;
    const int s = t % g.S; t /= g.S;
    const int r = t % g.R; t /= g.R;
    const int c = t % g.C; t /= g.C;
    const int n = t % g.N, b = t / g.N;
    const int hh = __ldg(idx + 2 * n) + r, ww = __ldg(idx + 2 * n + 1) + s;
    float z = 0.f;
    if (hh >= 0 && hh < g.H && ww >= 0 && ww < g.W) {
        const int32_t *m = map + 3 * ((long long)hh * g.W + ww);
        const int bx = __ldg(m);
        if (bx >= 0) {
            const int hx = __ldg(m + 1), wx = __ldg(m + 2);
            z = DT<T>::to_f(x[(((long long)(b * g.N + bx) * g.C + c) * Rx + hx) * Sx + wx]);
        } else {
            z = DT<T>::to_f(y[(((long long)b * g.C + c) * g.H + hh) * g.W + ww]);
        }
        z = affine_act<kFast>(z, scale, shift, act, act_first, b, c, hh, ww);
    }
    out[i] = DT<T>::from_f(z);
}

template <typename T, int V, bool kFast>
__global__ void scatter_gather_nhwc_kernel(long long total, TileGeom g, int Rx, int Sx, const T *__restrict__ x,
                                           const T *__restrict__ y, T *__restrict__ out,
                                           const int32_t *__restrict__ idx, const int32_t *__restrict__ map,
                                           Bcast scale, Bcast shift, int act, bool act_first) {
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int CV = g.C / V;
    long long t = i;
    const int cv = t % CV; t /= CV;
    const int s = t % g.S; t /= g.S;
    const int r = t % g.R; t /= g.R;
    const int n = t % g.N, b = t / g.N;
    const int hh = __ldg(idx + 2 * n) + r, ww = __ldg(idx + 2 * n + 1) + s;
    const int c0 = cv * V;
    T res[V];
    if (hh >= 0 && hh < g.H && ww >= 0 && ww < g.W) {
        const int32_t *m = map + 3 * ((long long)hh * g.W + ww);
        const int bx = __ldg(m);
        const T *src;
        if (bx >= 0) {
            const int hx = __ldg(m + 1), wx = __ldg(m + 2);
            src = x + (((long long)(b * g.N + bx) * Rx + hx) * Sx + wx) * g.C + c0;
        } else {
            src = y + (((long long)b * g.H + hh) * g.W + ww) * g.C + c0;
        }
        if (V == DT<T>::vec) {
            *reinterpret_cast<Vec16<T> *>(res) = *reinterpret_cast<const Vec16<T> *>(src);
        } else {
#pragma unroll
            for (int k = 0; k < V; ++k) res[k] = src[k];
        }
#pragma unroll
        for (int k = 0; k < V; ++k)
            res[k] = DT<T>::from_f(
                affine_act<kFast>(DT<T>::to_f(res[k]), scale, shift, act, act_first, b, c0 + k, hh, ww));
    } else {
#pragma unroll
        for (int k = 0; k < V; ++k) res[k] = DT<T>::from_f(0.f);
    }
    T *dst = out + i * V;
    if (V == DT<T>::vec) {
        *reinterpret_cast<Vec16<T> *>(dst) = *reinterpret_cast<const Vec16<T> *>(res);
    } else {
#pragma unroll
        for (int k = 0; k < V; ++k) dst[k] = res[k];
    }
}

// ----------------------------------------------------------------------------
// reduce_mask  (reference sige/utils.py:8-37) — device-side, ordered compaction.
// One CTA walks the pooled grid in row-major chunks of blockDim.x candidates; each
// thread tests its R x S window, a ballot + warp-total scan gives the rank, so the
// output order equals torch.nonzero's row-major order bit for bit.  Writes the first
// `capacity` origins and returns the number of active tiles (to every thread).
// ----------------------------------------------------------------------------
__device__ int reduce_mask_cta(const uint8_t *__restrict__ mask, int H, int W, int R, int S, int strideH, int strideW,
                               int padH, int padW, int nI, int nJ, int32_t *__restrict__ out, int capacity) {
    __shared__ int warp_tot[32];
    __shared__ int base_s;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    if (threadIdx.x == 0) base_s = 0;
    __syncthreads();
    const int total = nI * nJ;                  // < 2^31 (checked on the host)
    // unsigned: the step past the last chunk may reach 2^31
    for (unsigned start = 0; start < (unsigned)total; start += blockDim.x) {
        const unsigned cand = start + threadIdx.x;
        bool any = false;
        int i = 0, j = 0;
        if (cand < (unsigned)total) {
            i = cand / nJ; j = cand % nJ;
            const int h0 = max(i * strideH - padH, 0), h1 = min(i * strideH - padH + R, H);
            const int w0 = max(j * strideW - padW, 0), w1 = min(j * strideW - padW + S, W);
            for (int hh = h0; hh < h1 && !any; ++hh)
                for (int ww = w0; ww < w1; ++ww)
                    if (mask[(long long)hh * W + ww]) { any = true; break; }
        }
        const unsigned bal = __ballot_sync(0xffffffffu, any);
        if (lane == 0) warp_tot[warp] = __popc(bal);
        __syncthreads();
        int before = 0, chunk = 0;
        for (int wdx = 0; wdx < nwarps; ++wdx) {
            const int v = warp_tot[wdx];
            if (wdx < warp) before += v;
            chunk += v;
        }
        const int base = base_s;
        if (any) {
            const int pos = base + before + __popc(bal & ((1u << lane) - 1u));
            if (pos < capacity) {
                out[2LL * pos] = strideH * i - padH;
                out[2LL * pos + 1] = strideW * j - padW;
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) base_s = base + chunk;
        __syncthreads();
    }
    return base_s;
}

__global__ void reduce_mask_kernel(const uint8_t *__restrict__ mask, int H, int W, int R, int S, int strideH,
                                   int strideW, int padH, int padW, int nI, int nJ, int32_t *__restrict__ out,
                                   int capacity, int32_t *__restrict__ count) {
    const int total = reduce_mask_cta(mask, H, W, R, S, strideH, strideW, padH, padW, nI, nJ, out, capacity);
    if (threadIdx.x == 0) *count = total;
}

// E masks of one geometry, one CTA per mask: image e's list goes to rows e*cap .. e*cap + cap - 1 (the per-image layout of
// sige_tile_conv_t.idx_per_image), SIGE_TILE_NONE behind its tiles.
__global__ void reduce_mask_batched_kernel(const uint8_t *__restrict__ masks, int H, int W, int R, int S, int strideH,
                                           int strideW, int padH, int padW, int nI, int nJ, int32_t *__restrict__ out,
                                           int cap, int32_t *__restrict__ counts, int32_t *__restrict__ status) {
    const int e = blockIdx.x;
    int32_t *seg = out + 2LL * e * cap;
    const int total = reduce_mask_cta(masks + (long long)e * H * W, H, W, R, S, strideH, strideW, padH, padW, nI, nJ, seg, cap);
    for (long long i = 2LL * min(total, cap) + threadIdx.x; i < 2LL * cap; i += blockDim.x) seg[i] = SIGE_TILE_NONE;
    if (threadIdx.x == 0) {
        counts[e] = total;
        if (total > cap) atomicOr(status, 1);
    }
}

// ----------------------------------------------------------------------------
// weight repack OIHW -> [tap][Cin/64][Cout][64]: the slab a CTA streams for one (tap, 64-channel chunk,
// Cout block) is ONE contiguous run of Cout_block*128 bytes (DRAM-page friendly, one TMA box).
// If Cin is not a multiple of 64 the plain [tap][Cout][Cin] order is used (generic consumers only).
// ----------------------------------------------------------------------------
template <typename TS, typename TD>
__global__ void pack_weight_kernel(long long total, const TS *__restrict__ w, TD *__restrict__ out, int Cout,
                                   int Cin, int taps) {
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= total) return;
    long long t = i;
    int ci, co, tap;
    if (Cin % 64 == 0) {
        const int k = t % 64; t /= 64;
        co = t % Cout; t /= Cout;
        const int chunk = t % (Cin / 64); t /= (Cin / 64);
        tap = t;
        ci = chunk * 64 + k;
    } else {
        ci = t % Cin; t /= Cin;
        co = t % Cout; t /= Cout;
        tap = t;
    }
    out[i] = DT<TD>::from_f(DT<TS>::to_f(w[((long long)co * Cin + ci) * taps + tap]));
}

// ----------------------------------------------------------------------------
// host launchers
// ----------------------------------------------------------------------------
template <typename T>
static int launch_gather(const void *x, int layout, TileGeom g, const int32_t *idx, const Bcast &sc,
                         const Bcast &sh, int act, int act_first, void *out, cudaStream_t st) {
    constexpr bool kFast = !std::is_same<T, float>::value;
    const long long elems = (long long)g.B * g.N * g.C * g.R * g.S;
    if (layout == SIGE_NCHW) {
        gather_nchw_kernel<T, kFast><<<ceil_div(elems, kThreads), kThreads, 0, st>>>(
            elems, g, (const T *)x, (T *)out, idx, sc, sh, act, act_first != 0);
    } else if (g.C % DT<T>::vec == 0 && ((uintptr_t)x % 16 == 0) && ((uintptr_t)out % 16 == 0)) {
        constexpr int V = DT<T>::vec;
        const long long total = elems / V;
        gather_nhwc_kernel<T, V, kFast><<<ceil_div(total, kThreads), kThreads, 0, st>>>(
            total, g, (const T *)x, (T *)out, idx, sc, sh, act, act_first != 0);
    } else {
        gather_nhwc_kernel<T, 1, kFast><<<ceil_div(elems, kThreads), kThreads, 0, st>>>(
            elems, g, (const T *)x, (T *)out, idx, sc, sh, act, act_first != 0);
    }
    return check_launch("sige_gather");
}

template <typename T>
static int launch_scatter(const void *x, void *out, int layout, TileGeom g, int offH, int offW, int strideH,
                          int strideW, const int32_t *idx, const Bcast &res, cudaStream_t st) {
    const long long elems = (long long)g.B * g.N * g.C * g.R * g.S;
    if (layout == SIGE_NCHW) {
        scatter_nchw_kernel<T><<<ceil_div(elems, kThreads), kThreads, 0, st>>>(
            elems, g, offH, offW, strideH, strideW, (const T *)x, (T *)out, idx, res);
    } else if (g.C % DT<T>::vec == 0 && ((uintptr_t)x % 16 == 0) && ((uintptr_t)out % 16 == 0)) {
        constexpr int V = DT<T>::vec;
        const long long total = elems / V;
        scatter_nhwc_kernel<T, V><<<ceil_div(total, kThreads), kThreads, 0, st>>>(
            total, g, offH, offW, strideH, strideW, (const T *)x, (T *)out, idx, res);
    } else {
        scatter_nhwc_kernel<T, 1><<<ceil_div(elems, kThreads), kThreads, 0, st>>>(
            elems, g, offH, offW, strideH, strideW, (const T *)x, (T *)out, idx, res);
    }
    return check_launch("sige_scatter");
}

template <typename T>
static int launch_calibrate(const void *x1, const void *y1, void *out, int layout, TileGeom g, const int32_t *idx,
                            cudaStream_t st) {
    const long long elems = (long long)g.B * g.N * g.C * g.R * g.S;
    if (layout == SIGE_NCHW)
        calibrate_kernel<T, false><<<ceil_div(elems, kThreads), kThreads, 0, st>>>(elems, g, (const T *)x1,
                                                                                   (const T *)y1, (T *)out, idx);
    else
        calibrate_kernel<T, true><<<ceil_div(elems, kThreads), kThreads, 0, st>>>(elems, g, (const T *)x1,
                                                                                  (const T *)y1, (T *)out, idx);
    return check_launch("sige_scatter_with_block_residual/calibrate");
}

template <typename T>
static int launch_scatter_gather(const void *x, const void *y, int layout, TileGeom g, int Rx, int Sx,
                                 const int32_t *idx, const int32_t *map, const Bcast &sc, const Bcast &sh, int act,
                                 int act_first, void *out, cudaStream_t st) {
    constexpr bool kFast = !std::is_same<T, float>::value;
    const long long elems = (long long)g.B * g.N * g.C * g.R * g.S;
    if (layout == SIGE_NCHW) {
        scatter_gather_nchw_kernel<T, kFast><<<ceil_div(elems, kThreads), kThreads, 0, st>>>(
            elems, g, Rx, Sx, (const T *)x, (const T *)y, (T *)out, idx, map, sc, sh, act, act_first != 0);
    } else if (g.C % DT<T>::vec == 0 && ((uintptr_t)x % 16 == 0) && ((uintptr_t)y % 16 == 0) &&
               ((uintptr_t)out % 16 == 0)) {
        constexpr int V = DT<T>::vec;
        const long long total = elems / V;
        scatter_gather_nhwc_kernel<T, V, kFast><<<ceil_div(total, kThreads), kThreads, 0, st>>>(
            total, g, Rx, Sx, (const T *)x, (const T *)y, (T *)out, idx, map, sc, sh, act, act_first != 0);
    } else {
        scatter_gather_nhwc_kernel<T, 1, kFast><<<ceil_div(elems, kThreads), kThreads, 0, st>>>(
            elems, g, Rx, Sx, (const T *)x, (const T *)y, (T *)out, idx, map, sc, sh, act, act_first != 0);
    }
    return check_launch("sige_scatter_gather");
}

static size_t dtype_size(int dtype) { return dtype == SIGE_F32 ? 4 : 2; }

#define SIGE_DISPATCH_DTYPE(dtype, CALL)                         \
    switch (dtype) {                                             \
        case SIGE_F32: { using T = float; CALL; }                \
        case SIGE_F16: { using T = __half; CALL; }               \
        case SIGE_BF16: { using T = __nv_bfloat16; CALL; }       \
        default: ::sige::set_error("unsupported dtype %d", dtype); return 1; \
    }

// Candidate tiles nI x nJ of the pooled grid: padded extent (H + pad + R), window R, floor mode -> (H + pad)/stride + 1
// (reference sige/utils.py:27-28).  reduce_mask_cta counts them, and the tiles it finds, in an int, so 2^31 or more are refused:
// -1 with the error set.
static long long reduce_mask_candidates(const char *what, int H, int W, int strideH, int strideW, int padH, int padW) {
    const long long n = (((long long)H + padH) / strideH + 1) * (((long long)W + padW) / strideW + 1);
    if (n < 2147483648LL) return n;
    set_error("%s: too many candidate tiles (%lld, the limit is 2^31 - 1)", what, n);
    return -1;
}

}  // namespace sige

using namespace sige;

extern "C" {

int sige_reduce_mask_capacity(int H, int W, int R, int S, int strideH, int strideW, int padH, int padW) {
    (void)R; (void)S;
    if (H <= 0 || W <= 0 || strideH <= 0 || strideW <= 0) return 0;
    return (int)reduce_mask_candidates("sige_reduce_mask_capacity", H, W, strideH, strideW, padH, padW);
}

int sige_reduce_mask(const uint8_t *mask, int H, int W, int R, int S, int strideH, int strideW, int padH, int padW,
                     int32_t *idx_out, int capacity, int32_t *count_out, sige_stream_t stream) {
    SIGE_REQUIRE(mask && count_out, "sige_reduce_mask: null pointer");
    SIGE_REQUIRE(H > 0 && W > 0 && R > 0 && S > 0 && strideH > 0 && strideW > 0 && padH >= 0 && padW >= 0,
                 "sige_reduce_mask: bad geometry H=%d W=%d R=%d S=%d stride=(%d,%d) pad=(%d,%d)", H, W, R, S,
                 strideH, strideW, padH, padW);
    if (reduce_mask_candidates("sige_reduce_mask", H, W, strideH, strideW, padH, padW) < 0) return 1;
    SIGE_REQUIRE(capacity == 0 || idx_out, "sige_reduce_mask: idx_out is null with capacity %d", capacity);
    const int nI = (int)(((long long)H + padH) / strideH + 1), nJ = (int)(((long long)W + padW) / strideW + 1);
    reduce_mask_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(mask, H, W, R, S, strideH, strideW, padH, padW, nI, nJ,
                                                             idx_out, capacity, count_out);
    return check_launch("sige_reduce_mask");
}

int sige_reduce_mask_batched(const uint8_t *masks, int E, int H, int W, int R, int S, int strideH, int strideW, int padH,
                             int padW, int32_t *idx_out, int cap, int32_t *counts_out, int32_t *status,
                             sige_stream_t stream) {
    SIGE_REQUIRE(E >= 0 && cap >= 0, "sige_reduce_mask_batched: negative E (%d) or cap (%d)", E, cap);
    if (E == 0) return 0;
    SIGE_REQUIRE(masks && counts_out && status, "sige_reduce_mask_batched: null pointer");
    SIGE_REQUIRE(H > 0 && W > 0 && R > 0 && S > 0 && strideH > 0 && strideW > 0 && padH >= 0 && padW >= 0,
                 "sige_reduce_mask_batched: bad geometry H=%d W=%d R=%d S=%d stride=(%d,%d) pad=(%d,%d)", H, W, R, S,
                 strideH, strideW, padH, padW);
    if (reduce_mask_candidates("sige_reduce_mask_batched", H, W, strideH, strideW, padH, padW) < 0) return 1;
    SIGE_REQUIRE(cap == 0 || idx_out, "sige_reduce_mask_batched: idx_out is null with cap %d", cap);
    const int nI = (int)(((long long)H + padH) / strideH + 1), nJ = (int)(((long long)W + padW) / strideW + 1);
    reduce_mask_batched_kernel<<<E, 1024, 0, (cudaStream_t)stream>>>(masks, H, W, R, S, strideH, strideW, padH, padW, nI,
                                                                     nJ, idx_out, cap, counts_out, status);
    return check_launch("sige_reduce_mask_batched");
}

int sige_gather(const void *x, int dtype, int layout, int B, int C, int H, int W, int R, int S, const int32_t *idx,
                int N, const sige_bcast_t *scale, const sige_bcast_t *shift, int act, int act_first, void *out,
                sige_stream_t stream) {
    return sige_gather_upsampled(x, dtype, layout, B, C, H, W, 0, R, S, idx, N, scale, shift, act, act_first, out, stream);
}

int sige_gather_upsampled(const void *x, int dtype, int layout, int B, int C, int H, int W, int up, int R, int S,
                          const int32_t *idx, int N, const sige_bcast_t *scale, const sige_bcast_t *shift, int act,
                          int act_first, void *out, sige_stream_t stream) {
    SIGE_REQUIRE(B > 0 && C > 0 && H > 0 && W > 0 && R > 0 && S > 0 && N >= 0, "sige_gather: bad shape");
    SIGE_REQUIRE(up == 0 || (up == 1 && H % 2 == 0 && W % 2 == 0), "sige_gather_upsampled: up must be 0 or 1 (even H, W)");
    SIGE_REQUIRE(layout == SIGE_NCHW || layout == SIGE_NHWC, "sige_gather: bad layout %d", layout);
    SIGE_REQUIRE(act == SIGE_ACT_IDENTITY || act == SIGE_ACT_SWISH, "sige_gather: unknown activation %d", act);
    if (N == 0) return 0;
    SIGE_REQUIRE(x && out && idx, "sige_gather: null pointer");
    Bcast sc, sh;
    if (make_bcast(scale, B, C, H, W, "scale", &sc) || make_bcast(shift, B, C, H, W, "shift", &sh)) return 1;
    TileGeom g{B, C, H, W, N, R, S, up};
    SIGE_DISPATCH_DTYPE(dtype, return launch_gather<T>(x, layout, g, idx, sc, sh, act, act_first, out,
                                                       (cudaStream_t)stream));
}

int sige_scatter(const void *x, const void *y, void *out, int dtype, int layout, int B, int C, int H, int W, int Ro,
                 int So, int offH, int offW, int strideH, int strideW, const int32_t *idx, int N,
                 const sige_bcast_t *residual, sige_stream_t stream) {
    SIGE_REQUIRE(B > 0 && C > 0 && H > 0 && W > 0 && Ro > 0 && So > 0 && N >= 0, "sige_scatter: bad shape");
    SIGE_REQUIRE(strideH > 0 && strideW > 0, "sige_scatter: bad stride");
    SIGE_REQUIRE(layout == SIGE_NCHW || layout == SIGE_NHWC, "sige_scatter: bad layout %d", layout);
    SIGE_REQUIRE(out, "sige_scatter: null output");
    SIGE_REQUIRE(dtype >= 0 && dtype <= 2, "sige_scatter: unsupported dtype %d", dtype);
    if (y && y != out) {
        cudaError_t e = cudaMemcpyAsync(out, y, (size_t)B * C * H * W * dtype_size(dtype), cudaMemcpyDeviceToDevice,
                                        (cudaStream_t)stream);
        SIGE_REQUIRE(e == cudaSuccess, "sige_scatter: copy of the cached tensor failed: %s", cudaGetErrorString(e));
    }
    if (N == 0) return 0;
    SIGE_REQUIRE(x && idx, "sige_scatter: null pointer");
    Bcast res;
    if (make_bcast(residual, B, C, H, W, "residual", &res)) return 1;
    TileGeom g{B, C, H, W, N, Ro, So, 0};
    SIGE_DISPATCH_DTYPE(dtype, return launch_scatter<T>(x, out, layout, g, offH, offW, strideH, strideW, idx, res,
                                                        (cudaStream_t)stream));
}

int sige_scatter_with_block_residual(const void *x0, const void *y0, const void *x1, const void *y1, void *out,
                                     int dtype, int layout, int B, int C, int H, int W, int R0, int S0, int R1,
                                     int S1, int offH, int offW, int strideH, int strideW, const int32_t *idx0,
                                     int N0, const int32_t *idx1, int N1, sige_stream_t stream) {
    SIGE_REQUIRE(y1, "sige_scatter_with_block_residual: y1 (cached shortcut output) is null");
    SIGE_REQUIRE(N1 >= 0 && R1 > 0 && S1 > 0, "sige_scatter_with_block_residual: bad shortcut shape");
    sige_bcast_t r;
    r.ptr = y1;
    r.dims[0] = B; r.dims[1] = C; r.dims[2] = H; r.dims[3] = W;
    if (layout == SIGE_NCHW) {
        r.stride[0] = (int64_t)C * H * W; r.stride[1] = (int64_t)H * W; r.stride[2] = W; r.stride[3] = 1;
    } else {
        r.stride[0] = (int64_t)C * H * W; r.stride[1] = 1; r.stride[2] = (int64_t)W * C; r.stride[3] = C;
    }
    r.dtype = dtype;
    if (sige_scatter(x0, y0, out, dtype, layout, B, C, H, W, R0, S0, offH, offW, strideH, strideW, idx0, N0, &r, stream))
        return 1;
    if (N1 == 0) return 0;
    SIGE_REQUIRE(x1 && idx1, "sige_scatter_with_block_residual: null pointer");
    TileGeom g{B, C, H, W, N1, R1, S1, 0};
    SIGE_DISPATCH_DTYPE(dtype, return launch_calibrate<T>(x1, y1, out, layout, g, idx1, (cudaStream_t)stream));
}

int sige_get_scatter_map(int H, int W, int R, int S, int kH, int kW, int offH, int offW, int strideH, int strideW,
                         const int32_t *idx, int N, int32_t *map_out, sige_stream_t stream) {
    SIGE_REQUIRE(H > 0 && W > 0 && R >= kH && S >= kW && kH > 0 && kW > 0 && strideH > 0 && strideW > 0 && N >= 0,
                 "sige_get_scatter_map: bad geometry");
    SIGE_REQUIRE(map_out, "sige_get_scatter_map: null output");
    const int Ro = (R - kH) / strideH + 1, So = (S - kW) / strideW + 1;
    const long long total = (long long)N * Ro * So;
    SIGE_REQUIRE(total <= 2147483647LL * kThreads, "sige_get_scatter_map: grid too large (%lld tile pixels)", total);
    SIGE_REQUIRE(N == 0 || idx, "sige_get_scatter_map: null index list");
    cudaError_t e = cudaMemsetAsync(map_out, 0xFF, sizeof(int32_t) * 3 * (size_t)H * W, (cudaStream_t)stream);
    SIGE_REQUIRE(e == cudaSuccess, "sige_get_scatter_map: memset failed: %s", cudaGetErrorString(e));
    if (N == 0) return 0;
    scatter_map_kernel<<<ceil_div(total, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
        total, H, W, Ro, So, offH, offW, strideH, strideW, map_out, idx);
    return check_launch("sige_get_scatter_map");
}

int sige_scatter_gather(const void *x, const void *y, int dtype, int layout, int B, int C, int H, int W, int Rx,
                        int Sx, int R, int S, const int32_t *idx, int N, const int32_t *scatter_map,
                        const sige_bcast_t *scale, const sige_bcast_t *shift, int act, int act_first, void *out,
                        sige_stream_t stream) {
    SIGE_REQUIRE(B > 0 && C > 0 && H > 0 && W > 0 && R > 0 && S > 0 && Rx > 0 && Sx > 0 && N >= 0,
                 "sige_scatter_gather: bad shape");
    SIGE_REQUIRE(layout == SIGE_NCHW || layout == SIGE_NHWC, "sige_scatter_gather: bad layout %d", layout);
    SIGE_REQUIRE(act == SIGE_ACT_IDENTITY || act == SIGE_ACT_SWISH, "sige_scatter_gather: unknown activation %d", act);
    if (N == 0) return 0;
    SIGE_REQUIRE(x && y && out && idx && scatter_map, "sige_scatter_gather: null pointer");
    Bcast sc, sh;
    if (make_bcast(scale, B, C, H, W, "scale", &sc) || make_bcast(shift, B, C, H, W, "shift", &sh)) return 1;
    TileGeom g{B, C, H, W, N, R, S, 0};
    SIGE_DISPATCH_DTYPE(dtype, return launch_scatter_gather<T>(x, y, layout, g, Rx, Sx, idx, scatter_map, sc, sh, act,
                                                               act_first, out, (cudaStream_t)stream));
}

int sige_pack_conv_weight(const void *w, int src_dtype, int Cout, int Cin, int kH, int kW, void *out, int dst_dtype,
                          sige_stream_t stream) {
    SIGE_REQUIRE(w && out && Cout > 0 && Cin > 0 && kH > 0 && kW > 0, "sige_pack_conv_weight: bad arguments");
    SIGE_REQUIRE(dst_dtype == SIGE_F16 || dst_dtype == SIGE_BF16, "sige_pack_conv_weight: dst dtype must be f16/bf16");
    const int taps = kH * kW;
    const long long total = (long long)taps * Cout * Cin;
    const int grid = ceil_div(total, kThreads);
    cudaStream_t st = (cudaStream_t)stream;
#define SIGE_PACK(TS, TD) pack_weight_kernel<TS, TD><<<grid, kThreads, 0, st>>>(total, (const TS *)w, (TD *)out, Cout, Cin, taps)
    if (dst_dtype == SIGE_F16) {
        if (src_dtype == SIGE_F32) SIGE_PACK(float, __half);
        else if (src_dtype == SIGE_F16) SIGE_PACK(__half, __half);
        else if (src_dtype == SIGE_BF16) SIGE_PACK(__nv_bfloat16, __half);
        else { set_error("sige_pack_conv_weight: bad src dtype %d", src_dtype); return 1; }
    } else {
        if (src_dtype == SIGE_F32) SIGE_PACK(float, __nv_bfloat16);
        else if (src_dtype == SIGE_F16) SIGE_PACK(__half, __nv_bfloat16);
        else if (src_dtype == SIGE_BF16) SIGE_PACK(__nv_bfloat16, __nv_bfloat16);
        else { set_error("sige_pack_conv_weight: bad src dtype %d", src_dtype); return 1; }
    }
#undef SIGE_PACK
    return check_launch("sige_pack_conv_weight");
}

}  // extern "C"
