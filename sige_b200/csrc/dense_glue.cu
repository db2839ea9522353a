// dense_glue.cu — the three dense, non-tile-shaped layers of a DDPM step, NHWC fp16/bf16:
//   conv_in   3x3, 3 -> C channels on the full image        (reference sige_fused_unet.py:395)
//   GroupNorm statistics of the final activation, folded to per-channel (scale, shift)
//   conv_out  SiLU(x*scale+shift) -> 3x3, C -> 3 channels   (reference sige_fused_unet.py:431-433)
// The reference leaves these to cuDNN / ATen; at a 1.2 % edit they are ~20 % of the step
// (the channels-last GroupNorm alone was one of the longest launches of the step), and
// they are pure HBM streams: 16.8 MB written (conv_in) or read (stats, conv_out) at 256x256x128.
//
// All three are deterministic (fixed reduction order), stream-ordered and allocation-free.
#include "common.cuh"

namespace sige {

// Programmatic dependent launch for the glue kernels: each one releases its successor right away
// (pdl_release: the successor's launch latency and constant staging overlap this kernel) and waits for its
// predecessor's results just before the first dependent read (pdl_acquire; a no-op when the launch carries no
// programmatic edge).  Always on: both instructions are harmless in an ordinary stream, and every glue launch carries
// the PDL attribute (launch_ex errors surface through check_launch()).

// ------------------------------------------------------------------------------------------
// conv_in: Cin <= 4, Cout % 8 == 0.  One thread = one pixel x 8 output channels (one 16-byte store);
// the 9*Cin inputs come through L1, the 9*Cin*8 weights of the thread's channel octet from shared.
// ------------------------------------------------------------------------------------------
__host__ __device__ inline int conv_in_pitch(int Cin) {
    int v = 9 * Cin * 2;          // row length in 16-byte units
    if ((v & 1) == 0) ++v;        // make it odd
    return v * 4;                 // floats
}

struct InAux {
    void *ptr;
    const float *scale, *shift;
    int act;
};

// One thread = 4 horizontally adjacent pixels x 8 output channels: each weight octet read from shared memory is used
// four times (the weight reads were the bottleneck of the one-pixel version: 54 LDS.128 per pixel), each input value
// up to three times.  Requires W % 4 == 0.
template <typename T>
__global__ void __launch_bounds__(256) conv_in_kernel(const T *__restrict__ x, const T *__restrict__ w, const T *__restrict__ bias,
                                                      T *__restrict__ out, int B, int H, int W, int Cin, int Cout, int n_aux, InAux a0,
                                                      InAux a1) {
    extern __shared__ float wsm[];   // [Cout/8][pitch] (rows of 9*Cin*8 weights, padded) + bias [Cout]
    const int K = 9 * Cin, OV = Cout / 8;
    const int pitch = conv_in_pitch(Cin);
    for (int e0 = threadIdx.x; e0 < Cout * K; e0 += blockDim.x * 8) {      // 8 coalesced loads in flight per thread
        T v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) { const int e = e0 + j * blockDim.x; v[j] = e < Cout * K ? w[e] : DT<T>::from_f(0.f); }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int e = e0 + j * blockDim.x;
            if (e >= Cout * K) break;
            const int co = e / K, k = e - co * K;          // k = ci*9 + tap in OIHW
            const int ci = k / 9, tap = k - ci * 9;
            wsm[(co >> 3) * pitch + (tap * Cin + ci) * 8 + (co & 7)] = DT<T>::to_f(v[j]);
        }
    }
    float *bsm = wsm + OV * pitch;
    for (int e = threadIdx.x; e < Cout; e += blockDim.x) bsm[e] = bias ? DT<T>::to_f(bias[e]) : 0.f;
    pdl_release();
    __syncthreads();
    pdl_acquire();
    const int WQ = W / 4;
    const int total = B * H * WQ * OV;      // < 2^29 (checked on the host), so the int loop index below cannot wrap
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int ov = i % OV;
        int q = i / OV;
        const int wq = q % WQ; q /= WQ;
        const int hh = q % H;
        const int b = q / H;
        const int w0 = wq * 4;
        float acc[4][8];
#pragma unroll
        for (int px = 0; px < 4; ++px)
#pragma unroll
            for (int z = 0; z < 8; ++z) acc[px][z] = bsm[ov * 8 + z];
        const float *wv = wsm + ov * pitch;
        for (int ky = 0; ky < 3; ++ky) {
            const int y = hh + ky - 1;
            if (y < 0 || y >= H) continue;
            const T *row = x + ((long long)b * H + y) * W * Cin;
            for (int ci = 0; ci < Cin; ++ci) {
                float in[6];                                  // columns w0-1 .. w0+4
#pragma unroll
                for (int c = 0; c < 6; ++c) {
                    const int xx = w0 - 1 + c;
                    in[c] = (xx >= 0 && xx < W) ? DT<T>::to_f(row[(long long)xx * Cin + ci]) : 0.f;
                }
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const float4 wa = *reinterpret_cast<const float4 *>(wv + ((ky * 3 + kx) * Cin + ci) * 8);
                    const float4 wb = *reinterpret_cast<const float4 *>(wv + ((ky * 3 + kx) * Cin + ci) * 8 + 4);
                    const float wz[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w};
#pragma unroll
                    for (int px = 0; px < 4; ++px)
#pragma unroll
                        for (int z = 0; z < 8; ++z) acc[px][z] = fmaf(in[px + kx], wz[z], acc[px][z]);
                }
            }
        }
        float sc0[8], sh0[8], sc1[8], sh1[8];
#pragma unroll
        for (int z = 0; z < 8; ++z) {
            sc0[z] = (n_aux > 0 && a0.scale) ? __ldg(a0.scale + ov * 8 + z) : 1.f;
            sh0[z] = (n_aux > 0 && a0.shift) ? __ldg(a0.shift + ov * 8 + z) : 0.f;
            sc1[z] = (n_aux > 1 && a1.scale) ? __ldg(a1.scale + ov * 8 + z) : 1.f;
            sh1[z] = (n_aux > 1 && a1.shift) ? __ldg(a1.shift + ov * 8 + z) : 0.f;
        }
#pragma unroll
        for (int px = 0; px < 4; ++px) {
            const long long o8 = ((((long long)b * H + hh) * W + w0 + px) * OV + ov) * 8;
            uint4 o;
            T *oe = reinterpret_cast<T *>(&o);
#pragma unroll
            for (int z = 0; z < 8; ++z) oe[z] = DT<T>::from_f(acc[px][z]);
            *reinterpret_cast<uint4 *>(out + o8) = o;
            if (n_aux > 0) {   // the consumers' GroupNorm affine + SiLU, applied once here
                uint4 oa;
                T *ae = reinterpret_cast<T *>(&oa);
#pragma unroll
                for (int z = 0; z < 8; ++z) ae[z] = DT<T>::from_f(activate<true>(a0.act, fmaf(acc[px][z], sc0[z], sh0[z])));
                *reinterpret_cast<uint4 *>(reinterpret_cast<T *>(a0.ptr) + o8) = oa;
            }
            if (n_aux > 1) {
                uint4 oa;
                T *ae = reinterpret_cast<T *>(&oa);
#pragma unroll
                for (int z = 0; z < 8; ++z) ae[z] = DT<T>::from_f(activate<true>(a1.act, fmaf(acc[px][z], sc1[z], sh1[z])));
                *reinterpret_cast<uint4 *>(reinterpret_cast<T *>(a1.ptr) + o8) = oa;
            }
        }
    }
}

// conv_in restricted to a list of R x S pixel tiles (tile t covers rows idx[2t] .. +R-1, columns idx[2t+1] .. +S-1 of
// image b = t / n_tiles; pixels outside the image are skipped).  At a small edit every later layer reads the stem's
// output only inside the active halo tiles, so this is all of it that has to exist.  One thread = one pixel x 8 output
// channels.  Overlapping tiles recompute the shared pixels and store identical values.
template <typename T>
__global__ void __launch_bounds__(256) conv_in_tiles_kernel(const T *__restrict__ x, const T *__restrict__ w, const T *__restrict__ bias,
                                                            T *__restrict__ out, int H, int W, int Cin, int Cout,
                                                            const int32_t *__restrict__ idx, int n_tiles, int NT, int R, int S,
                                                            int idx_per_image, int n_aux, InAux a0, InAux a1) {
    extern __shared__ float wsm[];   // same layout as conv_in_kernel
    const int K = 9 * Cin, OV = Cout / 8;
    const int pitch = conv_in_pitch(Cin);
    for (int e0 = threadIdx.x; e0 < Cout * K; e0 += blockDim.x * 8) {      // 8 coalesced loads in flight per thread
        T v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) { const int e = e0 + j * blockDim.x; v[j] = e < Cout * K ? w[e] : DT<T>::from_f(0.f); }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int e = e0 + j * blockDim.x;
            if (e >= Cout * K) break;
            const int co = e / K, k = e - co * K;
            const int ci = k / 9, tap = k - ci * 9;
            wsm[(co >> 3) * pitch + (tap * Cin + ci) * 8 + (co & 7)] = DT<T>::to_f(v[j]);
        }
    }
    float *bsm = wsm + OV * pitch;
    for (int e = threadIdx.x; e < Cout; e += blockDim.x) bsm[e] = bias ? DT<T>::to_f(bias[e]) : 0.f;
    pdl_release();
    __syncthreads();
    pdl_acquire();
    const int total = NT * R * S * OV;      // < 2^31 - 1 (checked on the host)
    // long long: the last stride past `total` can pass 2^31
    for (long long i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int ov = (int)i % OV;
        int q = (int)i / OV;
        const int xx = q % S; q /= S;
        const int yy = q % R;
        const int t = q / R;
        const int b = t / n_tiles, tt = idx_per_image ? t : t - b * n_tiles;      // per-image lists: row b*n_tiles + i
        const int hh = __ldg(idx + 2LL * tt) + yy, ww = __ldg(idx + 2LL * tt + 1) + xx;
        if (hh < 0 || hh >= H || ww < 0 || ww >= W) continue;
        float acc[8];
#pragma unroll
        for (int z = 0; z < 8; ++z) acc[z] = bsm[ov * 8 + z];
        const float *wv = wsm + ov * pitch;
        for (int ky = 0; ky < 3; ++ky) {
            const int y = hh + ky - 1;
            if (y < 0 || y >= H) continue;
            const T *row = x + ((long long)b * H + y) * W * Cin;
            for (int ci = 0; ci < Cin; ++ci) {             // same accumulation order as conv_in_kernel: bit-identical results
                for (int kx = 0; kx < 3; ++kx) {
                    const int xc = ww + kx - 1;
                    if (xc < 0 || xc >= W) continue;
                    const float in = DT<T>::to_f(row[(long long)xc * Cin + ci]);
                    const float4 wa = *reinterpret_cast<const float4 *>(wv + ((ky * 3 + kx) * Cin + ci) * 8);
                    const float4 wb = *reinterpret_cast<const float4 *>(wv + ((ky * 3 + kx) * Cin + ci) * 8 + 4);
                    acc[0] = fmaf(in, wa.x, acc[0]); acc[1] = fmaf(in, wa.y, acc[1]); acc[2] = fmaf(in, wa.z, acc[2]); acc[3] = fmaf(in, wa.w, acc[3]);
                    acc[4] = fmaf(in, wb.x, acc[4]); acc[5] = fmaf(in, wb.y, acc[5]); acc[6] = fmaf(in, wb.z, acc[6]); acc[7] = fmaf(in, wb.w, acc[7]);
                }
            }
        }
        const long long o8 = ((((long long)b * H + hh) * W + ww) * OV + ov) * 8;
        uint4 o;
        T *oe = reinterpret_cast<T *>(&o);
#pragma unroll
        for (int z = 0; z < 8; ++z) oe[z] = DT<T>::from_f(acc[z]);
        *reinterpret_cast<uint4 *>(out + o8) = o;
        for (int ax = 0; ax < n_aux; ++ax) {   // the consumers' GroupNorm affine + SiLU, applied once here
            const InAux &A = ax == 0 ? a0 : a1;
            uint4 oa;
            T *ae = reinterpret_cast<T *>(&oa);
#pragma unroll
            for (int z = 0; z < 8; ++z) {
                const float sc = A.scale ? __ldg(A.scale + ov * 8 + z) : 1.f, sh = A.shift ? __ldg(A.shift + ov * 8 + z) : 0.f;
                ae[z] = DT<T>::from_f(activate<true>(A.act, fmaf(acc[z], sc, sh)));
            }
            *reinterpret_cast<uint4 *>(reinterpret_cast<T *>(A.ptr) + o8) = oa;
        }
    }
}

// ------------------------------------------------------------------------------------------
// GroupNorm fold.  Stage 1: every CTA reduces a contiguous pixel range to per-channel (sum, sumsq);
// stage 2: one CTA adds the partials in a fixed order and emits scale = gamma*rstd,
// shift = beta - mean*rstd*gamma  (GroupNorm(x) == x*scale + shift, reference models/common.py:37-57).
// ------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) gn_partial_kernel(const T *__restrict__ x, int HW, int C, float *__restrict__ part, int nblk) {
    // grid = (nblk, B); thread = (pixel slot, channel octet)
    const int CV = C / 8;
    const int slots = blockDim.x / CV;
    const int cv = threadIdx.x % CV, slot = threadIdx.x / CV;
    const int b = blockIdx.y;
    // HW < 2^31 (checked on the host); the pixel positions are long long because the last CTA's range and loop steps may pass it
    const int per = HW / nblk + (HW % nblk != 0);
    const long long p0 = (long long)blockIdx.x * per, p1 = min((long long)HW, p0 + per);
    pdl_release();
    pdl_acquire();
    float s[8], q[8];
#pragma unroll
    for (int z = 0; z < 8; ++z) { s[z] = 0.f; q[z] = 0.f; }
    if (slot < slots) {
        constexpr int GB = 8;     // loads in flight per thread (same summation order as a plain loop)
        for (long long pb = p0 + slot; pb < p1; pb += slots * GB) {
            uint4 v[GB];
#pragma unroll
            for (int j = 0; j < GB; ++j) {
                const long long p = pb + j * slots;
                v[j] = make_uint4(0, 0, 0, 0);
                if (p < p1) v[j] = __ldg(reinterpret_cast<const uint4 *>(x + ((long long)b * HW + p) * C + cv * 8));
            }
#pragma unroll
            for (int j = 0; j < GB; ++j) {
                if (pb + j * slots >= p1) break;
                const T *e = reinterpret_cast<const T *>(&v[j]);
#pragma unroll
                for (int z = 0; z < 8; ++z) { const float f = DT<T>::to_f(e[z]); s[z] += f; q[z] = fmaf(f, f, q[z]); }
            }
        }
    }
    extern __shared__ float red[];   // [slots][C][2]
    if (slot < slots) {
#pragma unroll
        for (int z = 0; z < 8; ++z) { red[(slot * C + cv * 8 + z) * 2] = s[z]; red[(slot * C + cv * 8 + z) * 2 + 1] = q[z]; }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float ss = 0.f, qq = 0.f;
        for (int sl = 0; sl < slots; ++sl) { ss += red[(sl * C + c) * 2]; qq += red[(sl * C + c) * 2 + 1]; }
        float *o = part + (((long long)b * nblk + blockIdx.x) * C + c) * 2;
        o[0] = ss; o[1] = qq;
    }
}

template <typename T>
__global__ void __launch_bounds__(1024) gn_finalize_kernel(const float *__restrict__ part, int nblk, int HW, int C, int G, float eps,
                                                           const T *__restrict__ gamma, const T *__restrict__ beta,
                                                           float *__restrict__ scale, float *__restrict__ shift, int CPB) {
    // grid = (C / CPB, B): a CTA owns CPB channels (whole groups); block = 1024 threads = S slices x CPB channels;
    // fixed summation order -> deterministic
    extern __shared__ double dsm[];   // [S][CPB][2]
    const int b = blockIdx.y, c0 = blockIdx.x * CPB;
    const int S = max(1, (int)blockDim.x / CPB);
    const int cl = threadIdx.x % CPB, sl = threadIdx.x / CPB;
    const int c = c0 + cl;
    pdl_release();
    pdl_acquire();
    if (sl < S) {
        double ss = 0.0, qq = 0.0;
        constexpr int FB = 8;     // loads in flight per thread (same summation order as a plain loop)
        for (int k0 = sl; k0 < nblk; k0 += S * FB) {
            float2 v[FB];
#pragma unroll
            for (int j = 0; j < FB; ++j) {
                const int k = k0 + j * S;
                v[j] = make_float2(0.f, 0.f);
                if (k < nblk) v[j] = *reinterpret_cast<const float2 *>(part + (((long long)b * nblk + k) * C + c) * 2);
            }
#pragma unroll
            for (int j = 0; j < FB; ++j) {
                if (k0 + j * S >= nblk) break;
                ss += v[j].x; qq += v[j].y;
            }
        }
        dsm[(sl * CPB + cl) * 2] = ss; dsm[(sl * CPB + cl) * 2 + 1] = qq;
    }
    __syncthreads();
    if (threadIdx.x < CPB) {
        double ss = 0.0, qq = 0.0;
        for (int k = 0; k < S; ++k) { ss += dsm[(k * CPB + cl) * 2]; qq += dsm[(k * CPB + cl) * 2 + 1]; }
        dsm[cl * 2] = ss; dsm[cl * 2 + 1] = qq;         // slice 0 row now holds the per-channel totals
    }
    __syncthreads();
    if (threadIdx.x < CPB) {
        const int per = C / G, gl = cl / per;           // CPB is a multiple of the group size
        double ss = 0.0, qq = 0.0;
        for (int k = 0; k < per; ++k) { ss += dsm[2 * (gl * per + k)]; qq += dsm[2 * (gl * per + k) + 1]; }
        const double n = (double)per * HW;
        const double mean = ss / n;
        double var = qq / n - mean * mean;
        if (var < 0) var = 0;
        const float rstd = (float)(1.0 / sqrt(var + (double)eps));
        const float ga = gamma ? DT<T>::to_f(gamma[c]) : 1.f, be = beta ? DT<T>::to_f(beta[c]) : 0.f;
        scale[(long long)b * C + c] = ga * rstd;
        shift[(long long)b * C + c] = be - (float)mean * rstd * ga;
    }
}

// ------------------------------------------------------------------------------------------
// conv_out: y = conv3x3(act(x*scale+shift)), C -> Cout <= 8, output NCHW.
// CTA = 8 x 32 output pixels, one warp per output row.  The (8+2) x (32+2) halo is transformed ONCE into shared
// memory (row pitch cc*2+16 bytes -> conflict-free ldmatrix), then the conv is an implicit GEMM on the legacy tensor
// path: M = 16 consecutive pixels of the row, N = 8 (Cout zero-padded), K = 9*C, mma.sync.m16n8k16; the A fragment of
// tap (ky,kx) is a set of ldmatrix row pointers into the halo tile shifted by (ky,kx).
// The halo holds cc channels at a time (cc divides C): all of them when they fit beside the weights, else the halo is
// filled and consumed once per chunk of cc channels (the Stable Diffusion VAE encoder's 512-channel conv_out), with the
// accumulators carried across chunks.  With cc == C the MMA order is the single-fill order.
// ------------------------------------------------------------------------------------------
constexpr int CO_TH = 8, CO_TW = 32;

static size_t conv_out_smem(int C, int cc) {
    return (((size_t)(CO_TH + 2) * (CO_TW + 2) * (cc * 2 + 16) + 15) & ~(size_t)15) + (size_t)8 * (9 * C * 2 + 16);
}

// Channels per halo fill: the largest multiple of 16 that divides C and fits in shared memory beside the weights (0: none).
static int conv_out_chunk(int C) {
    for (int cc = C; cc >= 16; cc -= 16)
        if (C % cc == 0 && conv_out_smem(C, cc) <= 227 * 1024) return cc;
    return 0;
}

template <typename T>
__global__ void __launch_bounds__(CO_TH * 32) conv_out_kernel(const T *__restrict__ x, const float *__restrict__ scale,
                                                                const float *__restrict__ shift, int act, const T *__restrict__ w,
                                                                const T *__restrict__ bias, T *__restrict__ out, int B, int H, int W,
                                                                int C, int Cout, int cc) {
    extern __shared__ __align__(16) unsigned char smraw[];
    const int pitch = cc * 2 + 16;
    const int HP = CO_TH + 2, WP = CO_TW + 2;
    const int K = 9 * C, wpitch = K * 2 + 16;                                 // bytes per weight row (odd number of 16-byte units)
    unsigned char *tile = smraw;                                             // [HP*WP][pitch]: channels c0 .. c0+cc-1
    unsigned char *wsm = smraw + ((HP * WP * pitch + 15) & ~15);             // [8][wpitch]: B operand, row n = output channel
    const int b = blockIdx.z, ty0 = blockIdx.y * CO_TH, tx0 = blockIdx.x * CO_TW;
    {
        constexpr int WB = 8;     // weight elements in flight per thread (the staging is a chain of scattered 2-byte loads)
        for (int e0 = threadIdx.x; e0 < 8 * K; e0 += blockDim.x * WB) {
            T v[WB];
#pragma unroll
            for (int j = 0; j < WB; ++j) {
                const int e = e0 + j * blockDim.x;
                const int n = e / K, k = e - n * K;                          // k = tap*C + ci
                const int tap = k / C, ci = k - tap * C;
                v[j] = (e < 8 * K && n < Cout) ? w[((long long)n * C + ci) * 9 + tap] : DT<T>::from_f(0.f);
            }
#pragma unroll
            for (int j = 0; j < WB; ++j) {
                const int e = e0 + j * blockDim.x;
                if (e >= 8 * K) break;
                const int n = e / K, k = e - n * K;
                *reinterpret_cast<T *>(wsm + n * wpitch + k * 2) = v[j];
            }
        }
    }
    const int CV = cc / 8;
    const bool pre = scale || shift || act != SIGE_ACT_IDENTITY;
    pdl_release();
    pdl_acquire();                 // the weights above are constants; x, scale and shift come from the preceding kernels
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;            // warp = output row inside the tile
    float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
    for (int c0 = 0; c0 < C; c0 += cc) {
        if (c0) __syncthreads();       // every warp is done with the previous chunk's halo
        if (blockDim.x % CV == 0) {
            // every thread keeps ONE channel octet for all its pixels: its 8 (scale, shift) pairs live in registers and the
            // pixel walk is a fixed stride (the pre-op — 11 M SiLU evaluations per 256x256x128 step — is this kernel's cost)
            const int cv = threadIdx.x % CV, pstep = blockDim.x / CV;
            float sc[8], sh[8];
#pragma unroll
            for (int z = 0; z < 8; ++z) {
                sc[z] = scale ? __ldg(scale + (long long)b * C + c0 + cv * 8 + z) : 1.f;
                sh[z] = shift ? __ldg(shift + (long long)b * C + c0 + cv * 8 + z) : 0.f;
            }
            // loads are issued in batches of HB before any is consumed: one DRAM round trip per batch instead of per pixel
            constexpr int HB = 8;
            for (int pp0 = threadIdx.x / CV; pp0 < HP * WP; pp0 += pstep * HB) {
                uint4 v[HB];
                bool ok[HB];
#pragma unroll
                for (int j = 0; j < HB; ++j) {
                    const int pp = pp0 + j * pstep;
                    const int py = pp / WP, px = pp - py * WP;
                    const int hh = ty0 + py - 1, ww = tx0 + px - 1;
                    ok[j] = pp < HP * WP && hh >= 0 && hh < H && ww >= 0 && ww < W;
                    v[j] = make_uint4(0, 0, 0, 0);
                    if (ok[j]) v[j] = __ldg(reinterpret_cast<const uint4 *>(x + (((long long)b * H + hh) * W + ww) * C + c0 + cv * 8));
                }
#pragma unroll
                for (int j = 0; j < HB; ++j) {
                    const int pp = pp0 + j * pstep;
                    if (pp >= HP * WP) break;
                    if (pre && ok[j]) {
                        T *el = reinterpret_cast<T *>(&v[j]);
#pragma unroll
                        for (int z = 0; z < 8; ++z) el[z] = DT<T>::from_f(activate<true>(act, fmaf(DT<T>::to_f(el[z]), sc[z], sh[z])));
                    }
                    *reinterpret_cast<uint4 *>(tile + pp * pitch + cv * 16) = v[j];   // zero padding AFTER the pre-op
                }
            }
        } else {
            for (int e = threadIdx.x; e < HP * WP * CV; e += blockDim.x) {
                const int cv = e % CV, pp = e / CV;
                const int py = pp / WP, px = pp - py * WP;
                const int hh = ty0 + py - 1, ww = tx0 + px - 1;
                uint4 v = make_uint4(0, 0, 0, 0);
                if (hh >= 0 && hh < H && ww >= 0 && ww < W) {
                    v = __ldg(reinterpret_cast<const uint4 *>(x + (((long long)b * H + hh) * W + ww) * C + c0 + cv * 8));
                    if (pre) {
                        T *el = reinterpret_cast<T *>(&v);
#pragma unroll
                        for (int z = 0; z < 8; ++z) {
                            const int c = c0 + cv * 8 + z;
                            float f = DT<T>::to_f(el[z]);
                            f = fmaf(f, scale ? scale[(long long)b * C + c] : 1.f, shift ? shift[(long long)b * C + c] : 0.f);
                            el[z] = DT<T>::from_f(activate<true>(act, f));
                        }
                    }
                }
                *reinterpret_cast<uint4 *>(tile + pp * pitch + cv * 16) = v;   // zero padding AFTER the pre-op
            }
        }
        __syncthreads();
        const uint32_t tbase = smem_u32(tile), wbase = smem_u32(wsm);
        const int a_row = lane & 15, a_khalf = lane >> 4;                      // ldmatrix.x4: 16 pixel rows x {k-lo, k-hi}
        const int b_row = lane & 7, b_khalf = (lane >> 3) & 1;                 // ldmatrix.x2: 8 channel rows x {k-lo, k-hi}
        for (int tap = 0; tap < 9; ++tap) {
            const int ky = tap / 3, kx = tap - 3 * ky;
            const uint32_t arow0 = tbase + ((warp + ky) * WP + kx + a_row) * pitch + a_khalf * 16;
            const uint32_t brow = wbase + b_row * wpitch + (tap * C + c0) * 2 + b_khalf * 16;
            for (int kk = 0; kk < cc / 16; ++kk) {
                uint32_t b0, b1;
                asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];\n" : "=r"(b0), "=r"(b1) : "r"(brow + kk * 32));
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    uint32_t a[4];
                    ldmatrix_x4(arow0 + i * 16 * pitch + kk * 32, a[0], a[1], a[2], a[3]);
                    mma_m16n8k16<T>(acc[i], a, b0, b1);
                }
            }
        }
    }
    // accumulator fragment: rows (pixels) lane/4 and lane/4+8, columns (channels) 2*(lane%4), +1
    const int hh = ty0 + warp;
    if (hh < H) {
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const int ww = tx0 + i * 16 + (lane >> 2) + half * 8;
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const int co = 2 * (lane & 3) + q;
                    if (co < Cout && ww < W)
                        out[(((long long)b * Cout + co) * H + hh) * W + ww] =
                            DT<T>::from_f(acc[i][half * 2 + q] + (bias ? DT<T>::to_f(bias[co]) : 0.f));
                }
            }
    }
}

}  // namespace sige

using namespace sige;

// Weights of more than 48 KB (Cout > ~320: the Stable Diffusion VAE decoder's 4 -> 512 stem) need the dynamic shared-memory opt-in.
template <typename K> static bool conv_in_smem_ok(K kernel, size_t smem) {
    if (smem <= 48 * 1024) return true;
    if (smem > 227 * 1024 || cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
        (void)cudaGetLastError();
        return false;
    }
    return true;
}

extern "C" {

int sige_conv_in_nhwc(const void *x, const void *w, const void *bias, void *out, int dtype, int B, int H, int W, int Cin, int Cout,
                      int n_aux, const sige_conv_aux_t *aux, sige_stream_t stream) {
    SIGE_REQUIRE(x && w && out, "sige_conv_in_nhwc: null pointer");
    SIGE_REQUIRE(B > 0 && H > 0 && W > 0 && W % 4 == 0 && Cin >= 1 && Cin <= 4 && Cout > 0 && Cout % 8 == 0, "sige_conv_in_nhwc: needs W %% 4 == 0, Cin <= 4 and Cout %% 8 == 0");
    SIGE_REQUIRE(((uintptr_t)out & 15) == 0, "sige_conv_in_nhwc: output not 16-byte aligned");
    const size_t smem = sizeof(float) * ((size_t)(Cout / 8) * conv_in_pitch(Cin) + Cout);
    SIGE_REQUIRE(dtype != SIGE_F16 || conv_in_smem_ok(conv_in_kernel<__half>, smem), "sige_conv_in_nhwc: weights do not fit in shared memory");
    SIGE_REQUIRE(dtype != SIGE_BF16 || conv_in_smem_ok(conv_in_kernel<__nv_bfloat16>, smem), "sige_conv_in_nhwc: weights do not fit in shared memory");
    const long long total = (long long)B * H * (W / 4) * (Cout / 8);
    SIGE_REQUIRE(total * 4 < 2147483647LL, "sige_conv_in_nhwc: tensor too large");
    const long long want_blocks = (total + 255) / 256;
    const int grid = (int)(want_blocks < 2LL * sm_count() ? want_blocks : 2LL * sm_count());   // persistent: the weight staging is paid once per CTA
    cudaStream_t st = (cudaStream_t)stream;
    SIGE_REQUIRE(n_aux >= 0 && n_aux <= 2 && (n_aux == 0 || aux), "sige_conv_in_nhwc: n_aux must be 0..2");
    InAux ia[2] = {{nullptr, nullptr, nullptr, 0}, {nullptr, nullptr, nullptr, 0}};
    for (int i = 0; i < n_aux; ++i) {
        SIGE_REQUIRE(aux[i].ptr && aux[i].C == Cout && aux[i].c0 == 0 && ((uintptr_t)aux[i].ptr & 15) == 0, "sige_conv_in_nhwc: bad aux destination %d", i);
        SIGE_REQUIRE(aux[i].act == SIGE_ACT_IDENTITY || aux[i].act == SIGE_ACT_SWISH, "sige_conv_in_nhwc: aux %d unknown activation %d", i, aux[i].act);
        ia[i] = InAux{aux[i].ptr, aux[i].scale, aux[i].shift, aux[i].act};
    }
    switch (dtype) {
        case SIGE_F16: (void)launch_ex(conv_in_kernel<__half>, dim3(grid), dim3(256), smem, st, true, dim3(1, 1, 1), (const __half *)x, (const __half *)w, (const __half *)bias, (__half *)out, B, H, W, Cin, Cout, n_aux, ia[0], ia[1]); break;
        case SIGE_BF16: (void)launch_ex(conv_in_kernel<__nv_bfloat16>, dim3(grid), dim3(256), smem, st, true, dim3(1, 1, 1), (const __nv_bfloat16 *)x, (const __nv_bfloat16 *)w, (const __nv_bfloat16 *)bias, (__nv_bfloat16 *)out, B, H, W, Cin, Cout, n_aux, ia[0], ia[1]); break;
        default: set_error("sige_conv_in_nhwc: dtype must be f16/bf16"); return 1;
    }
    return check_launch("sige_conv_in_nhwc");
}

int sige_conv_in_nhwc_tiles(const void *x, const void *w, const void *bias, void *out, int dtype, int B, int H, int W, int Cin, int Cout,
                            const int32_t *idx, int n_tiles, int R, int S, int idx_per_image, int n_aux, const sige_conv_aux_t *aux,
                            sige_stream_t stream) {
    SIGE_REQUIRE(x && w && out && idx, "sige_conv_in_nhwc_tiles: null pointer");
    SIGE_REQUIRE(B > 0 && H > 0 && W > 0 && Cin >= 1 && Cin <= 4 && Cout > 0 && Cout % 8 == 0, "sige_conv_in_nhwc_tiles: needs Cin <= 4 and Cout %% 8 == 0");
    SIGE_REQUIRE(n_tiles >= 0 && R > 0 && S > 0, "sige_conv_in_nhwc_tiles: bad tile list");
    SIGE_REQUIRE(((uintptr_t)out & 15) == 0, "sige_conv_in_nhwc_tiles: output not 16-byte aligned");
    if (n_tiles == 0) return 0;
    const size_t smem = sizeof(float) * ((size_t)(Cout / 8) * conv_in_pitch(Cin) + Cout);
    SIGE_REQUIRE(dtype != SIGE_F16 || conv_in_smem_ok(conv_in_tiles_kernel<__half>, smem), "sige_conv_in_nhwc_tiles: weights do not fit in shared memory");
    SIGE_REQUIRE(dtype != SIGE_BF16 || conv_in_smem_ok(conv_in_tiles_kernel<__nv_bfloat16>, smem), "sige_conv_in_nhwc_tiles: weights do not fit in shared memory");
    const long long NT = (long long)B * n_tiles;
    const long long total = NT * R * S * (Cout / 8);
    SIGE_REQUIRE(total < 2147483647LL && (long long)B * H * W * Cout < 2147483647LL * 8, "sige_conv_in_nhwc_tiles: tensor too large");
    const long long want_blocks = (total + 255) / 256;
    const int grid = (int)(want_blocks < 4LL * sm_count() ? want_blocks : 4LL * sm_count());
    cudaStream_t st = (cudaStream_t)stream;
    SIGE_REQUIRE(n_aux >= 0 && n_aux <= 2 && (n_aux == 0 || aux), "sige_conv_in_nhwc_tiles: n_aux must be 0..2");
    InAux ia[2] = {{nullptr, nullptr, nullptr, 0}, {nullptr, nullptr, nullptr, 0}};
    for (int i = 0; i < n_aux; ++i) {
        SIGE_REQUIRE(aux[i].ptr && aux[i].C == Cout && aux[i].c0 == 0 && ((uintptr_t)aux[i].ptr & 15) == 0, "sige_conv_in_nhwc_tiles: bad aux destination %d", i);
        SIGE_REQUIRE(aux[i].act == SIGE_ACT_IDENTITY || aux[i].act == SIGE_ACT_SWISH, "sige_conv_in_nhwc_tiles: aux %d unknown activation %d", i, aux[i].act);
        ia[i] = InAux{aux[i].ptr, aux[i].scale, aux[i].shift, aux[i].act};
    }
    switch (dtype) {
        case SIGE_F16: (void)launch_ex(conv_in_tiles_kernel<__half>, dim3(grid), dim3(256), smem, st, true, dim3(1, 1, 1), (const __half *)x, (const __half *)w, (const __half *)bias, (__half *)out, H, W, Cin, Cout, idx, n_tiles, (int)NT, R, S, idx_per_image, n_aux, ia[0], ia[1]); break;
        case SIGE_BF16: (void)launch_ex(conv_in_tiles_kernel<__nv_bfloat16>, dim3(grid), dim3(256), smem, st, true, dim3(1, 1, 1), (const __nv_bfloat16 *)x, (const __nv_bfloat16 *)w, (const __nv_bfloat16 *)bias, (__nv_bfloat16 *)out, H, W, Cin, Cout, idx, n_tiles, (int)NT, R, S, idx_per_image, n_aux, ia[0], ia[1]); break;
        default: set_error("sige_conv_in_nhwc_tiles: dtype must be f16/bf16"); return 1;
    }
    return check_launch("sige_conv_in_nhwc_tiles");
}

// partial-sum blocks of the GroupNorm reduction: two per SM of the current device (the workspace query and the call must see
// the same device)
static int gn_partial_blocks() { return 2 * sm_count(); }

static long long gn_workspace_floats(int B, int nblk, int C) { return (long long)B * nblk * C * 2; }

int sige_group_norm_fold_workspace(int B, int C) {
    const long long n = gn_workspace_floats(B, gn_partial_blocks(), C);
    if (n <= 2147483647LL) return (int)n;
    set_error("sige_group_norm_fold_workspace: %lld floats exceed 2^31 - 1", n);
    return -1;
}

int sige_group_norm_fold(const void *x, int dtype, int B, int H, int W, int C, int groups, float eps, const void *gamma, const void *beta,
                         float *scale, float *shift, float *workspace, int workspace_floats, sige_stream_t stream) {
    SIGE_REQUIRE(x && scale && shift && workspace, "sige_group_norm_fold: null pointer");
    SIGE_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && C <= 1024 && groups > 0 && C % groups == 0, "sige_group_norm_fold: bad shape (C %% 8, C <= 1024)");
    SIGE_REQUIRE(((uintptr_t)x & 15) == 0, "sige_group_norm_fold: input not 16-byte aligned");
    SIGE_REQUIRE((long long)H * W <= 2147483647LL, "sige_group_norm_fold: image too large (H * W = %lld, the limit is 2^31 - 1)", (long long)H * W);
    const int HW = H * W;
    int nblk = min(gn_partial_blocks(), max(1, HW / 64));
    SIGE_REQUIRE(workspace_floats >= gn_workspace_floats(B, nblk, C), "sige_group_norm_fold: workspace too small (%d floats, need %lld)", workspace_floats, gn_workspace_floats(B, nblk, C));
    const int CV = C / 8;
    SIGE_REQUIRE(CV <= 256, "sige_group_norm_fold: too many channels");
    const int slots = 256 / CV;
    const size_t smem1 = sizeof(float) * (size_t)slots * C * 2;
    cudaStream_t st = (cudaStream_t)stream;
    dim3 g1(nblk, B);
    // finalize: 32 channels per CTA when that is a whole number of groups (4 CTAs x 32 slices for C = 128), else one CTA
    const int per_group = C / groups;
    const int cpb = (C % 32 == 0 && 32 % per_group == 0) ? 32 : C;
#define SIGE_GN(T)                                                                                                                       \
    do {                                                                                                                                 \
        if (smem1 > 48 * 1024) cudaFuncSetAttribute(gn_partial_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem1);        \
        (void)launch_ex(gn_partial_kernel<T>, g1, dim3(256), smem1, st, true, dim3(1, 1, 1), (const T *)x, HW, C, workspace, nblk);       \
        (void)launch_ex(gn_finalize_kernel<T>, dim3(C / cpb, B), dim3(1024), sizeof(double) * 2 * cpb * (1024 / cpb > 0 ? 1024 / cpb : 1), \
                        st, true, dim3(1, 1, 1), (const float *)workspace, nblk, HW, C, groups, eps, (const T *)gamma, (const T *)beta,    \
                        scale, shift, cpb);                                                                                                \
    } while (0)
    switch (dtype) {
        case SIGE_F16: SIGE_GN(__half); break;
        case SIGE_BF16: SIGE_GN(__nv_bfloat16); break;
        default: set_error("sige_group_norm_fold: dtype must be f16/bf16"); return 1;
    }
#undef SIGE_GN
    return check_launch("sige_group_norm_fold");
}

int sige_conv_out_nhwc(const void *x, const float *scale, const float *shift, int act, const void *w, const void *bias, void *out, int dtype,
                       int B, int H, int W, int C, int Cout, sige_stream_t stream) {
    SIGE_REQUIRE(x && w && out, "sige_conv_out_nhwc: null pointer");
    SIGE_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && C % 16 == 0 && Cout >= 1 && Cout <= 8, "sige_conv_out_nhwc: needs C %% 16 == 0 and Cout <= 8");
    SIGE_REQUIRE(act == SIGE_ACT_IDENTITY || act == SIGE_ACT_SWISH, "sige_conv_out_nhwc: unknown activation %d", act);
    SIGE_REQUIRE(((uintptr_t)x & 15) == 0, "sige_conv_out_nhwc: input not 16-byte aligned");
    const int cc = conv_out_chunk(C);
    SIGE_REQUIRE(cc > 0, "sige_conv_out_nhwc: %d channels do not fit in shared memory", C);
    const size_t smem = conv_out_smem(C, cc);
    dim3 grid((W + CO_TW - 1) / CO_TW, (H + CO_TH - 1) / CO_TH, B);
    cudaStream_t st = (cudaStream_t)stream;
#define SIGE_CO(T)                                                                                                        \
    do {                                                                                                                  \
        cudaFuncSetAttribute(conv_out_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);                  \
        (void)launch_ex(conv_out_kernel<T>, grid, dim3(CO_TH * 32), smem, st, true, dim3(1, 1, 1), (const T *)x, scale, shift, act,  \
                        (const T *)w, (const T *)bias, (T *)out, B, H, W, C, Cout, cc);                                               \
    } while (0)
    switch (dtype) {
        case SIGE_F16: SIGE_CO(__half); break;
        case SIGE_BF16: SIGE_CO(__nv_bfloat16); break;
        default: set_error("sige_conv_out_nhwc: dtype must be f16/bf16"); return 1;
    }
#undef SIGE_CO
    return check_launch("sige_conv_out_nhwc");
}

}  // extern "C"
