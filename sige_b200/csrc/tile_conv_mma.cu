// tile_conv_mma.cu — fused gather -> (affine + SiLU) -> tile convolution -> (+bias, +residual)
// -> scatter, ONE launch per wrapped layer, fp16/bf16 storage, fp32 accumulation, NHWC.
//
// Replaces, for one layer, the reference's call triple
//     Gather.forward  (sige/nn/gather.py:76-89  -> sige/cuda/gather_kernel.cu)
//     SIGEConv2d      (sige/nn/base.py:88-89    -> cuDNN on the [B*N, C, R, S] stack)
//     Scatter.forward (sige/nn/scatter.py:41-60 -> y.clone() + sige/cuda/scatter_kernel.cu)
// and, because the source may be the previous layer's in-place-updated full tensor, also
// ScatterGather (sige/cuda/scatter_gather_kernel.cu) — no scatter map is needed.
//
// Formulation: implicit GEMM.  M = (active tiles) x (Ro*So output pixels), N = Cout,
// K = kH*kW*Cin.  A CTA owns `tpc` tiles and a BN-wide slice of Cout.  For every 64-channel
// chunk of Cin the halo tiles [tpc][R*S pixels][64 ch] are staged ONCE in shared memory (the
// pointwise pre-op is applied on the way in; out-of-image pixels are zero AFTER the pre-op,
// reference gather_kernel.cu:33-42) and re-used by all kH*kW taps: the A fragments of tap
// (ky,kx) are just ldmatrix row pointers into the halo tile shifted by (ky,kx).  Weights are
// pre-packed [tap][ceil(Cin/64)][Cout][64] and streamed through a cp.async ring.
// A single source whose Cin is a multiple of 8 but not of 64 (the narrow layers of pruned /
// compressed models) ends in a partial chunk: its channels >= Cin are zero in shared memory
// (never read from global memory), its weights are zero-padded, and only the k16 steps that
// hold real channels are issued — the skipped ones would add exact zeros.  The epilogue stages the
// fp32 accumulators in shared memory and writes 16-byte channel vectors straight into the
// destination tensor (coalesced 128-byte lines per pixel), adding bias and the residual.
// The MOD instantiations (sige_tile_conv_modulated) apply SPADE's modulation in the same register-staged
// halo path: leaky((x*scale + shift) * (1 + gamma) + beta) with gamma / beta read at the halo pixel, so
// the modulated tile stack the reference gathers and modulates with pointwise torch calls never exists.
//
// Tensor-core instruction: mma.sync.m16n8k16 (HMMA on sm_90a).  The wgmma/TMA variant
// for large edit ratios lives in tile_conv_tc5.cu (when built); this kernel is the latency-
// oriented path used when the GEMM M dimension is a few hundred rows.
#include <cooperative_groups.h>

#include <cmath>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace sige {

constexpr int KC = 64;        // channels per K chunk (128 bytes of fp16/bf16 per pixel row)

struct ConvSeg {
    const void *ptr;
    int pitch;   // elements from one pixel to the next: the segment's channel count, or more for a channel window of a wider
                 // NHWC buffer (sige_tile_conv_strided; ptr then points at the window's first channel)
    int up;      // nearest x2 upsample on read
};

struct AuxDst {
    void *ptr;
    int C, c0;
    const float *scale, *shift;
    int act;
};

struct ConvParams {
    ConvSeg seg[2];
    int C0;                 // channels of segment 0 (segment 1 starts here)
    int H, W;               // logical source extent
    int src_is_stack;
    const int32_t *idx;
    int N, NT;              // tiles per batch element, total tiles (B*N)
    int padded;             // SIGE_CONV_PADDED (B == 1): whole CTAs of padding may follow the real tiles
    int idx_per_image;      // 1: idx holds B*N entries (row b*N + i = tile i of image b), else N shared by all images
    int R, S, RS;
    const float *scale, *shift;
    int affine_bstride;
    int act;
    const void *w;          // [taps][ceil(Cin/64)][Cout][64], zero-padded along Cin
    const float *bias;
    int Cin, Cout, kH, kW, taps, stride;
    int Ro, So, P;          // output tile extent, pixels per tile
    int tpc;                // tiles per CTA
    int ksplit;             // split-K factor == cluster size along z (1, 2, 4 or 8)
    int pdl;                // launched with programmatic dependent launch
    void *dst;
    int dst_is_stack;
    int dH, dW, dC, dst_c0;
    int offH, offW;
    const void *residual;
    int rC, res_c0;
    int n_aux;
    AuxDst aux[2];
    // SPADE modulation in the gather stage (MOD instantiations only): gamma / beta are NHWC [B, H, W, gC / bC] at the logical
    // source extent, read from channels [g_c0 / b_c0 + c]
    const void *gamma, *beta;
    int gC, g_c0, bC, b_c0;
    float slope;
};

// swizzle key of a halo pixel at in-tile coordinates (y, x): the 8 rows of one ldmatrix 8x8
// block are 2 image rows x 4 columns of a 4x4 output tile, so (x&3 | (y&1)<<2) is distinct
// for all 8 -> conflict-free ldmatrix.
__device__ __forceinline__ int halo_key(int y, int x) { return (x & 3) | ((y & 1) << 2); }

template <typename T, int WM, int WN, int WARPS_M, int WARPS_N, int HALO_PIX, int NSTAGE>
struct ConvCfg {
    static constexpr int BM = WARPS_M * WM * 16;
    static constexpr int BN = WARPS_N * WN * 8;
    static constexpr int NTHREADS = 32 * WARPS_M * WARPS_N;
    static constexpr int HALO_BYTES = HALO_PIX * KC * 2;          // one halo buffer
    static constexpr int B_STAGE_BYTES = BN * KC * 2;
    static constexpr int MAIN_BYTES = 2 * HALO_BYTES + NSTAGE * B_STAGE_BYTES;
    static constexpr int EPI_PITCH = BN + 8;                      // floats
    static constexpr int EPI_BYTES = BM * EPI_PITCH * 4;
    static constexpr int SMEM_BYTES = MAIN_BYTES > EPI_BYTES ? MAIN_BYTES : EPI_BYTES;
    static constexpr int HALO_UNITS = HALO_PIX * 8;               // 16-byte units per halo buffer
    static constexpr int LOADS = (HALO_UNITS + NTHREADS - 1) / NTHREADS;
};

template <typename T, int WM, int WN, int WARPS_M, int WARPS_N, int HALO_PIX, int NSTAGE, bool MOD>
__global__ void __launch_bounds__(32 * WARPS_M * WARPS_N)
tile_conv_mma_kernel(const __grid_constant__ ConvParams p) {
    using Cfg = ConvCfg<T, WM, WN, WARPS_M, WARPS_N, HALO_PIX, NSTAGE>;
    constexpr int BM = Cfg::BM, BN = Cfg::BN, NTHREADS = Cfg::NTHREADS, LOADS = Cfg::LOADS;
    extern __shared__ __align__(128) unsigned char smem[];
    unsigned char *halo[2] = {smem, smem + Cfg::HALO_BYTES};
    unsigned char *bst = smem + 2 * Cfg::HALO_BYTES;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int warp_m = warp / WARPS_N, warp_n = warp % WARPS_N;
    const int tile0 = blockIdx.x * p.tpc;          // first tile of this CTA
    const int n0 = blockIdx.y * BN;                // first output channel of this CTA
    // fixed-capacity tile lists: a CTA whose first tile is SIGE_TILE_NONE padding has nothing to do (see tile_conv_tc5.cu)
    if (p.padded && __ldg(p.idx + 2 * tile0) <= SIGE_TILE_NONE) return;
    const int ntile = min(p.tpc, p.NT - tile0);    // tiles actually present
    const int NC = (p.Cin + KC - 1) / KC;          // K chunks (the last one partial on a narrow source)
    const int J = NC * p.taps;                     // (chunk, tap) steps of the whole K loop
    // split-K: the cluster's CTAs (rank = blockIdx.z) each take a contiguous slice of the K loop
    const int kr = blockIdx.z;
    const int j_begin = (int)(((long long)J * kr) / p.ksplit), j_end = (int)(((long long)J * (kr + 1)) / p.ksplit);
    const int c_first = j_begin / p.taps, c_last = (j_end - 1) / p.taps;

    // ---------------- halo loader bookkeeping (fixed per thread) ----------------
    // unit q -> (pixel, 16B unit u); pixel -> (tile_local, y, x)
    int ld_pix[LOADS];     // pixel index in the (logical) source image, or -1 (zero)
    int ld_img[LOADS];     // image (batch or stack row) index
    int ld_smem[LOADS];    // byte offset in the halo buffer, -1 = no work
    int ld_ab[LOADS];      // affine batch row
#pragma unroll
    for (int k = 0; k < LOADS; ++k) {
        const int q = tid + k * NTHREADS;
        ld_smem[k] = -1; ld_pix[k] = -1; ld_img[k] = 0; ld_ab[k] = 0;
        if (q < p.tpc * p.RS * 8) {
            const int pix = q >> 3, u = q & 7;
            const int tl = pix / p.RS, rem = pix - tl * p.RS;
            const int y = rem / p.S, x = rem - y * p.S;
            ld_smem[k] = pix * 128 + ((u ^ halo_key(y, x)) << 4);
            const int t = tile0 + tl;
            if (t < p.NT) {
                const int n = p.idx_per_image ? t : t % p.N, b = t / p.N;
                int hh = y, ww = x, img = t;
                if (!p.src_is_stack) {
                    hh += __ldg(p.idx + 2 * n); ww += __ldg(p.idx + 2 * n + 1); img = b;
                }
                ld_img[k] = img; ld_ab[k] = b;
                if (hh >= 0 && hh < p.H && ww >= 0 && ww < p.W) ld_pix[k] = (hh << 16) | ww;
            }
        }
    }
    uint4 ld_reg[LOADS];

    auto halo_issue = [&](int c) {   // global -> registers (raw)
        const int cbase = c * KC;
        const int sg = cbase >= p.C0 ? 1 : 0;
        const ConvSeg &seg = p.seg[sg];
        const int cl = cbase - (sg ? p.C0 : 0);
        const int Hs = p.H >> seg.up, Ws = p.W >> seg.up;
#pragma unroll
        for (int k = 0; k < LOADS; ++k) {
            ld_reg[k] = make_uint4(0, 0, 0, 0);
            const int u = (tid + k * NTHREADS) & 7;
            if (ld_smem[k] >= 0 && ld_pix[k] >= 0 && cbase + u * 8 < p.Cin) {   // channels >= Cin: zero
                const int hh = (ld_pix[k] >> 16) >> seg.up, ww = (ld_pix[k] & 0xffff) >> seg.up;
                const T *src = reinterpret_cast<const T *>(seg.ptr) +
                               (((long long)ld_img[k] * Hs + hh) * Ws + ww) * seg.pitch + cl + u * 8;
                ld_reg[k] = __ldg(reinterpret_cast<const uint4 *>(src));
            }
        }
    };
    auto halo_store = [&](int c, unsigned char *buf) {   // registers -> pre-op [-> modulation] -> shared
        const bool pre = MOD || (p.scale != nullptr) || (p.shift != nullptr) || (p.act != SIGE_ACT_IDENTITY);
#pragma unroll
        for (int k = 0; k < LOADS; ++k) {
            if (ld_smem[k] < 0) continue;
            uint4 v = ld_reg[k];
            const int ch = c * KC + ((tid + k * NTHREADS) & 7) * 8;
            if (pre && ld_pix[k] >= 0 && ch < p.Cin) {   // scale / shift hold Cin entries: padding units stay zero
                T *e = reinterpret_cast<T *>(&v);
                float sc[8], sh[8];
#pragma unroll
                for (int z = 0; z < 8; ++z) { sc[z] = 1.f; sh[z] = 0.f; }
                if (p.scale) {
                    const float4 *s4 = reinterpret_cast<const float4 *>(p.scale + (long long)ld_ab[k] * p.affine_bstride + ch);
                    const float4 a = __ldg(s4), b = __ldg(s4 + 1);
                    sc[0] = a.x; sc[1] = a.y; sc[2] = a.z; sc[3] = a.w; sc[4] = b.x; sc[5] = b.y; sc[6] = b.z; sc[7] = b.w;
                }
                if (p.shift) {
                    const float4 *s4 = reinterpret_cast<const float4 *>(p.shift + (long long)ld_ab[k] * p.affine_bstride + ch);
                    const float4 a = __ldg(s4), b = __ldg(s4 + 1);
                    sh[0] = a.x; sh[1] = a.y; sh[2] = a.z; sh[3] = a.w; sh[4] = b.x; sh[5] = b.y; sh[6] = b.z; sh[7] = b.w;
                }
                if constexpr (MOD) {
                    // leaky((x*scale + shift) * (1 + gamma) + beta) at the same (logical) pixel, rounded once; gamma / beta are
                    // only read where x is (in the image, channel < Cin)
                    const long long px = ((long long)ld_img[k] * p.H + (ld_pix[k] >> 16)) * p.W + (ld_pix[k] & 0xffff);
                    const uint4 gr = __ldg(reinterpret_cast<const uint4 *>(reinterpret_cast<const T *>(p.gamma) + px * p.gC + p.g_c0 + ch));
                    const uint4 br = __ldg(reinterpret_cast<const uint4 *>(reinterpret_cast<const T *>(p.beta) + px * p.bC + p.b_c0 + ch));
                    const T *ge = reinterpret_cast<const T *>(&gr), *be = reinterpret_cast<const T *>(&br);
#pragma unroll
                    for (int z = 0; z < 8; ++z) {
                        float f = fmaf(DT<T>::to_f(e[z]), sc[z], sh[z]);
                        f = fmaf(f, 1.f + DT<T>::to_f(ge[z]), DT<T>::to_f(be[z]));
                        e[z] = DT<T>::from_f(f < 0.f ? f * p.slope : f);
                    }
                } else {
#pragma unroll
                    for (int z = 0; z < 8; ++z) {
                        float f = fmaf(DT<T>::to_f(e[z]), sc[z], sh[z]);
                        f = activate<true>(p.act, f);
                        e[z] = DT<T>::from_f(f);
                    }
                }
            }
            *reinterpret_cast<uint4 *>(buf + ld_smem[k]) = v;
        }
    };

    // ---------------- weight tile loader ----------------
    auto b_issue = [&](int j) {
        if (j < j_end) {
            const int c = j / p.taps, tap = j - c * p.taps;
            unsigned char *st = bst + ((j - j_begin) % NSTAGE) * Cfg::B_STAGE_BYTES;
            // packed [tap][ceil(Cin/64)][Cout][64]: this CTA's slab is one contiguous run of BN*128 bytes
            const T *wbase = reinterpret_cast<const T *>(p.w) + (((long long)tap * NC + c) * p.Cout) * KC;
            for (int q = tid; q < BN * 8; q += NTHREADS) {
                const int n = q >> 3, u = q & 7;
                const bool ok = (n0 + n) < p.Cout;
                const T *src = wbase + (long long)(ok ? (n0 + n) : 0) * KC + u * 8;
                cp_async16_zfill(smem_u32(st + n * 128 + ((u ^ (n & 7)) << 4)), src, ok);
            }
        }
        cp_async_commit();
    };

    // ---------------- per-thread A row bookkeeping ----------------
    int a_pix0[WM], a_x0[WM], a_y0[WM];
#pragma unroll
    for (int i = 0; i < WM; ++i) {
        const int m = warp_m * (WM * 16) + i * 16 + (lane & 15);
        int tl = m / p.P, pp = m - tl * p.P;
        if (tl >= p.tpc) { tl = 0; pp = 0; }   // idle row: read something valid, discard later
        const int oy = pp / p.So, ox = pp - oy * p.So;
        a_y0[i] = oy * p.stride; a_x0[i] = ox * p.stride;
        a_pix0[i] = tl * p.RS + a_y0[i] * p.S + a_x0[i];
    }
    const int a_khalf = lane >> 4;
    // B row bookkeeping: lane -> (n within a 16-wide pair, k half)
    const int b_nl = ((lane >> 4) << 3) + (lane & 7);
    const int b_khalf = (lane >> 3) & 1;

    float acc[WM][WN][4];
#pragma unroll
    for (int i = 0; i < WM; ++i)
#pragma unroll
        for (int jn = 0; jn < WN; ++jn)
#pragma unroll
            for (int z = 0; z < 4; ++z) acc[i][jn][z] = 0.f;

    // ---------------- prologue ----------------
    // weights do not depend on the previous kernel: start streaming them before the grid dependency wait
#pragma unroll
    for (int s = 0; s < NSTAGE - 1; ++s) b_issue(j_begin + s);
    if (p.pdl) {
        pdl_release();   // let the next layer begin ITS weight prefetch
        pdl_acquire();   // previous layer's activations are now visible
    }
    halo_issue(c_first);
    halo_store(c_first, halo[0]);

    // ---------------- main loop over this CTA's K slice ----------------
    int hb = 0;
    for (int j = j_begin; j < j_end; ++j) {
        const int c = j / p.taps, tap = j - c * p.taps;
        if ((j == j_begin || tap == 0) && c < c_last) halo_issue(c + 1);   // prefetch the next chunk into registers
        const uint32_t hbase = smem_u32(halo[hb]);
        cp_async_wait<NSTAGE - 2>();
        __syncthreads();
        b_issue(j + NSTAGE - 1);
        const int ky = tap / p.kW, kx = tap - ky * p.kW;
        const int ksteps = min(KC / 16, (p.Cin - c * KC + 15) / 16);   // k16 steps holding real channels (4 unless partial)
        const uint32_t bbase = smem_u32(bst + ((j - j_begin) % NSTAGE) * Cfg::B_STAGE_BYTES);
        uint32_t a_addr[WM];
        int a_key[WM];
#pragma unroll
        for (int i = 0; i < WM; ++i) {
            a_addr[i] = hbase + (a_pix0[i] + ky * p.S + kx) * 128;
            a_key[i] = halo_key(a_y0[i] + ky, a_x0[i] + kx);
        }
#pragma unroll
        for (int kk = 0; kk < KC / 16; ++kk) {
            if (kk >= ksteps) break;
            uint32_t af[WM][4];
#pragma unroll
            for (int i = 0; i < WM; ++i)
                ldmatrix_x4(a_addr[i] + ((((kk << 1) | a_khalf) ^ a_key[i]) << 4), af[i][0], af[i][1], af[i][2], af[i][3]);
#pragma unroll
            for (int jp = 0; jp < WN / 2; ++jp) {
                const int n = warp_n * (WN * 8) + jp * 16 + b_nl;
                uint32_t b0, b1, b2, b3;
                ldmatrix_x4(bbase + n * 128 + ((((kk << 1) | b_khalf) ^ (n & 7)) << 4), b0, b1, b2, b3);
#pragma unroll
                for (int i = 0; i < WM; ++i) {
                    mma_m16n8k16<T>(acc[i][2 * jp], af[i], b0, b1);
                    mma_m16n8k16<T>(acc[i][2 * jp + 1], af[i], b2, b3);
                }
            }
        }
        if ((tap == p.taps - 1 || j == j_end - 1) && c < c_last) {   // chunk finished: publish the prefetched one
            halo_store(c + 1, halo[hb ^ 1]);
            hb ^= 1;
        }
    }
    cp_async_wait<0>();
    __syncthreads();

    // ---------------- epilogue: accumulators -> smem (fp32) -> 16-byte channel vectors ----------------
    float *cst = reinterpret_cast<float *>(smem);
#pragma unroll
    for (int i = 0; i < WM; ++i)
#pragma unroll
        for (int jn = 0; jn < WN; ++jn) {
            const int m = warp_m * (WM * 16) + i * 16 + (lane >> 2);
            const int n = warp_n * (WN * 8) + jn * 8 + ((lane & 3) << 1);
            *reinterpret_cast<float2 *>(cst + m * Cfg::EPI_PITCH + n) = make_float2(acc[i][jn][0], acc[i][jn][1]);
            *reinterpret_cast<float2 *>(cst + (m + 8) * Cfg::EPI_PITCH + n) = make_float2(acc[i][jn][2], acc[i][jn][3]);
        }
    __syncthreads();

    // split-K reduction over distributed shared memory: every CTA of the cluster staged its partial tile;
    // rank r then sums ALL partials for its share of the rows (fixed order -> deterministic) and stores them.
    const int rows = ntile * p.P;
    int m_lo = 0, m_hi = rows;
    const float *part[8];
    part[0] = cst;
    if (p.ksplit > 1) {
        cg::cluster_group cluster = cg::this_cluster();
        cluster.sync();
        const int per = (rows + p.ksplit - 1) / p.ksplit;
        m_lo = min(rows, kr * per);
        m_hi = min(rows, m_lo + per);
#pragma unroll
        for (int r = 0; r < 8; ++r) part[r] = r < p.ksplit ? cluster.map_shared_rank(cst, r) : cst;
    }
    for (int q = tid + m_lo * (BN / 8); q < m_hi * (BN / 8); q += NTHREADS) {
        const int m = q / (BN / 8), nv = q - m * (BN / 8);
        const int n = n0 + nv * 8;
        if (n >= p.Cout) continue;
        const int tl = m / p.P, pp = m - tl * p.P;
        const int oy = pp / p.So, ox = pp - oy * p.So;
        const int t = tile0 + tl;
        int hh = oy, ww = ox, img = t;
        if (!p.dst_is_stack) {
            const int nn = p.idx_per_image ? t : t % p.N;
            hh += (p.offH + __ldg(p.idx + 2 * nn)) / p.stride;
            ww += (p.offW + __ldg(p.idx + 2 * nn + 1)) / p.stride;
            img = t / p.N;
        }
        if (hh < 0 || hh >= p.dH || ww < 0 || ww >= p.dW) continue;
        float v[8];
#pragma unroll
        for (int z = 0; z < 8; ++z) v[z] = 0.f;
        for (int r = 0; r < p.ksplit; ++r) {
            const float *cs = part[r] + m * Cfg::EPI_PITCH + nv * 8;
            const float4 c0 = *reinterpret_cast<const float4 *>(cs), c1 = *reinterpret_cast<const float4 *>(cs + 4);
            v[0] += c0.x; v[1] += c0.y; v[2] += c0.z; v[3] += c0.w; v[4] += c1.x; v[5] += c1.y; v[6] += c1.z; v[7] += c1.w;
        }
        if (p.bias) {
            const float4 b0 = __ldg(reinterpret_cast<const float4 *>(p.bias + n));
            const float4 b1 = __ldg(reinterpret_cast<const float4 *>(p.bias + n + 4));
            v[0] += b0.x; v[1] += b0.y; v[2] += b0.z; v[3] += b0.w; v[4] += b1.x; v[5] += b1.y; v[6] += b1.z; v[7] += b1.w;
        }
        const long long pixel = ((long long)img * p.dH + hh) * p.dW + ww;
        if (p.residual) {
            const uint4 r = __ldg(reinterpret_cast<const uint4 *>(reinterpret_cast<const T *>(p.residual) + pixel * p.rC + p.res_c0 + n));
            const T *re = reinterpret_cast<const T *>(&r);
#pragma unroll
            for (int z = 0; z < 8; ++z) v[z] += DT<T>::to_f(re[z]);
        }
        uint4 o;
        T *oe = reinterpret_cast<T *>(&o);
#pragma unroll
        for (int z = 0; z < 8; ++z) oe[z] = DT<T>::from_f(v[z]);
        if (p.dst) *reinterpret_cast<uint4 *>(reinterpret_cast<T *>(p.dst) + pixel * p.dC + p.dst_c0 + n) = o;
        for (int ax = 0; ax < p.n_aux; ++ax) {   // extra destinations: the consumer's pre-op applied by the producer
            const AuxDst &A = p.aux[ax];
            float w8[8];
#pragma unroll
            for (int z = 0; z < 8; ++z) w8[z] = v[z];
            if (A.scale) {
                const float4 s0 = __ldg(reinterpret_cast<const float4 *>(A.scale + n)), s1 = __ldg(reinterpret_cast<const float4 *>(A.scale + n + 4));
                w8[0] *= s0.x; w8[1] *= s0.y; w8[2] *= s0.z; w8[3] *= s0.w; w8[4] *= s1.x; w8[5] *= s1.y; w8[6] *= s1.z; w8[7] *= s1.w;
            }
            if (A.shift) {
                const float4 s0 = __ldg(reinterpret_cast<const float4 *>(A.shift + n)), s1 = __ldg(reinterpret_cast<const float4 *>(A.shift + n + 4));
                w8[0] += s0.x; w8[1] += s0.y; w8[2] += s0.z; w8[3] += s0.w; w8[4] += s1.x; w8[5] += s1.y; w8[6] += s1.z; w8[7] += s1.w;
            }
            uint4 oa;
            T *ae = reinterpret_cast<T *>(&oa);
#pragma unroll
            for (int z = 0; z < 8; ++z) ae[z] = DT<T>::from_f(activate<true>(A.act, w8[z]));
            *reinterpret_cast<uint4 *>(reinterpret_cast<T *>(A.ptr) + pixel * A.C + A.c0 + n) = oa;
        }
    }
    if (p.ksplit > 1) cg::this_cluster().sync();   // nobody leaves while a peer still reads its partial tile
}

template <typename T, int WM, int WN, int WARPS_M, int WARPS_N, int HALO_PIX, int NSTAGE, bool MOD>
static int launch_cfg(ConvParams &p, cudaStream_t st) {
    using Cfg = ConvCfg<T, WM, WN, WARPS_M, WARPS_N, HALO_PIX, NSTAGE>;
    auto kern = tile_conv_mma_kernel<T, WM, WN, WARPS_M, WARPS_N, HALO_PIX, NSTAGE, MOD>;
    static int attr_dev = -1;   // per instantiation; one process drives one GPU, but stay correct if not
    int dev = 0;
    cudaGetDevice(&dev);
    if (attr_dev != dev) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
        if (e != cudaSuccess) {
            set_error("sige_tile_conv: cannot reserve %d bytes of shared memory: %s", Cfg::SMEM_BYTES, cudaGetErrorString(e));
            return 2;
        }
        attr_dev = dev;
    }
    p.tpc = min(Cfg::BM / p.P, HALO_PIX / p.RS);
    if (p.tpc < 1) {
        set_error("sige_tile_conv: tile %dx%d (%d output pixels) does not fit the CTA tile (BM=%d, halo %d px)", p.R, p.S,
                  p.P, Cfg::BM, HALO_PIX);
        return 1;
    }
    const int J = ceil_div(p.Cin, KC) * p.taps;
    const long long base = (long long)ceil_div(p.NT, p.tpc) * ceil_div(p.Cout, Cfg::BN);
    if (p.ksplit <= 0) {
        // auto split-K: aim for ~2 CTAs per SM, keep >= 4 K steps per slice, cluster size <= 8 (portable limit)
        int ks = 1;
        while (ks < 8 && base * (ks * 2) <= 2 * sm_count() && J / (ks * 2) >= 4) ks *= 2;
        p.ksplit = ks;
    }
    if (p.ksplit > J) p.ksplit = 1;
    if (p.ksplit != 1 && p.ksplit != 2 && p.ksplit != 4 && p.ksplit != 8) {
        set_error("sige_tile_conv: ksplit must be 1, 2, 4 or 8 (got %d)", p.ksplit);
        return 1;
    }
    const dim3 grid(ceil_div(p.NT, p.tpc), ceil_div(p.Cout, Cfg::BN), p.ksplit);
    const cudaError_t e = launch_ex(kern, grid, dim3(Cfg::NTHREADS), Cfg::SMEM_BYTES, st, p.pdl != 0, dim3(1, 1, p.ksplit), p);
    if (e != cudaSuccess) {
        set_error("sige_tile_conv: launch failed (grid %d x %d x %d, %d threads, %d B smem): %s", grid.x, grid.y, grid.z,
                  Cfg::NTHREADS, Cfg::SMEM_BYTES, cudaGetErrorString(e));
        (void)cudaGetLastError();
        return 2;
    }
    return 0;
}

// CTA-count estimate used to pick a configuration: small grids want small CTA tiles.
static inline long long ctas_for(int NT, int P, int RS, int Cout, int BM, int BN, int halo_pix) {
    int tpc = min(BM / P, halo_pix / RS);
    if (tpc < 1) return -1;
    return (long long)ceil_div(NT, tpc) * ceil_div(Cout, BN);
}

template <typename T, bool MOD> static int launch_tile_conv(ConvParams &p, cudaStream_t st) {
    // L: 128x128 CTA tile, 8 warps, 5-stage weight ring; M: 64x64, 4 warps, 8 stages; S: 32x64, 4 warps, 8 stages.
    // Prefer the largest tile that still fills the machine; below that, the smallest tile plus split-K.
    const long long cL = ctas_for(p.NT, p.P, p.RS, p.Cout, 128, 128, 288);
    const long long cM = ctas_for(p.NT, p.P, p.RS, p.Cout, 64, 64, 144);
    const long long cS = ctas_for(p.NT, p.P, p.RS, p.Cout, 32, 64, 72);
    const int sms = sm_count();
    if (cL >= 2 * sms) return launch_cfg<T, 2, 8, 4, 2, 288, 5, MOD>(p, st);
    if (cM >= sms || cS < 0) {
        if (cM > 0) return launch_cfg<T, 2, 4, 2, 2, 144, 8, MOD>(p, st);
        return launch_cfg<T, 2, 8, 4, 2, 288, 5, MOD>(p, st);
    }
    return launch_cfg<T, 2, 2, 1, 4, 72, 8, MOD>(p, st);
}

bool tc5_supported(const sige_tile_conv_t *a, int pitch0);
int tc5_launch(const sige_tile_conv_t *a, int pitch0, cudaStream_t st);

// Argument checks and launch of sige_tile_conv; m != nullptr: sige_tile_conv_modulated, pitch0 > 0: sige_tile_conv_strided (whose
// own refusals come first).  pitch0 = elements per pixel of the single source (0: its channel count).
static int tile_conv(const sige_tile_conv_t *a, const sige_conv_modulation_t *m, int pitch0, sige_stream_t stream) {
    SIGE_REQUIRE(a != nullptr, "sige_tile_conv: null descriptor");
    SIGE_REQUIRE(a->dtype == SIGE_F16 || a->dtype == SIGE_BF16,
                 "sige_tile_conv: tensor-core path needs f16/bf16 (got dtype %d); use sige_tile_conv_generic", a->dtype);
    SIGE_REQUIRE(a->n_src == 1 || a->n_src == 2, "sige_tile_conv: n_src must be 1 or 2");
    SIGE_REQUIRE(a->B > 0 && a->N >= 0 && a->R > 0 && a->S > 0 && a->kH > 0 && a->kW > 0 && a->stride > 0,
                 "sige_tile_conv: bad geometry");
    SIGE_REQUIRE(a->R >= a->kH && a->S >= a->kW, "sige_tile_conv: tile smaller than the kernel");
    if (a->N == 0) return 0;
    if (m) {
        const int cin = a->Cin;
        SIGE_REQUIRE(m->gamma && m->beta, "sige_tile_conv_modulated: null gamma / beta");
        SIGE_REQUIRE(((uintptr_t)m->gamma & 15) == 0 && ((uintptr_t)m->beta & 15) == 0, "sige_tile_conv_modulated: gamma / beta not 16-byte aligned");
        SIGE_REQUIRE(m->gamma_C % 8 == 0 && m->gamma_c0 % 8 == 0 && m->gamma_c0 >= 0 && m->gamma_c0 + cin <= m->gamma_C,
                     "sige_tile_conv_modulated: gamma channel window [%d, %d) of %d channels (multiples of 8 within the buffer)", m->gamma_c0, m->gamma_c0 + cin, m->gamma_C);
        SIGE_REQUIRE(m->beta_C % 8 == 0 && m->beta_c0 % 8 == 0 && m->beta_c0 >= 0 && m->beta_c0 + cin <= m->beta_C,
                     "sige_tile_conv_modulated: beta channel window [%d, %d) of %d channels (multiples of 8 within the buffer)", m->beta_c0, m->beta_c0 + cin, m->beta_C);
    }
    int csum = 0;
    bool narrow = false;   // a source whose channel count is a multiple of 8 but not of 64: partial last K chunk
    for (int s = 0; s < a->n_src; ++s) {
        SIGE_REQUIRE(a->src[s].ptr != nullptr, "sige_tile_conv: source %d is null", s);
        SIGE_REQUIRE(a->src[s].C > 0 && a->src[s].C % 8 == 0, "sige_tile_conv: source %d has %d channels; the tensor-core path needs a multiple of 8", s, a->src[s].C);
        narrow = narrow || a->src[s].C % KC != 0;
        SIGE_REQUIRE(a->src[s].up == 0 || a->src[s].up == 1, "sige_tile_conv: bad upsample flag");
        SIGE_REQUIRE(((uintptr_t)a->src[s].ptr & 15) == 0, "sige_tile_conv: source %d is not 16-byte aligned", s);
        csum += a->src[s].C;
    }
    SIGE_REQUIRE(csum == a->Cin, "sige_tile_conv: source channels (%d) != Cin (%d)", csum, a->Cin);
    SIGE_REQUIRE(!narrow || a->n_src == 1, "sige_tile_conv: a source whose channel count is not a multiple of %d cannot be concatenated with another", KC);
    SIGE_REQUIRE(!narrow || a->n_src2 == 0, "sige_tile_conv: the fused shortcut needs a main source whose channel count is a multiple of %d (got Cin %d)", KC, a->Cin);
    SIGE_REQUIRE(a->Cout > 0 && a->Cout % 8 == 0, "sige_tile_conv: Cout (%d) must be a multiple of 8", a->Cout);
    SIGE_REQUIRE(a->w_packed && (a->dst || a->n_aux > 0), "sige_tile_conv: null weight/destination");
    SIGE_REQUIRE(a->src_is_stack || a->idx, "sige_tile_conv: index list missing");
    SIGE_REQUIRE(a->dst_is_stack || a->idx, "sige_tile_conv: index list missing");
    SIGE_REQUIRE(!(a->src_is_stack && a->n_src != 1), "sige_tile_conv: a stack source cannot be concatenated");
    SIGE_REQUIRE(a->H < 65536 && a->W < 65536, "sige_tile_conv: extent too large");
    if (a->dst) {
        SIGE_REQUIRE(a->dC % 8 == 0 && a->dst_c0 % 8 == 0 && ((uintptr_t)a->dst & 15) == 0, "sige_tile_conv: destination must be 16-byte aligned per pixel");
        SIGE_REQUIRE(a->dst_c0 + a->Cout <= a->dC, "sige_tile_conv: destination channel window out of range");
    }
    if (a->residual)
        SIGE_REQUIRE(a->rC % 8 == 0 && a->res_c0 % 8 == 0 && a->res_c0 + a->Cout <= a->rC && ((uintptr_t)a->residual & 15) == 0,
                     "sige_tile_conv: bad residual channel window");
    SIGE_REQUIRE(((uintptr_t)a->w_packed & 15) == 0, "sige_tile_conv: packed weights not 16-byte aligned");
    if (a->scale) SIGE_REQUIRE(((uintptr_t)a->scale & 15) == 0, "sige_tile_conv: scale not 16-byte aligned");
    if (a->shift) SIGE_REQUIRE(((uintptr_t)a->shift & 15) == 0, "sige_tile_conv: shift not 16-byte aligned");
    if (a->bias) SIGE_REQUIRE(((uintptr_t)a->bias & 15) == 0, "sige_tile_conv: bias not 16-byte aligned");
    SIGE_REQUIRE(a->affine_bstride == 0 || a->affine_bstride == a->Cin, "sige_tile_conv: affine_bstride must be 0 or Cin");
    SIGE_REQUIRE(a->act == SIGE_ACT_IDENTITY || a->act == SIGE_ACT_SWISH, "sige_tile_conv: unknown activation %d", a->act);
    SIGE_REQUIRE(a->ksplit >= 0 && a->ksplit <= 8, "sige_tile_conv: ksplit out of range");
    SIGE_REQUIRE(a->n_aux >= 0 && a->n_aux <= 2, "sige_tile_conv: n_aux must be 0, 1 or 2");
    for (int i = 0; i < a->n_aux; ++i) {
        const sige_conv_aux_t &x = a->aux[i];
        SIGE_REQUIRE(x.ptr && ((uintptr_t)x.ptr & 15) == 0 && x.C % 8 == 0 && x.c0 % 8 == 0 && x.c0 + a->Cout <= x.C, "sige_tile_conv: bad aux destination %d", i);
        SIGE_REQUIRE((!x.scale || ((uintptr_t)x.scale & 15) == 0) && (!x.shift || ((uintptr_t)x.shift & 15) == 0), "sige_tile_conv: aux %d affine not 16-byte aligned", i);
        SIGE_REQUIRE(x.act == SIGE_ACT_IDENTITY || x.act == SIGE_ACT_SWISH || x.act == SIGE_ACT_RELU, "sige_tile_conv: aux %d unknown activation", i);
    }

    SIGE_REQUIRE(!a->idx_per_image || (!a->src_is_stack && !a->dst_is_stack), "sige_tile_conv: per-image tile lists need full-tensor source and destination");
    SIGE_REQUIRE(a->n_src2 >= 0 && a->n_src2 <= 2, "sige_tile_conv: n_src2 must be 0, 1 or 2");
    if (a->n_src2 > 0) {
        int c2 = 0;
        for (int s2 = 0; s2 < a->n_src2; ++s2) {
            SIGE_REQUIRE(a->src2[s2].ptr && a->src2[s2].C > 0 && a->src2[s2].C % KC == 0 && ((uintptr_t)a->src2[s2].ptr & 15) == 0, "sige_tile_conv: bad shortcut source %d", s2);
            c2 += a->src2[s2].C;
        }
        SIGE_REQUIRE(c2 == a->Cin2 && a->w2_packed && ((uintptr_t)a->w2_packed & 15) == 0, "sige_tile_conv: shortcut channels/weights mismatch");
        SIGE_REQUIRE(!a->src_is_stack && !a->dst_is_stack, "sige_tile_conv: the fused shortcut needs full-tensor source and destination");
        SIGE_REQUIRE((a->flags & SIGE_CONV_TC5) && tc5_supported(a, 0), "sige_tile_conv: the fused shortcut is implemented by the wgmma kernel only (3x3 stride-1 on 6x6 tiles, SIGE_CONV_TC5)");
        SIGE_REQUIRE(a->sc_flags == nullptr || a->residual != nullptr, "sige_tile_conv: sc_flags given without the cached shortcut (residual)");
    }
    // Hopper-native path (wgmma + TMA, tile_conv_tc5.cu) when requested and the geometry fits
    if (!m && (a->flags & SIGE_CONV_TC5) && tc5_supported(a, pitch0)) return tc5_launch(a, pitch0, (cudaStream_t)stream);

    ConvParams p;
    p.seg[0] = ConvSeg{a->src[0].ptr, pitch0 > 0 ? pitch0 : a->src[0].C, a->src[0].up};
    p.seg[1] = a->n_src == 2 ? ConvSeg{a->src[1].ptr, a->src[1].C, a->src[1].up} : p.seg[0];
    p.C0 = a->src[0].C;
    p.src_is_stack = a->src_is_stack;
    p.H = a->src_is_stack ? a->R : a->H;
    p.W = a->src_is_stack ? a->S : a->W;
    p.idx = a->idx;
    p.N = a->N;
    p.NT = a->B * a->N;
    p.idx_per_image = a->idx_per_image ? 1 : 0;
    p.padded = ((a->flags & SIGE_CONV_PADDED) && a->B == 1 && a->idx && !a->src_is_stack && !a->dst_is_stack) ? 1 : 0;
    p.R = a->R; p.S = a->S; p.RS = a->R * a->S;
    p.scale = a->scale; p.shift = a->shift; p.affine_bstride = a->affine_bstride; p.act = a->act;
    p.w = a->w_packed; p.bias = a->bias;
    p.Cin = a->Cin; p.Cout = a->Cout; p.kH = a->kH; p.kW = a->kW; p.taps = a->kH * a->kW; p.stride = a->stride;
    p.Ro = (a->R - a->kH) / a->stride + 1;
    p.So = (a->S - a->kW) / a->stride + 1;
    p.P = p.Ro * p.So;
    p.dst = a->dst; p.dst_is_stack = a->dst_is_stack;
    p.dH = a->dst_is_stack ? p.Ro : a->dH;
    p.dW = a->dst_is_stack ? p.So : a->dW;
    p.dC = a->dC; p.dst_c0 = a->dst_c0;
    p.offH = a->offH; p.offW = a->offW;
    p.residual = a->residual; p.rC = a->rC; p.res_c0 = a->res_c0;
    p.n_aux = a->n_aux;
    for (int i = 0; i < a->n_aux; ++i) p.aux[i] = AuxDst{a->aux[i].ptr, a->aux[i].C, a->aux[i].c0, a->aux[i].scale, a->aux[i].shift, a->aux[i].act};
    p.tpc = 1;
    p.ksplit = a->ksplit;
    p.pdl = (a->flags & SIGE_CONV_PDL) ? 1 : 0;
    p.gamma = p.beta = nullptr;
    p.gC = p.g_c0 = p.bC = p.b_c0 = 0;
    p.slope = 1.f;
    if (m) {
        p.gamma = m->gamma; p.gC = m->gamma_C; p.g_c0 = m->gamma_c0;
        p.beta = m->beta; p.bC = m->beta_C; p.b_c0 = m->beta_c0;
        p.slope = m->negative_slope;
        if (a->dtype == SIGE_F16) return launch_tile_conv<__half, true>(p, (cudaStream_t)stream);
        return launch_tile_conv<__nv_bfloat16, true>(p, (cudaStream_t)stream);
    }
    if (a->dtype == SIGE_F16) return launch_tile_conv<__half, false>(p, (cudaStream_t)stream);
    return launch_tile_conv<__nv_bfloat16, false>(p, (cudaStream_t)stream);
}

}  // namespace sige

using namespace sige;

extern "C" int sige_tile_conv(const sige_tile_conv_t *a, sige_stream_t stream) { return tile_conv(a, nullptr, 0, stream); }

extern "C" int sige_tile_conv_strided(const sige_tile_conv_t *a, int src_pixel_stride, sige_stream_t stream) {
    SIGE_REQUIRE(a != nullptr, "sige_tile_conv_strided: null descriptor");
    SIGE_REQUIRE(a->n_src == 1, "sige_tile_conv_strided: one source segment (got n_src %d)", a->n_src);
    SIGE_REQUIRE(!a->src_is_stack, "sige_tile_conv_strided: the source must be a full tensor read through the tile list, not a stack");
    SIGE_REQUIRE(a->n_src2 == 0, "sige_tile_conv_strided: no fused shortcut");
    SIGE_REQUIRE(!a->idx_per_image, "sige_tile_conv_strided: per-image tile lists are not supported");
    SIGE_REQUIRE(src_pixel_stride >= a->src[0].C && src_pixel_stride % 8 == 0,
                 "sige_tile_conv_strided: pixel stride %d must be a multiple of 8 and at least the source's %d channels", src_pixel_stride, a->src[0].C);
    SIGE_REQUIRE(((uintptr_t)a->src[0].ptr & 15) == 0, "sige_tile_conv_strided: source is not 16-byte aligned");
    return tile_conv(a, nullptr, src_pixel_stride, stream);
}

extern "C" int sige_tile_conv_modulated_supported(int Cin, int Cout, int k, int stride, int dtype) {
    return (dtype == SIGE_F16 || dtype == SIGE_BF16) && Cin > 0 && Cin % 8 == 0 && Cout > 0 && Cout % 8 == 0 && k >= 1 && stride >= 1 ? 1 : 0;
}

extern "C" int sige_tile_conv_modulated(const sige_tile_conv_t *a, const sige_conv_modulation_t *m, sige_stream_t stream) {
    SIGE_REQUIRE(a != nullptr && m != nullptr, "sige_tile_conv_modulated: null descriptor");
    SIGE_REQUIRE(a->n_src == 1, "sige_tile_conv_modulated: one source segment (got n_src %d)", a->n_src);
    SIGE_REQUIRE(!a->src_is_stack, "sige_tile_conv_modulated: the source must be a full tensor read through the tile list, not a stack");
    SIGE_REQUIRE(a->act == SIGE_ACT_IDENTITY, "sige_tile_conv_modulated: act must be identity (negative_slope is the activation)");
    SIGE_REQUIRE(a->n_src2 == 0, "sige_tile_conv_modulated: no fused shortcut");
    SIGE_REQUIRE(!a->idx_per_image, "sige_tile_conv_modulated: per-image tile lists are not supported");
    SIGE_REQUIRE(isfinite(m->negative_slope), "sige_tile_conv_modulated: negative_slope must be finite");
    return tile_conv(a, m, 0, stream);
}

// conv1 -> conv2 of one residual block as one call (see include/sige_b200.h).
extern "C" int sige_resblock(const sige_tile_conv_t *conv1, const sige_tile_conv_t *conv2, sige_stream_t stream) {
    using namespace sige;
    SIGE_REQUIRE(conv1 && conv2, "sige_resblock: null descriptor");
    bool chained = false;       // conv2 must read what conv1 writes
    for (int s = 0; s < conv2->n_src; ++s) {
        if (conv1->dst && conv2->src[s].ptr == conv1->dst) chained = true;
        for (int a = 0; a < conv1->n_aux; ++a)
            if (conv2->src[s].ptr == conv1->aux[a].ptr) chained = true;
    }
    SIGE_REQUIRE(chained, "sige_resblock: conv2 does not gather from conv1's destination (or one of its aux views)");
    int rc = sige_tile_conv(conv1, stream);
    if (rc != 0) return rc;
    sige_tile_conv_t second = *conv2;
    second.flags |= SIGE_CONV_PDL;
    return sige_tile_conv(&second, stream);
}
