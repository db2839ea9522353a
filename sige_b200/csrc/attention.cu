// attention.cu — single-head dense attention core of the DDPM AttnBlock on NHWC tokens, one launch.
//
// Replaces the reference's torch ops in diffusion/models/ddpm_arch/sige_fused_unet.py:185-199 (q·k^T · c^-0.5 → softmax →
// ·v) for the DENSE attention blocks (16x16 and 8x8 resolution: the reference never runs these tile-sparse).  The
// tokens live in the NHWC qkv buffer the fused 1x1 conv just produced: row n = pixel n, [q | k | v] of C channels
// each, q already scaled by c^-0.5 (folded into the conv's weights by the engine).
//
// Latency, not throughput, is what matters (134 MFLOP on the step's critical path): see the kernel comment for the
// cluster work split.
#include <cooperative_groups.h>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace sige {
namespace attn {

constexpr int QB = 32;        // queries per CTA
constexpr int KPC = 64;       // keys (and values) per CTA
constexpr int NTHREADS = 256;

// one contiguous row, global -> shared, completion counted in bytes on an mbarrier (TMA bulk copy, no tensor map)
__device__ __forceinline__ void bulk_row(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}

// shared-memory layout (bytes).  Rows are padded by 16 bytes: the 8 rows of an ldmatrix 8x8 then start 4 banks apart.
template <int C, int KS> struct Lay {
    static constexpr int N = KS * KPC;                     // tokens
    static constexpr int CO = C / KS;                      // output channels owned by one CTA of the cluster
    static constexpr int QK_PITCH = C * 2 + 16;
    static constexpr int V_PITCH = CO * 2 + 16;
    static constexpr int P_PITCH = N * 2 + 16;
    static constexpr int OFF_Q = 0;                                  // [QB][C]      this CTA's queries
    static constexpr int OFF_K = OFF_Q + QB * QK_PITCH;              // [KPC][C]     its 64 keys
    static constexpr int OFF_V = OFF_K + KPC * QK_PITCH;             // [N][CO]      ALL values, its channel slice
    static constexpr int OFF_P = OFF_V + N * V_PITCH;                // [QB][N]      softmax numerators of the whole cluster
    static constexpr int OFF_RED = OFF_P + QB * P_PITCH;             // [4][QB] floats, max then sum
    static constexpr int OFF_M = OFF_RED + 4 * QB * 4;               // [QB] floats
    static constexpr int OFF_STAT = OFF_M + QB * 4;                  // [KS][QB][2] floats: (m, l) of every key slice
    static constexpr int OFF_BAR = OFF_STAT + KS * QB * 2 * 4;       // 2 mbarriers
    static constexpr int TOTAL = OFF_BAR + 16;
    static_assert(TOTAL <= 232448, "shared memory");
    static_assert(CO % 64 == 0, "each of the four warp columns owns a multiple of 16 channels");
};

struct Params {
    const void *qkv;   // [B][N][3C]
    void *out;         // [B][N][C]
    int pdl;
};

// Work split: grid (N/32 query blocks, KS, B), the KS CTAs of a query block form a cluster.  CTA kr computes the
// logits of its 64 keys, S = Q K_kr^T, the local softmax numerators p = exp(S - m_kr) with statistics (m_kr, l_kr),
// and WRITES p (16-bit) and the statistics into every CTA of the cluster (distributed shared memory, 4 KB per peer).
// After one cluster barrier every CTA holds the numerators for all N keys and multiplies them with ITS channel slice
// of V (all N values x C/KS channels), re-weighting key slice r by exp(m_r - M): out = sum_r w_r (P_r V_r) / sum_r w_r l_r.
template <typename T, int C, int KS>
__global__ void __launch_bounds__(NTHREADS, 1) attention_kernel(const Params p) {
    using L = Lay<C, KS>;
    constexpr int N = L::N, CO = L::CO;
    constexpr int CQ = CO / 4;            // output channels per warp column
    constexpr int NT2 = CQ / 8;           // n-tiles per warp in P·V
    extern __shared__ __align__(128) unsigned char smem[];
    const uint32_t sb = smem_u32(smem);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q0 = blockIdx.x * QB, kr = blockIdx.y, b = blockIdx.z;
    const T *base = reinterpret_cast<const T *>(p.qkv) + (long long)b * N * 3 * C;
    float *s_red = reinterpret_cast<float *>(smem + L::OFF_RED);
    float *s_m = reinterpret_cast<float *>(smem + L::OFF_M);
    float *s_stat = reinterpret_cast<float *>(smem + L::OFF_STAT);
    const uint32_t bar_qk = sb + L::OFF_BAR, bar_v = bar_qk + 8;

    if (tid == 0) {
        mbar_init(bar_qk, 1);
        mbar_init(bar_v, 1);
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();
    if (KS > 1) cg::this_cluster().barrier_arrive();     // "this CTA is running": matched by barrier_wait() before the first remote store
    if (p.pdl) {
        pdl_release();
        pdl_acquire();     // the qkv convolution has completed
    }
    if (tid == 0) {
        mbar_expect_tx(bar_qk, (QB + KPC) * C * 2);
        mbar_expect_tx(bar_v, N * CO * 2);
    }
    __syncthreads();
    for (int r = tid; r < QB + KPC + N; r += NTHREADS) {
        if (r < QB) bulk_row(sb + L::OFF_Q + r * L::QK_PITCH, base + (long long)(q0 + r) * 3 * C, C * 2, bar_qk);
        else if (r < QB + KPC) bulk_row(sb + L::OFF_K + (r - QB) * L::QK_PITCH, base + (long long)(kr * KPC + r - QB) * 3 * C + C, C * 2, bar_qk);
        else bulk_row(sb + L::OFF_V + (r - QB - KPC) * L::V_PITCH, base + (long long)(r - QB - KPC) * 3 * C + 2 * C + kr * CO, CO * 2, bar_v);
    }

    // ---- S = Q K^T: warp (mi, kq) owns 16 queries x 16 of this CTA's 64 keys
    const int mi = warp & 1, kq = warp >> 1;
    float sacc[2][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int z = 0; z < 4; ++z) sacc[i][z] = 0.f;
    mbar_wait(bar_qk, 0);
    {
        const int arow = mi * 16 + (lane & 15), ahalf = lane >> 4;
        const int brow = kq * 16 + ((lane >> 4) << 3) + (lane & 7), bhalf = (lane >> 3) & 1;
        const uint32_t a_base = sb + L::OFF_Q + arow * L::QK_PITCH + ahalf * 16, b_base = sb + L::OFF_K + brow * L::QK_PITCH + bhalf * 16;
#pragma unroll 8
        for (int kk = 0; kk < C / 16; ++kk) {
            uint32_t a[4], b0, b1, b2, b3;
            ldmatrix_x4(a_base + kk * 32, a[0], a[1], a[2], a[3]);
            ldmatrix_x4(b_base + kk * 32, b0, b1, b2, b3);
            mma_m16n8k16<T>(sacc[0], a, b0, b1);
            mma_m16n8k16<T>(sacc[1], a, b2, b3);
        }
    }
    // ---- local softmax numerators: rows g and g+8 of this warp's 16 queries, columns 2t,2t+1 of two key tiles
    const int g = lane >> 2, tq = lane & 3;
    float mx[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float m = fmaxf(fmaxf(sacc[0][2 * h], sacc[0][2 * h + 1]), fmaxf(sacc[1][2 * h], sacc[1][2 * h + 1]));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
        if (tq == 0) s_red[kq * QB + mi * 16 + g + 8 * h] = m;
    }
    __syncthreads();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int r = mi * 16 + g + 8 * h;
        mx[h] = fmaxf(fmaxf(s_red[r], s_red[QB + r]), fmaxf(s_red[2 * QB + r], s_red[3 * QB + r]));
        if (kq == 0 && tq == 0) s_m[r] = mx[h];
    }
    __syncthreads();                                   // s_red is reused for the sums
    cg::cluster_group cluster = cg::this_cluster();
    if (KS > 1) cluster.barrier_wait();                // every peer is running: remote stores are legal
    {
        unsigned char *sp = smem + L::OFF_P;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = mi * 16 + g + 8 * h;
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const float e0 = __expf(sacc[i][2 * h] - mx[h]), e1 = __expf(sacc[i][2 * h + 1] - mx[h]);
                const uint32_t pk = pack2<T>(e0, e1);
                // the row sum is taken over the ROUNDED numerators, the values P·V actually uses
                const T *pe = reinterpret_cast<const T *>(&pk);
                s += DT<T>::to_f(pe[0]) + DT<T>::to_f(pe[1]);
                const int col = kr * KPC + kq * 16 + i * 8 + 2 * tq;        // key index within the N keys
                uint32_t *dst = reinterpret_cast<uint32_t *>(sp + r * L::P_PITCH + col * 2);
#pragma unroll
                for (int rk = 0; rk < KS; ++rk) *(rk == kr ? dst : cluster.map_shared_rank(dst, rk)) = pk;
            }
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            if (tq == 0) s_red[kq * QB + r] = s;
        }
    }
    __syncthreads();
    if (tid < QB) {                                    // (m, l) of this key slice, to every CTA of the cluster
        const float2 ml = make_float2(s_m[tid], s_red[tid] + s_red[QB + tid] + s_red[2 * QB + tid] + s_red[3 * QB + tid]);
        float2 *st = reinterpret_cast<float2 *>(s_stat) + kr * QB + tid;
#pragma unroll
        for (int rk = 0; rk < KS; ++rk) *(rk == kr ? st : cluster.map_shared_rank(st, rk)) = ml;
    }
    if (KS > 1) cluster.sync(); else __syncthreads();  // all numerators and statistics have landed everywhere

    // ---- out[:, kr*CO ...] = sum_r w_r (P_r V_r) / L: warp (mi, cq) owns 16 queries x CO/4 channels
    const int cq = warp >> 1;
    float wgt[KS][2], inv[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int r = mi * 16 + g + 8 * h;
        float M = -INFINITY, Lsum = 0.f;
#pragma unroll
        for (int rk = 0; rk < KS; ++rk) M = fmaxf(M, s_stat[(rk * QB + r) * 2]);
#pragma unroll
        for (int rk = 0; rk < KS; ++rk) {
            wgt[rk][h] = __expf(s_stat[(rk * QB + r) * 2] - M);
            Lsum += wgt[rk][h] * s_stat[(rk * QB + r) * 2 + 1];
        }
        inv[h] = 1.f / Lsum;
    }
    float oacc[NT2][4];
#pragma unroll
    for (int i = 0; i < NT2; ++i)
#pragma unroll
        for (int z = 0; z < 4; ++z) oacc[i][z] = 0.f;
    mbar_wait(bar_v, 0);
    {
        const int arow = mi * 16 + (lane & 15), ahalf = lane >> 4;
        const uint32_t a_base = sb + L::OFF_P + arow * L::P_PITCH + ahalf * 16;
        const int vkey = ((lane >> 3) & 1) * 8 + (lane & 7), vsel = lane >> 4;   // matrix id: bit0 = key half, bit1 = n-tile of the pair
        const uint32_t v_base = sb + L::OFF_V + vkey * L::V_PITCH + (cq * CQ + vsel * 8) * 2;
#pragma unroll
        for (int rk = 0; rk < KS; ++rk) {
            float t[NT2][4];
#pragma unroll
            for (int i = 0; i < NT2; ++i)
#pragma unroll
                for (int z = 0; z < 4; ++z) t[i][z] = 0.f;
#pragma unroll
            for (int k4 = 0; k4 < KPC / 16; ++k4) {
                const int kk = rk * (KPC / 16) + k4;                  // 16-key step
                uint32_t a[4];
                ldmatrix_x4(a_base + kk * 32, a[0], a[1], a[2], a[3]);
#pragma unroll
                for (int n2 = 0; n2 < NT2 / 2; ++n2) {
                    uint32_t b0, b1, b2, b3;
                    ldmatrix_x4_trans(v_base + kk * 16 * L::V_PITCH + n2 * 32, b0, b1, b2, b3);
                    mma_m16n8k16<T>(t[2 * n2], a, b0, b1);
                    mma_m16n8k16<T>(t[2 * n2 + 1], a, b2, b3);
                }
            }
#pragma unroll
            for (int i = 0; i < NT2; ++i) {
                oacc[i][0] = fmaf(wgt[rk][0], t[i][0], oacc[i][0]);
                oacc[i][1] = fmaf(wgt[rk][0], t[i][1], oacc[i][1]);
                oacc[i][2] = fmaf(wgt[rk][1], t[i][2], oacc[i][2]);
                oacc[i][3] = fmaf(wgt[rk][1], t[i][3], oacc[i][3]);
            }
        }
    }
    T *out = reinterpret_cast<T *>(p.out) + (long long)b * N * C;
#pragma unroll
    for (int i = 0; i < NT2; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = mi * 16 + g + 8 * h;
            const int ch = kr * CO + cq * CQ + i * 8 + 2 * tq;
            *reinterpret_cast<uint32_t *>(out + (long long)(q0 + r) * C + ch) = pack2<T>(oacc[i][2 * h] * inv[h], oacc[i][2 * h + 1] * inv[h]);
        }
}

template <typename T, int C, int KS> static int launch(const Params &p, int B, cudaStream_t stream) {
    using L = Lay<C, KS>;
    static int attr_dev = -1;       // the opt-in is per device (and per kernel instantiation)
    int dev = 0;
    cudaGetDevice(&dev);
    if (attr_dev != dev) {
        if (cudaFuncSetAttribute(attention_kernel<T, C, KS>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL) != cudaSuccess) {
            set_error("sige_attention_tokens: cannot reserve %d bytes of shared memory", L::TOTAL);
            (void)cudaGetLastError();
            return 2;
        }
        attr_dev = dev;
    }
    const cudaError_t e = launch_ex(attention_kernel<T, C, KS>, dim3(L::N / QB, KS, B), dim3(NTHREADS), L::TOTAL, stream, p.pdl != 0,
                                    dim3(1, KS, 1), p);
    if (e != cudaSuccess) {
        set_error("sige_attention_tokens: launch failed: %s", cudaGetErrorString(e));
        (void)cudaGetLastError();
        return 2;
    }
    return 0;
}

template <typename T, int C> static int dispatch_ks(const Params &p, int B, int ks, cudaStream_t stream) {
    switch (ks) {
        case 1: return launch<T, C, 1>(p, B, stream);
        case 2: return launch<T, C, 2>(p, B, stream);
        case 4: return launch<T, C, 4>(p, B, stream);
    }
    set_error("sige_attention_tokens: %d tokens not supported", ks * KPC);
    return 1;
}

template <typename T> static int dispatch_c(const Params &p, int B, int C, int ks, cudaStream_t stream) {
    switch (C) {
        case 256: return dispatch_ks<T, 256>(p, B, ks, stream);
        case 512: return dispatch_ks<T, 512>(p, B, ks, stream);
    }
    set_error("sige_attention_tokens: C = %d is not one of 256, 512", C);
    return 1;
}

}  // namespace attn
}  // namespace sige

extern "C" int sige_attention_tokens_supported(int N, int C, int dtype) {
    const int ks = N / sige::attn::KPC;
    return (N > 0 && N % sige::attn::KPC == 0 && (ks == 1 || ks == 2 || ks == 4) && (C == 256 || C == 512) &&
            (dtype == SIGE_F16 || dtype == SIGE_BF16)) ? 1 : 0;
}

extern "C" int sige_attention_tokens(const void *qkv, void *out, int B, int N, int C, int dtype, int flags, sige_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    using namespace sige;
    SIGE_REQUIRE(qkv && out, "sige_attention_tokens: null buffer");
    SIGE_REQUIRE(B >= 1, "sige_attention_tokens: B = %d", B);
    SIGE_REQUIRE(sige_attention_tokens_supported(N, C, dtype),
                 "sige_attention_tokens: unsupported shape N = %d (64, 128 or 256 tokens), C = %d (256, 512), dtype %d (f16, bf16)", N, C, dtype);
    attn::Params p;
    p.qkv = qkv;
    p.out = out;
    p.pdl = (flags & SIGE_CONV_PDL) ? 1 : 0;
    const int ks = N / attn::KPC;
    return dtype == SIGE_F16 ? attn::dispatch_c<__half>(p, B, C, ks, stream) : attn::dispatch_c<__nv_bfloat16>(p, B, C, ks, stream);
}
