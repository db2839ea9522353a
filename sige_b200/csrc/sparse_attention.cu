// sparse_attention.cu — multi-head attention core of Stable Diffusion's transformer blocks for SPARSE queries:
//   out[bh, i, :] = softmax_j( scale * q[bh, i, :] . k[bh, j, :] ) v[bh, j, :]
// Replaces the reference's torch.bmm -> * scale -> softmax -> torch.bmm in
// stable-diffusion/ldm/modules/attention.py:81-93 (attn1: the queries are the tokens of the active tiles only, the keys /
// values all tokens of the scattered full tensor, sige_attention.py:79,153-160) and sige_attention.py:44-58 (attn2: the same
// sparse queries against the text keys / values cached by the dense pass), one launch instead of three plus the
// [Nq x Nk] logits round trip through HBM.
//
// Shape of the problem (SD v1, 64x64 latent, 15 % edit): B*heads = 16, Nq = 16 * active tiles (a few hundred .. ~1000),
// Nk = 4096 / 1024 / 256 / 64 (self) or 77 (text), head dim D = 40 / 80 / 160.  Flash-attention structure: a CTA owns 64
// queries of one (batch, head) — 16 per warp, fragments resident in registers — and streams keys / values in blocks of 64
// through a double-buffered cp.async ring; logits, running max / sum and the output accumulator never leave registers.
// Tensor cores: mma.sync.m16n8k16 (fp32 accumulate).  Head dims that are not a multiple of 16 (40) are zero-padded in
// shared memory only.
#include "common.cuh"

namespace sige {
namespace sattn {

constexpr int BM = 64;        // queries per CTA
constexpr int BNK = 64;       // keys per ring stage
constexpr int NTHREADS = 128;

__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;\n" : "=f"(y) : "f"(x));
    return y;
}

struct Params {
    const void *q, *k, *v;
    void *out;
    int heads, Nq, Nk;
    long long q_sb, q_sh, q_sn;      // element strides: batch, head, token (the head dim is contiguous)
    long long k_sb, k_sh, k_sn;
    long long v_sb, v_sh, v_sn;
    long long o_sb, o_sh, o_sn;
    float scale_log2e;               // softmax scale * log2(e)
};

template <int D> struct Lay {
    static constexpr int DP = (D + 15) / 16 * 16;       // head dim padded to the MMA K step
    static constexpr int PITCH = DP * 2 + 16;           // bytes; +16: the 8 rows of an ldmatrix 8x8 start 4 banks apart
    static constexpr int OFF_Q = 0;
    static constexpr int OFF_K = OFF_Q + BM * PITCH;               // [2][BNK] rows
    static constexpr int OFF_V = OFF_K + 2 * BNK * PITCH;          // [2][BNK] rows
    static constexpr int TOTAL = OFF_V + 2 * BNK * PITCH;
    static_assert(TOTAL <= 232448, "shared memory");
};

// grid (ceil(Nq / 64), B * heads).  Warp w owns query rows 16w .. 16w+15 of the CTA's 64.
template <typename T, int D>
__global__ void __launch_bounds__(NTHREADS, 2) sparse_attention_kernel(const Params p) {
    using L = Lay<D>;
    constexpr int DP = L::DP, PITCH = L::PITCH;
    constexpr int CH = D / 8;                 // real 16-byte chunks per row
    constexpr int CHP = DP / 8;               // chunks per padded row
    constexpr int KS = DP / 16;               // k-steps of Q K^T
    constexpr int NT = DP / 8;                // n-tiles of P V (output channels / 8)
    extern __shared__ __align__(128) unsigned char smem[];
    const uint32_t sb = smem_u32(smem);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q0 = blockIdx.x * BM;
    const int bh = blockIdx.y, b = bh / p.heads, h = bh - b * p.heads;
    const T *qp = reinterpret_cast<const T *>(p.q) + b * p.q_sb + h * p.q_sh;
    const T *kp = reinterpret_cast<const T *>(p.k) + b * p.k_sb + h * p.k_sh;
    const T *vp = reinterpret_cast<const T *>(p.v) + b * p.v_sb + h * p.v_sh;

    // padding columns D .. DP-1 of every row: zero once (the ring only ever rewrites the real chunks)
    if (CHP > CH) {
        for (int r = tid; r < BM + 4 * BNK; r += NTHREADS)
#pragma unroll
            for (int c = CH; c < CHP; ++c) *reinterpret_cast<uint4 *>(smem + r * PITCH + c * 16) = make_uint4(0, 0, 0, 0);
    }
    auto load_q = [&]() {
        for (int i = tid; i < BM * CH; i += NTHREADS) {
            const int r = i / CH, c = i - r * CH;
            const bool ok = q0 + r < p.Nq;
            cp_async16_zfill(sb + L::OFF_Q + r * PITCH + c * 16, qp + (ok ? (long long)(q0 + r) * p.q_sn + c * 8 : 0), ok);
        }
    };
    auto load_kv = [&](int t, int stage) {
        const int k0 = t * BNK;
        for (int i = tid; i < BNK * CH; i += NTHREADS) {
            const int r = i / CH, c = i - r * CH;
            const bool ok = k0 + r < p.Nk;           // rows past the last key: zero fill (their logits are masked, 0 * V must stay finite)
            const long long tok = ok ? (long long)(k0 + r) : 0;
            cp_async16_zfill(sb + L::OFF_K + (stage * BNK + r) * PITCH + c * 16, kp + tok * p.k_sn + c * 8, ok);
            cp_async16_zfill(sb + L::OFF_V + (stage * BNK + r) * PITCH + c * 16, vp + tok * p.v_sn + c * 8, ok);
        }
    };
    const int ntiles = (p.Nk + BNK - 1) / BNK;
    load_q();
    load_kv(0, 0);
    cp_async_commit();

    const int g = lane >> 2, tq = lane & 3;
    uint32_t qf[KS][4];
    float o[NT][4];
#pragma unroll
    for (int i = 0; i < NT; ++i)
#pragma unroll
        for (int z = 0; z < 4; ++z) o[i][z] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};

    for (int t = 0; t < ntiles; ++t) {
        const int stage = t & 1;
        if (t + 1 < ntiles) load_kv(t + 1, stage ^ 1);
        cp_async_commit();
        cp_async_wait<1>();                     // tile t (and, for t == 0, the queries) has landed
        __syncthreads();
        if (t == 0) {
            const int arow = warp * 16 + (lane & 15), ahalf = lane >> 4;
            const uint32_t a_base = sb + L::OFF_Q + arow * PITCH + ahalf * 16;
#pragma unroll
            for (int kk = 0; kk < KS; ++kk) ldmatrix_x4(a_base + kk * 32, qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3]);
        }
        // ---- S = Q K^T: 16 queries x 64 keys per warp
        float s[BNK / 8][4];
#pragma unroll
        for (int i = 0; i < BNK / 8; ++i)
#pragma unroll
            for (int z = 0; z < 4; ++z) s[i][z] = 0.f;
        {
            const int brow = ((lane >> 4) << 3) + (lane & 7), bhalf = (lane >> 3) & 1;
            const uint32_t b_base = sb + L::OFF_K + (stage * BNK + brow) * PITCH + bhalf * 16;
#pragma unroll
            for (int kk = 0; kk < KS; ++kk)
#pragma unroll
                for (int n2 = 0; n2 < BNK / 16; ++n2) {
                    uint32_t b0, b1, b2, b3;
                    ldmatrix_x4(b_base + n2 * 16 * PITCH + kk * 32, b0, b1, b2, b3);
                    mma_m16n8k16<T>(s[2 * n2], qf[kk], b0, b1);
                    mma_m16n8k16<T>(s[2 * n2 + 1], qf[kk], b2, b3);
                }
        }
        // ---- keys past Nk (last tile only): -inf
        const int k0 = t * BNK;
        if (k0 + BNK > p.Nk) {
#pragma unroll
            for (int i = 0; i < BNK / 8; ++i) {
                const int key = k0 + i * 8 + 2 * tq;
                if (key >= p.Nk) { s[i][0] = -INFINITY; s[i][2] = -INFINITY; }
                if (key + 1 >= p.Nk) { s[i][1] = -INFINITY; s[i][3] = -INFINITY; }
            }
        }
        // ---- online softmax: rows g (h2 = 0) and g + 8 (h2 = 1) of this warp's 16 queries
        uint32_t pf[BNK / 16][4];
#pragma unroll
        for (int h2 = 0; h2 < 2; ++h2) {
            float mx = -INFINITY;
#pragma unroll
            for (int i = 0; i < BNK / 8; ++i) mx = fmaxf(mx, fmaxf(s[i][2 * h2], s[i][2 * h2 + 1]));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float m_new = fmaxf(m[h2], mx);                    // finite: every tile holds at least one real key
            const float corr = fast_exp2((m[h2] - m_new) * p.scale_log2e);
            const float mb = m_new * p.scale_log2e;
            m[h2] = m_new;
            float sum = 0.f;
#pragma unroll
            for (int i = 0; i < BNK / 8; ++i) {
                const float e0 = fast_exp2(fmaf(s[i][2 * h2], p.scale_log2e, -mb)), e1 = fast_exp2(fmaf(s[i][2 * h2 + 1], p.scale_log2e, -mb));
                sum += e0 + e1;
                pf[i >> 1][(i & 1) * 2 + h2] = pack2<T>(e0, e1);
            }
            l[h2] = fmaf(l[h2], corr, sum);
#pragma unroll
            for (int i = 0; i < NT; ++i) { o[i][2 * h2] *= corr; o[i][2 * h2 + 1] *= corr; }
        }
        // ---- O += P V
        {
            const int vkey = ((lane >> 3) & 1) * 8 + (lane & 7), vsel = lane >> 4;
            const uint32_t v_base = sb + L::OFF_V + (stage * BNK + vkey) * PITCH + vsel * 16;
#pragma unroll
            for (int kk = 0; kk < BNK / 16; ++kk)
#pragma unroll
                for (int n2 = 0; n2 < NT / 2; ++n2) {
                    uint32_t b0, b1, b2, b3;
                    ldmatrix_x4_trans(v_base + kk * 16 * PITCH + n2 * 32, b0, b1, b2, b3);
                    mma_m16n8k16<T>(o[2 * n2], pf[kk], b0, b1);
                    mma_m16n8k16<T>(o[2 * n2 + 1], pf[kk], b2, b3);
                }
        }
        __syncthreads();                  // this stage is rewritten by the prefetch of the next iteration
    }
    // ---- out = O / l
    T *op = reinterpret_cast<T *>(p.out) + b * p.o_sb + h * p.o_sh;
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {
        float sum = l[h2];
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);
        const float inv = 1.f / sum;
        const int row = q0 + warp * 16 + g + 8 * h2;
        if (row < p.Nq) {
#pragma unroll
            for (int i = 0; i < NT; ++i) {
                const int d = i * 8 + 2 * tq;
                if (d < D) *reinterpret_cast<uint32_t *>(op + (long long)row * p.o_sn + d) = pack2<T>(o[i][2 * h2] * inv, o[i][2 * h2 + 1] * inv);
            }
        }
    }
}

template <typename T, int D> static int launch(const Params &p, int BH, cudaStream_t stream) {
    using L = Lay<D>;
    static int attr_dev = -1;       // the opt-in is per device (and per kernel instantiation)
    int dev = 0;
    cudaGetDevice(&dev);
    if (attr_dev != dev) {
        if (cudaFuncSetAttribute(sparse_attention_kernel<T, D>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL) != cudaSuccess) {
            set_error("sige_sparse_attention: cannot reserve %d bytes of shared memory", L::TOTAL);
            (void)cudaGetLastError();
            return 2;
        }
        attr_dev = dev;
    }
    const dim3 grid(ceil_div(p.Nq, BM), BH);
    sparse_attention_kernel<T, D><<<grid, NTHREADS, L::TOTAL, stream>>>(p);
    return check_launch("sige_sparse_attention");
}

template <typename T> static int dispatch(const Params &p, int BH, int D, cudaStream_t stream) {
    switch (D) {
        case 32: return launch<T, 32>(p, BH, stream);
        case 40: return launch<T, 40>(p, BH, stream);
        case 64: return launch<T, 64>(p, BH, stream);
        case 80: return launch<T, 80>(p, BH, stream);
        case 128: return launch<T, 128>(p, BH, stream);
        case 160: return launch<T, 160>(p, BH, stream);
    }
    set_error("sige_sparse_attention: head dim %d is not one of 32, 40, 64, 80, 128, 160", D);
    return 1;
}

}  // namespace sattn
}  // namespace sige

extern "C" int sige_sparse_attention_supported(int D, int dtype) {
    return ((D == 32 || D == 40 || D == 64 || D == 80 || D == 128 || D == 160) && (dtype == SIGE_F16 || dtype == SIGE_BF16)) ? 1 : 0;
}

extern "C" int sige_sparse_attention(const sige_sparse_attention_t *a, sige_stream_t stream_) {
    using namespace sige;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    SIGE_REQUIRE(a, "sige_sparse_attention: null descriptor");
    SIGE_REQUIRE(a->B >= 0 && a->heads >= 1 && a->Nq >= 0 && a->Nk >= 1, "sige_sparse_attention: B = %d, heads = %d, Nq = %d, Nk = %d", a->B, a->heads,
                 a->Nq, a->Nk);
    SIGE_REQUIRE(sige_sparse_attention_supported(a->D, a->dtype), "sige_sparse_attention: unsupported head dim %d (32, 40, 64, 80, 128, 160) / dtype %d (f16, bf16)",
                 a->D, a->dtype);
    // scale = 0 makes the last-block mask -inf * 0 = NaN; scale < 0 takes the running maximum at the wrong end
    SIGE_REQUIRE(a->scale > 0.f && isfinite(a->scale), "sige_sparse_attention: scale = %g must be positive and finite", (double)a->scale);
    if (a->B == 0 || a->Nq == 0) return 0;          // no active tile: nothing to do
    SIGE_REQUIRE(a->q && a->k && a->v && a->out, "sige_sparse_attention: null buffer");
    const long long strides[12] = {a->q_stride[0], a->q_stride[1], a->q_stride[2], a->k_stride[0], a->k_stride[1], a->k_stride[2],
                                   a->v_stride[0], a->v_stride[1], a->v_stride[2], a->out_stride[0], a->out_stride[1], a->out_stride[2]};
    for (int i = 0; i < 12; ++i) SIGE_REQUIRE(strides[i] % 8 == 0, "sige_sparse_attention: strides must be multiples of 8 elements (16-byte rows)");
    SIGE_REQUIRE(((uintptr_t)a->q | (uintptr_t)a->k | (uintptr_t)a->v | (uintptr_t)a->out) % 16 == 0, "sige_sparse_attention: buffers must be 16-byte aligned");
    SIGE_REQUIRE((long long)a->B * a->heads <= 65535, "sige_sparse_attention: B * heads = %lld exceeds the grid limit", (long long)a->B * a->heads);
    sattn::Params p;
    p.q = a->q; p.k = a->k; p.v = a->v; p.out = a->out;
    p.heads = a->heads; p.Nq = a->Nq; p.Nk = a->Nk;
    p.q_sb = a->q_stride[0]; p.q_sh = a->q_stride[1]; p.q_sn = a->q_stride[2];
    p.k_sb = a->k_stride[0]; p.k_sh = a->k_stride[1]; p.k_sn = a->k_stride[2];
    p.v_sb = a->v_stride[0]; p.v_sh = a->v_stride[1]; p.v_sn = a->v_stride[2];
    p.o_sb = a->out_stride[0]; p.o_sh = a->out_stride[1]; p.o_sn = a->out_stride[2];
    p.scale_log2e = a->scale * 1.4426950408889634f;
    const int BH = a->B * a->heads;
    return a->dtype == SIGE_F16 ? sattn::dispatch<__half>(p, BH, a->D, stream) : sattn::dispatch<__nv_bfloat16>(p, BH, a->D, stream);
}
