// separable_conv.cu — the separable convolutions of GAN Compression's sub-mobile SPADE (gamma AND beta of one SPADE layer) on
// the active tiles, one launch:
//   out_b = pw_b( dw'_b(x) ) + bias_b,   b in {gamma, beta}
// Replaces, per branch, the three calls of reference gaugan/models/mobile_modules.py:108-112 in sparse mode (depthwise 3x3
// SIGEConv2d with groups = Cin, `x * scale + shift` with the instance-norm statistics of the dense pass, 1x1 SIGEConv2d) and the
// Scatter / ScatterGather that follows them (gaugan/models/sige_normalization.py:157-165): the outputs are pasted in place into
// the persistent destination.  The instance-norm affine is folded into the depthwise weights on the host
// (w' = scale*w, b' = scale*b + shift).
//
// CTA = 8 tiles (6x6 halo -> 4x4 outputs: 128 GEMM rows) x one block of 64 output channels of one branch (gridDim.z).
//   gather     cp.async of 16-channel halo chunks into a 3-stage ring; the source is a channel window [c0, c0 + Cin) of an NHWC
//              buffer read through the origin list (zero outside the image; SIGE_TILE_NONE tiles read zeros and write nothing)
//              or of a tile stack — torch.split slices of mlp_shared's output are read in place;
//   depthwise  CUDA cores, fp32, a thread per (output pixel, 8-channel vector); rounded once to the storage type into the A
//              operand [128][Cin] in shared memory;
//   pointwise  mma.sync.m16n8k16 + ldmatrix from shared memory, fp32 accumulation; the weight block [64][Cin] is loaded before the
//              dependency wait (it does not depend on the previous kernel);
//   epilogue   + bias, rounded, staged in shared memory, written as 16-byte channel vectors into the destination (NHWC buffer
//              with its own channel count / offset, or a stack); rows of SIGE_TILE_NONE tiles are skipped for either kind.
// The depthwise is recomputed per output-channel block: 9 FMAs per element against Cout / 64 * 128 for the GEMM.
#include "common.cuh"

namespace sige {
namespace sep {

constexpr int TILES = 8;
constexpr int M = TILES * 16;          // GEMM rows (output pixels) per CTA
constexpr int BN = 64;                 // output channels per CTA
constexpr int KC = 16;                 // channels per halo chunk
constexpr int HPIX = 36;               // 6 x 6 halo pixels
constexpr int STAGES = 3;
constexpr int NTHREADS = 256;
constexpr int CHUNK_ELEMS = TILES * HPIX * KC;
constexpr int RING_BYTES = STAGES * CHUNK_ELEMS * 2;
constexpr int UNITS = TILES * HPIX * (KC / 8);           // 16-byte cp.async units per chunk
constexpr int UPT = (UNITS + NTHREADS - 1) / NTHREADS;
constexpr int STG_PITCH = BN + 8;                        // epilogue staging row (elements)
static_assert(M * STG_PITCH * 2 <= RING_BYTES, "epilogue staging overlays the halo ring");
constexpr int MAX_CIN = 256, MAX_COUT = 1024;

struct Params {
    const void *src;
    int src_is_stack, sC, sc0;
    int B, H, W;
    const int32_t *idx;
    int N, total;                      // tiles per image, B * N
    int Cin, Cout;
    const float *dw_w[2], *dw_b[2];    // fp32 [Cin][9], [Cin] (affine folded)
    const void *pw_w[2];               // [Cout][Cin] storage type
    const float *pw_b[2];              // fp32 [Cout] or null
    void *dst[2];
    int dst_is_stack[2], dH[2], dW[2], dC[2], dc0[2];
    int offH, offW;
    int pdl;
    int per_image;                     // SIGE_CONV_PER_IMAGE_OPERANDS: idx holds B * N rows (row b*N + i = tile i of image b)
};

__host__ __device__ constexpr int smem_bytes(int cin) {
    return RING_BYTES + (M + BN) * (cin + 8) * 2 + 10 * cin * 4;
}

template <typename T>
__global__ void __launch_bounds__(NTHREADS) separable_conv_kernel(const Params p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int br = blockIdx.z, n0 = blockIdx.y * BN, t0 = blockIdx.x * TILES;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int Cin = p.Cin, apitch = Cin + 8;
    T *ring = reinterpret_cast<T *>(smem);
    T *As = reinterpret_cast<T *>(smem + RING_BYTES);
    T *Ws = As + M * apitch;
    float *dww = reinterpret_cast<float *>(Ws + BN * apitch);     // [9][Cin]
    float *dwb = dww + 9 * Cin;

    // ---- independent of the previous kernel: the weights of this (branch, channel block)
    const T *pw = static_cast<const T *>(p.pw_w[br]);
    const int cv = Cin / 8;
    for (int u = tid; u < BN * cv; u += NTHREADS) {
        const int n = u / cv, v = u - n * cv;
        const bool ok = n0 + n < p.Cout;
        cp_async16_zfill(smem_u32(Ws + n * apitch + v * 8), ok ? pw + (size_t)(n0 + n) * Cin + v * 8 : pw, ok);
    }
    cp_async_commit();
    const float *dw = p.dw_w[br], *db = p.dw_b[br];
    for (int u = tid; u < 9 * Cin; u += NTHREADS) {
        const int c = u / 9;
        dww[(u - c * 9) * Cin + c] = dw[u];
    }
    for (int c = tid; c < Cin; c += NTHREADS) dwb[c] = db ? db[c] : 0.f;
    if (p.pdl) {
        pdl_release();
        pdl_acquire();
    }

    // ---- halo addressing: a thread owns the same UPT (tile, pixel, 8-channel half) units in every chunk
    const T *src = static_cast<const T *>(p.src);
    long long goff[UPT];
    bool gok[UPT];
#pragma unroll
    for (int i = 0; i < UPT; ++i) {
        const int u = tid + i * NTHREADS;
        const int t = u / (HPIX * 2), pix = (u - t * HPIX * 2) >> 1;
        const int gt = t0 + t;
        bool ok = u < UNITS && gt < p.total;
        long long off = 0;
        if (ok) {
            if (p.src_is_stack) {
                off = ((long long)gt * HPIX + pix) * p.sC;
            } else {
                const int b = gt / p.N, ti = p.per_image ? gt : gt - b * p.N;
                const int oh = p.idx[2 * ti], ow = p.idx[2 * ti + 1];
                const int h = oh + pix / 6, w = ow + pix % 6;
                ok = oh != SIGE_TILE_NONE && h >= 0 && h < p.H && w >= 0 && w < p.W;
                off = (((long long)b * p.H + h) * p.W + w) * p.sC;
            }
        }
        goff[i] = off + p.sc0 + (u & 1) * 8;
        gok[i] = ok;
    }
    auto halo_issue = [&](int k) {
        T *hb = ring + (k % STAGES) * CHUNK_ELEMS;
#pragma unroll
        for (int i = 0; i < UPT; ++i) {
            const int u = tid + i * NTHREADS;
            if (u < UNITS) cp_async16_zfill(smem_u32(hb + u * 8), gok[i] ? src + goff[i] + k * KC : src, gok[i]);
        }
    };

    // ---- depthwise 3x3 on 16-channel chunks: thread = (output pixel m, 8-channel half v)
    const int nk = Cin / KC;
#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < nk) halo_issue(s);
        cp_async_commit();
    }
    const int dm = tid >> 1, dv = tid & 1;
    const int dt = dm >> 4, doy = (dm >> 2) & 3, dox = dm & 3;
    for (int k = 0; k < nk; ++k) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        if (k + STAGES - 1 < nk) halo_issue(k + STAGES - 1);
        cp_async_commit();
        const T *hb = ring + (k % STAGES) * CHUNK_ELEMS + dt * HPIX * KC + dv * 8;
        const int c = k * KC + dv * 8;
        float acc[8];
        {
            const float4 b0 = *reinterpret_cast<const float4 *>(dwb + c), b1 = *reinterpret_cast<const float4 *>(dwb + c + 4);
            acc[0] = b0.x; acc[1] = b0.y; acc[2] = b0.z; acc[3] = b0.w;
            acc[4] = b1.x; acc[5] = b1.y; acc[6] = b1.z; acc[7] = b1.w;
        }
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const Vec16<T> xv = *reinterpret_cast<const Vec16<T> *>(hb + ((doy + ky) * 6 + dox + kx) * KC);
                const float *wt = dww + (ky * 3 + kx) * Cin + c;
                const float4 w0 = *reinterpret_cast<const float4 *>(wt), w1 = *reinterpret_cast<const float4 *>(wt + 4);
                const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
                for (int z = 0; z < 8; ++z) acc[z] = fmaf(DT<T>::to_f(xv.v[z]), wv[z], acc[z]);
            }
        Vec16<T> o;
#pragma unroll
        for (int z = 0; z < 8; ++z) o.v[z] = DT<T>::from_f(acc[z]);
        *reinterpret_cast<Vec16<T> *>(As + dm * apitch + c) = o;
    }
    cp_async_wait<0>();
    __syncthreads();

    // ---- pointwise 1x1: [128 x Cin] x [Cin x 64], 8 warps as 4 (rows) x 2 (columns) of 32 x 32
    const int wm = warp & 3, wn = warp >> 2;
    float acc[2][4][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int z = 0; z < 4; ++z) acc[i][j][z] = 0.f;
    const int b_nl = ((lane >> 4) << 3) + (lane & 7), b_kh = (lane >> 3) & 1;
    if (n0 + wn * 32 < p.Cout) {
        for (int kk = 0; kk < Cin; kk += 16) {
            uint32_t a[2][4];
#pragma unroll
            for (int i = 0; i < 2; ++i)
                ldmatrix_x4(smem_u32(As + (wm * 32 + i * 16 + (lane & 15)) * apitch + kk + (lane >> 4) * 8), a[i][0], a[i][1], a[i][2], a[i][3]);
#pragma unroll
            for (int jp = 0; jp < 2; ++jp) {
                uint32_t b[4];
                ldmatrix_x4(smem_u32(Ws + (wn * 32 + jp * 16 + b_nl) * apitch + kk + b_kh * 8), b[0], b[1], b[2], b[3]);
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    mma_m16n8k16<T>(acc[i][2 * jp], a[i], b[0], b[1]);
                    mma_m16n8k16<T>(acc[i][2 * jp + 1], a[i], b[2], b[3]);
                }
            }
        }
    }

    // ---- epilogue: + bias, one rounding, staged over the (idle) halo ring, 16-byte channel vectors out
    T *stg = ring;
    const float *pb = p.pw_b[br];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int n = wn * 32 + j * 8 + (lane & 3) * 2;
        const float bb0 = (pb && n0 + n < p.Cout) ? pb[n0 + n] : 0.f, bb1 = (pb && n0 + n + 1 < p.Cout) ? pb[n0 + n + 1] : 0.f;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int m = wm * 32 + i * 16 + (lane >> 2);
            stg[m * STG_PITCH + n] = DT<T>::from_f(acc[i][j][0] + bb0);
            stg[m * STG_PITCH + n + 1] = DT<T>::from_f(acc[i][j][1] + bb1);
            stg[(m + 8) * STG_PITCH + n] = DT<T>::from_f(acc[i][j][2] + bb0);
            stg[(m + 8) * STG_PITCH + n + 1] = DT<T>::from_f(acc[i][j][3] + bb1);
        }
    }
    __syncthreads();
    T *dst = static_cast<T *>(p.dst[br]);
    const int dC = p.dC[br], dc0 = p.dc0[br];
    for (int u = tid; u < M * (BN / 8); u += NTHREADS) {
        const int m = u >> 3, v = u & 7;
        const int n = n0 + v * 8, gt = t0 + (m >> 4);
        if (n >= p.Cout || gt >= p.total) continue;
        const int oy = (m >> 2) & 3, ox = m & 3;
        const int b = gt / p.N, ti = p.per_image ? gt : gt - b * p.N;
        const int oh = p.idx ? p.idx[2 * ti] : 0;            // no list: a stack-to-stack launch, every row is a tile
        if (oh == SIGE_TILE_NONE) continue;                  // padding tiles write nothing, to a stack as to a buffer
        long long off;
        if (p.dst_is_stack[br]) {
            off = (((long long)gt * 4 + oy) * 4 + ox) * dC;
        } else {
            const int h = oh + p.offH + oy, w = p.idx[2 * ti + 1] + p.offW + ox;
            if (h < 0 || h >= p.dH[br] || w < 0 || w >= p.dW[br]) continue;
            off = (((long long)b * p.dH[br] + h) * p.dW[br] + w) * dC;
        }
        *reinterpret_cast<Vec16<T> *>(dst + off + dc0 + n) = *reinterpret_cast<const Vec16<T> *>(stg + m * STG_PITCH + v * 8);
    }
}

template <typename T> static int launch(const Params &p, cudaStream_t st) {
    auto kern = separable_conv_kernel<T>;
    static int attr_dev = -1;
    int dev = 0;
    cudaGetDevice(&dev);
    if (attr_dev != dev) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes(MAX_CIN));
        if (e != cudaSuccess) {
            set_error("sige_separable_conv: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
            (void)cudaGetLastError();
            return 2;
        }
        attr_dev = dev;
    }
    const dim3 grid(ceil_div(p.total, TILES), ceil_div(p.Cout, BN), p.dst[1] ? 2 : 1);
    const int smem = smem_bytes(p.Cin);
    const cudaError_t e = launch_ex(kern, grid, dim3(NTHREADS), smem, st, p.pdl != 0, dim3(1, 1, 1), p);
    if (e != cudaSuccess) {
        set_error("sige_separable_conv: launch failed (grid %d x %d x %d, %d B smem): %s", grid.x, grid.y, grid.z, smem,
                  cudaGetErrorString(e));
        (void)cudaGetLastError();
        return 2;
    }
    return 0;
}

static bool supported(int Cin, int Cout, int k, int dtype) {
    return k == 3 && (dtype == SIGE_F16 || dtype == SIGE_BF16) && Cin >= 16 && Cin <= MAX_CIN && Cin % 16 == 0 && Cout >= 8 &&
           Cout <= MAX_COUT && Cout % 8 == 0;
}

}  // namespace sep
}  // namespace sige

extern "C" int sige_separable_conv_supported(int Cin, int Cout, int k, int dtype) { return sige::sep::supported(Cin, Cout, k, dtype) ? 1 : 0; }

extern "C" int sige_separable_conv(const sige_separable_conv_t *d, sige_stream_t stream) {
    using namespace sige;
    SIGE_REQUIRE(d != nullptr, "sige_separable_conv: null descriptor");
    SIGE_REQUIRE(sep::supported(d->Cin, d->Cout, 3, d->dtype),
                 "sige_separable_conv: unsupported Cin = %d / Cout = %d / dtype %d (Cin a multiple of 16 in [16, 256], Cout a multiple of 8 "
                 "in [8, 1024], f16 / bf16)", d->Cin, d->Cout, d->dtype);
    SIGE_REQUIRE(d->nbranch == 1 || d->nbranch == 2, "sige_separable_conv: nbranch must be 1 or 2 (got %d)", d->nbranch);
    SIGE_REQUIRE(d->B >= 1 && d->N >= 0, "sige_separable_conv: B = %d, N = %d", d->B, d->N);
    SIGE_REQUIRE(d->src_C % 8 == 0 && d->src_c0 % 8 == 0 && d->src_c0 >= 0 && d->src_c0 + d->Cin <= d->src_C,
                 "sige_separable_conv: source channel window [%d, %d) out of range of a %d-channel pixel (offset and pixel channels "
                 "multiples of 8)", d->src_c0, d->src_c0 + d->Cin, d->src_C);
    if (!d->src_is_stack) SIGE_REQUIRE(d->H > 0 && d->W > 0, "sige_separable_conv: source extent %d x %d", d->H, d->W);
    for (int b = 0; b < d->nbranch; ++b) {
        const sige_separable_branch_t &r = d->branch[b];
        SIGE_REQUIRE(r.dst_C % 8 == 0 && r.dst_c0 % 8 == 0 && r.dst_c0 >= 0 && r.dst_c0 + d->Cout <= r.dst_C,
                     "sige_separable_conv: branch %d: destination channel window [%d, %d) out of range of a %d-channel pixel (offset and "
                     "pixel channels multiples of 8)", b, r.dst_c0, r.dst_c0 + d->Cout, r.dst_C);
        if (!r.dst_is_stack) SIGE_REQUIRE(r.dH > 0 && r.dW > 0, "sige_separable_conv: branch %d: destination extent %d x %d", b, r.dH, r.dW);
    }
    const bool per_image = (d->flags & SIGE_CONV_PER_IMAGE_OPERANDS) != 0;
    if (per_image)
        SIGE_REQUIRE(!d->src_is_stack && !d->branch[0].dst_is_stack && (d->nbranch == 1 || !d->branch[1].dst_is_stack),
                     "sige_separable_conv: SIGE_CONV_PER_IMAGE_OPERANDS (per-image tile lists) needs a buffer source and buffer destinations, not stacks");
    if (d->N == 0) return 0;
    SIGE_REQUIRE(d->src != nullptr, "sige_separable_conv: null source");
    SIGE_REQUIRE(d->idx != nullptr || (d->src_is_stack && d->branch[0].dst_is_stack && (d->nbranch == 1 || d->branch[1].dst_is_stack)),
                 "sige_separable_conv: null tile list");
    SIGE_REQUIRE((uintptr_t)d->src % 16 == 0, "sige_separable_conv: source must be 16-byte aligned");
    for (int b = 0; b < d->nbranch; ++b) {
        const sige_separable_branch_t &r = d->branch[b];
        SIGE_REQUIRE(r.dw_weight && r.pw_weight && r.dst, "sige_separable_conv: branch %d: null weight or destination", b);
        SIGE_REQUIRE(((uintptr_t)r.dst | (uintptr_t)r.pw_weight) % 16 == 0 && (uintptr_t)r.dw_weight % 4 == 0,
                     "sige_separable_conv: branch %d: destination and pointwise weights must be 16-byte aligned", b);
    }
    sep::Params p = {};
    p.src = d->src;
    p.src_is_stack = d->src_is_stack;
    p.sC = d->src_C;
    p.sc0 = d->src_c0;
    p.B = d->B;
    p.H = d->H;
    p.W = d->W;
    p.idx = d->idx;
    p.N = d->N;
    p.total = d->B * d->N;
    p.Cin = d->Cin;
    p.Cout = d->Cout;
    for (int b = 0; b < d->nbranch; ++b) {
        const sige_separable_branch_t &r = d->branch[b];
        p.dw_w[b] = r.dw_weight;
        p.dw_b[b] = r.dw_bias;
        p.pw_w[b] = r.pw_weight;
        p.pw_b[b] = r.pw_bias;
        p.dst[b] = r.dst;
        p.dst_is_stack[b] = r.dst_is_stack;
        p.dH[b] = r.dH;
        p.dW[b] = r.dW;
        p.dC[b] = r.dst_C;
        p.dc0[b] = r.dst_c0;
    }
    p.offH = d->offH;
    p.offW = d->offW;
    p.pdl = (d->flags & SIGE_CONV_PDL) ? 1 : 0;
    p.per_image = per_image ? 1 : 0;
    cudaStream_t st = (cudaStream_t)stream;
    return d->dtype == SIGE_F16 ? sep::launch<__half>(p, st) : sep::launch<__nv_bfloat16>(p, st);
}
