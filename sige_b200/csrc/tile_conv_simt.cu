// tile_conv_simt.cu — generic tile convolution on a stack, CUDA cores, fp32 accumulation.
//
// The exact-fp32 / odd-shape companion of tile_conv_mma.cu: any storage dtype, any channel
// count (GauGAN's Cin = 36, RGB inputs), groups (depthwise) and dilation.  It computes what
// the reference obtains from F.conv2d(x, w, b, stride, (0,0), dilation, groups) on the
// gathered stack (reference sige/nn/base.py:88-89).  fp32 inputs are multiplied and
// accumulated in true fp32 (fmaf, no TF32), which is what the 1e-5 parity bar needs.
//
// One CTA = one tile x 64 output channels of one group.  Per 16-input-channel chunk the halo
// tile and the matching weight slab are staged in shared memory; a warp shares one output
// pixel group, so activation reads are smem broadcasts and weight reads are conflict-free
// (row pitch padded to an odd number of words).
#include <algorithm>

#include "common.cuh"

namespace sige {

constexpr int SIMT_CO = 64;    // output channels per CTA
constexpr int SIMT_CI = 16;    // input channels per chunk
constexpr int SIMT_PG = 4;     // pixel groups (threads = SIMT_CO * SIMT_PG)
constexpr int SIMT_MAXPP = 8;  // output pixels per thread per pass

struct SimtParams {
    int M, Cin, R, S, Cout, kH, kW, strideH, strideW, dilH, dilW, groups;
    int Ro, So, P, RS, taps, cig, cog;
    int nhwc;
};

template <typename T>
__global__ void __launch_bounds__(SIMT_CO *SIMT_PG)
tile_conv_simt_kernel(SimtParams p, const T *__restrict__ x, const T *__restrict__ w, const T *__restrict__ bias,
                      T *__restrict__ out) {
    extern __shared__ float sm[];
    float *xs = sm;                              // [SIMT_CI][RS]
    const int wpitch = SIMT_CI * p.taps + 1;     // odd pitch -> conflict-free across co
    float *ws = sm + SIMT_CI * p.RS;             // [SIMT_CO][wpitch]

    const int m = blockIdx.x, g = blockIdx.z;
    const int co_l = threadIdx.x % SIMT_CO, pg = threadIdx.x / SIMT_CO;
    const int co_in_g = blockIdx.y * SIMT_CO + co_l;         // channel index inside the group
    const bool co_ok = co_in_g < p.cog;
    const int co = g * p.cog + co_in_g;
    const int ci0g = g * p.cig;

    for (int pbase = 0; pbase < p.P; pbase += SIMT_PG * SIMT_MAXPP) {
        float acc[SIMT_MAXPP];
        int xoff[SIMT_MAXPP];
#pragma unroll
        for (int k = 0; k < SIMT_MAXPP; ++k) {
            acc[k] = 0.f;
            const int pp = pbase + pg + k * SIMT_PG;
            const int oy = pp / p.So, ox = pp - oy * p.So;
            xoff[k] = pp < p.P ? (oy * p.strideH) * p.S + ox * p.strideW : -1;
        }
        for (int c0 = 0; c0 < p.cig; c0 += SIMT_CI) {
            const int nci = min(SIMT_CI, p.cig - c0);
            __syncthreads();
            // halo tile chunk
            for (int e = threadIdx.x; e < nci * p.RS; e += blockDim.x) {
                int ci, pix;
                if (p.nhwc) { ci = e % nci; pix = e / nci; } else { pix = e % p.RS; ci = e / p.RS; }
                const long long src = p.nhwc ? (((long long)m * p.RS + pix) * p.Cin + ci0g + c0 + ci)
                                             : (((long long)m * p.Cin + ci0g + c0 + ci) * p.RS + pix);
                xs[ci * p.RS + pix] = DT<T>::to_f(x[src]);
            }
            // weight slab: w[co][c0:c0+nci][taps] is contiguous per co
            for (int e = threadIdx.x; e < SIMT_CO * nci * p.taps; e += blockDim.x) {
                const int cl = e / (nci * p.taps), rem = e - cl * (nci * p.taps);
                const int cg = blockIdx.y * SIMT_CO + cl;
                float v = 0.f;
                if (cg < p.cog) v = DT<T>::to_f(w[((long long)(g * p.cog + cg) * p.cig + c0) * p.taps + rem]);
                ws[cl * wpitch + rem] = v;
            }
            __syncthreads();
            const float *wr = ws + co_l * wpitch;
            for (int ci = 0; ci < nci; ++ci) {
                const float *xr = xs + ci * p.RS;
                for (int ky = 0; ky < p.kH; ++ky)
                    for (int kx = 0; kx < p.kW; ++kx) {
                        const float wv = wr[(ci * p.kH + ky) * p.kW + kx];
                        const int toff = ky * p.dilH * p.S + kx * p.dilW;
#pragma unroll
                        for (int k = 0; k < SIMT_MAXPP; ++k)
                            if (xoff[k] >= 0) acc[k] = fmaf(xr[xoff[k] + toff], wv, acc[k]);
                    }
            }
        }
        if (co_ok) {
            const float bv = bias ? DT<T>::to_f(bias[co]) : 0.f;
#pragma unroll
            for (int k = 0; k < SIMT_MAXPP; ++k) {
                const int pp = pbase + pg + k * SIMT_PG;
                if (pp < p.P) {
                    const long long dst = p.nhwc ? (((long long)m * p.P + pp) * p.Cout + co)
                                                 : (((long long)m * p.Cout + co) * p.P + pp);
                    out[dst] = DT<T>::from_f(acc[k] + bv);
                }
            }
        }
    }
}

// Depthwise form (groups == Cin == Cout: GauGAN's separable convolutions, reference gaugan/models/mobile_modules.py:83-91).  The
// generic kernel above gives one CTA of 256 threads to each (tile, channel) and uses one of them; here a thread owns one
// output pixel of one channel (NCHW) or of 8 / 4 adjacent channels (NHWC: 16-byte vectors, neighbouring threads = neighbouring
// channel vectors, so every tap is a coalesced row read that L1 serves for the other taps).  Same arithmetic: fp32 fmaf in
// (ky, kx) order.
template <typename T>
__global__ void __launch_bounds__(256) tile_conv_depthwise_kernel(SimtParams p, const T *__restrict__ x, const T *__restrict__ w,
                                                                  const T *__restrict__ bias, T *__restrict__ out) {
    constexpr int V = DT<T>::vec;
    if (p.nhwc == 1) {
        const int CV = p.Cin / V;
        const long long total = (long long)p.M * p.P * CV;
        for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
            const int cv = (int)(i % CV);
            const long long mp = i / CV;
            const int pp = (int)(mp % p.P);
            const long long m = mp / p.P;
            const int oy = pp / p.So, ox = pp - oy * p.So;
            const int c0 = cv * V;
            float acc[V];
#pragma unroll
            for (int z = 0; z < V; ++z) acc[z] = bias ? DT<T>::to_f(bias[c0 + z]) : 0.f;
            float part[V];
#pragma unroll
            for (int z = 0; z < V; ++z) part[z] = 0.f;
            for (int ky = 0; ky < p.kH; ++ky)
                for (int kx = 0; kx < p.kW; ++kx) {
                    const int pix = (oy * p.strideH + ky * p.dilH) * p.S + ox * p.strideW + kx * p.dilW;
                    const Vec16<T> xv = *reinterpret_cast<const Vec16<T> *>(x + (m * p.RS + pix) * p.Cin + c0);
#pragma unroll
                    for (int z = 0; z < V; ++z)
                        part[z] = fmaf(DT<T>::to_f(xv.v[z]), DT<T>::to_f(w[(long long)(c0 + z) * p.taps + ky * p.kW + kx]), part[z]);
                }
            Vec16<T> o;
#pragma unroll
            for (int z = 0; z < V; ++z) o.v[z] = DT<T>::from_f(part[z] + acc[z]);
            *reinterpret_cast<Vec16<T> *>(out + (m * p.P + pp) * p.Cout + c0) = o;
        }
        return;
    }
    const long long total = (long long)p.M * p.Cin * p.P;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int pp, c;
        long long m;
        if (p.nhwc) { c = (int)(i % p.Cin); pp = (int)((i / p.Cin) % p.P); m = i / ((long long)p.Cin * p.P); }
        else { pp = (int)(i % p.P); c = (int)((i / p.P) % p.Cin); m = i / ((long long)p.P * p.Cin); }
        const int oy = pp / p.So, ox = pp - oy * p.So;
        float acc = 0.f;
        for (int ky = 0; ky < p.kH; ++ky)
            for (int kx = 0; kx < p.kW; ++kx) {
                const int pix = (oy * p.strideH + ky * p.dilH) * p.S + ox * p.strideW + kx * p.dilW;
                const long long src = p.nhwc ? ((m * p.RS + pix) * p.Cin + c) : ((m * p.Cin + c) * p.RS + pix);
                acc = fmaf(DT<T>::to_f(x[src]), DT<T>::to_f(w[(long long)c * p.taps + ky * p.kW + kx]), acc);
            }
        const long long dst = p.nhwc ? ((m * p.P + pp) * p.Cout + c) : ((m * p.Cout + c) * p.P + pp);
        out[dst] = DT<T>::from_f(acc + (bias ? DT<T>::to_f(bias[c]) : 0.f));
    }
}

template <typename T>
static int launch_depthwise(const SimtParams &p, const void *x, const void *w, const void *bias, void *out, cudaStream_t st) {
    SimtParams q = p;
    const bool vec = p.nhwc && p.Cin % DT<T>::vec == 0 && ((uintptr_t)x % 16 == 0) && ((uintptr_t)out % 16 == 0);
    q.nhwc = p.nhwc ? (vec ? 1 : 2) : 0;          // 1 = NHWC with 16-byte channel vectors, 2 = NHWC scalar, 0 = NCHW scalar
    const long long items = vec ? (long long)p.M * p.P * (p.Cin / DT<T>::vec) : (long long)p.M * p.Cin * p.P;
    const int blocks = (int)std::min<long long>((items + 255) / 256, 16LL * sm_count());
    tile_conv_depthwise_kernel<T><<<blocks, 256, 0, st>>>(q, (const T *)x, (const T *)w, (const T *)bias, (T *)out);
    return check_launch("sige_tile_conv_generic(depthwise)");
}

template <typename T>
static int launch_simt(const SimtParams &p, const void *x, const void *w, const void *bias, void *out, cudaStream_t st) {
    const size_t smem = sizeof(float) * ((size_t)SIMT_CI * p.RS + (size_t)SIMT_CO * (SIMT_CI * p.taps + 1));
    auto kern = tile_conv_simt_kernel<T>;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) {
            set_error("sige_tile_conv_generic: tile too large for shared memory (%zu bytes): %s", smem, cudaGetErrorString(e));
            return 1;
        }
    }
    dim3 grid(p.M, ceil_div(p.cog, SIMT_CO), p.groups);
    kern<<<grid, SIMT_CO * SIMT_PG, smem, st>>>(p, (const T *)x, (const T *)w, (const T *)bias, (T *)out);
    return check_launch("sige_tile_conv_generic");
}

}  // namespace sige

using namespace sige;

extern "C" int sige_tile_conv_generic(const void *x, const void *w, const void *bias, void *out, int dtype, int layout,
                                      int M, int Cin, int R, int S, int Cout, int kH, int kW, int strideH, int strideW,
                                      int dilH, int dilW, int groups, sige_stream_t stream) {
    SIGE_REQUIRE(M >= 0 && Cin > 0 && Cout > 0 && R > 0 && S > 0 && kH > 0 && kW > 0 && strideH > 0 && strideW > 0 &&
                     dilH > 0 && dilW > 0 && groups > 0,
                 "sige_tile_conv_generic: bad shape");
    SIGE_REQUIRE(Cin % groups == 0 && Cout % groups == 0, "sige_tile_conv_generic: channels not divisible by groups");
    SIGE_REQUIRE(layout == SIGE_NCHW || layout == SIGE_NHWC, "sige_tile_conv_generic: bad layout %d", layout);
    const int eH = dilH * (kH - 1) + 1, eW = dilW * (kW - 1) + 1;
    SIGE_REQUIRE(R >= eH && S >= eW, "sige_tile_conv_generic: tile smaller than the (dilated) kernel");
    if (M == 0) return 0;
    SIGE_REQUIRE(M <= 2147483647 / 1, "sige_tile_conv_generic: too many tiles");
    SIGE_REQUIRE(x && w && out, "sige_tile_conv_generic: null pointer");
    SimtParams p;
    p.M = M; p.Cin = Cin; p.R = R; p.S = S; p.Cout = Cout; p.kH = kH; p.kW = kW;
    p.strideH = strideH; p.strideW = strideW; p.dilH = dilH; p.dilW = dilW; p.groups = groups;
    p.Ro = (R - eH) / strideH + 1; p.So = (S - eW) / strideW + 1; p.P = p.Ro * p.So;
    p.RS = R * S; p.taps = kH * kW; p.cig = Cin / groups; p.cog = Cout / groups;
    p.nhwc = layout == SIGE_NHWC;
    SIGE_REQUIRE(groups <= 65535 && ceil_div(p.cog, SIMT_CO) <= 65535, "sige_tile_conv_generic: grid too large");
    cudaStream_t st = (cudaStream_t)stream;
    if (groups == Cin && Cout == Cin) {            // depthwise: one thread per output (vector), not one CTA per (tile, channel)
        switch (dtype) {
            case SIGE_F32: return launch_depthwise<float>(p, x, w, bias, out, st);
            case SIGE_F16: return launch_depthwise<__half>(p, x, w, bias, out, st);
            case SIGE_BF16: return launch_depthwise<__nv_bfloat16>(p, x, w, bias, out, st);
            default: set_error("sige_tile_conv_generic: unsupported dtype %d", dtype); return 1;
        }
    }
    switch (dtype) {
        case SIGE_F32: return launch_simt<float>(p, x, w, bias, out, st);
        case SIGE_F16: return launch_simt<__half>(p, x, w, bias, out, st);
        case SIGE_BF16: return launch_simt<__nv_bfloat16>(p, x, w, bias, out, st);
        default: set_error("sige_tile_conv_generic: unsupported dtype %d", dtype); return 1;
    }
}
