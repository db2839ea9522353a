// spade_modulate.cu — SPADE's modulation of a tile stack, one launch:
//   out = act( x * (1 + gamma) + beta ),   act = identity or leaky_relu(slope)
// Replaces the four pointwise torch calls the reference issues per SPADE layer on the gathered tiles, between a Gather /
// ScatterGather and the SIGEConv2d that reads the result: gaugan/models/sige_normalization.py:84-86 (`normalized * (1 + gamma) +
// beta`, gamma / beta = the two channel halves of mlp_gamma_beta's scattered-and-regathered output) and the block's
// `F.leaky_relu(., 0.2)` (gaugan/models/spade_generators/sige_fused_spade_generator.py:200-201).
// Pure HBM traffic: 3 reads + 1 write of [pixels, C]; a thread owns one 16-byte channel vector of one pixel, every operand has
// its own pixel stride (gamma and beta are channel slices of one [pixels, 2C] tensor), channels innermost.  fp32 arithmetic,
// one rounding (the recorded calls round after each of their four steps).
#include "common.cuh"

namespace sige {

template <typename T>
__global__ void __launch_bounds__(256) spade_modulate_kernel(const T *__restrict__ x, long long xs, const T *__restrict__ g, long long gs,
                                                             const T *__restrict__ b, long long bs, T *__restrict__ out, long long os,
                                                             long long pixels, int C, float slope) {
    constexpr int V = DT<T>::vec;
    const int CV = C / V;
    const long long total = pixels * CV;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long pix = i / CV;
        const int c0 = (int)(i - pix * CV) * V;
        const Vec16<T> xv = *reinterpret_cast<const Vec16<T> *>(x + pix * xs + c0);
        const Vec16<T> gv = *reinterpret_cast<const Vec16<T> *>(g + pix * gs + c0);
        const Vec16<T> bv = *reinterpret_cast<const Vec16<T> *>(b + pix * bs + c0);
        Vec16<T> o;
#pragma unroll
        for (int z = 0; z < V; ++z) {
            float f = fmaf(DT<T>::to_f(xv.v[z]), 1.0f + DT<T>::to_f(gv.v[z]), DT<T>::to_f(bv.v[z]));
            f = f > 0.f ? f : f * slope;
            o.v[z] = DT<T>::from_f(f);
        }
        *reinterpret_cast<Vec16<T> *>(out + pix * os + c0) = o;
    }
}

template <typename T>
static int launch_spade(const void *x, long long xs, const void *g, long long gs, const void *b, long long bs, void *out, long long os, long long pixels,
                        int C, float slope, cudaStream_t st) {
    const long long items = pixels * (C / DT<T>::vec);
    const int blocks = (int)(items + 255 < 16LL * sm_count() * 256 ? (items + 255) / 256 : 16LL * sm_count());
    spade_modulate_kernel<T><<<blocks, 256, 0, st>>>((const T *)x, xs, (const T *)g, gs, (const T *)b, bs, (T *)out, os, pixels, C, slope);
    return check_launch("sige_spade_modulate");
}

}  // namespace sige

extern "C" int sige_spade_modulate(const void *x, long long x_pixel_stride, const void *gamma, long long gamma_pixel_stride, const void *beta,
                                   long long beta_pixel_stride, void *out, long long out_pixel_stride, long long pixels, int C,
                                   float negative_slope, int dtype, sige_stream_t stream) {
    using namespace sige;
    SIGE_REQUIRE(pixels >= 0 && C > 0, "sige_spade_modulate: pixels = %lld, C = %d", pixels, C);
    if (pixels == 0) return 0;
    SIGE_REQUIRE(x && gamma && beta && out, "sige_spade_modulate: null buffer");
    const int vec = dtype == SIGE_F32 ? 4 : 8;
    SIGE_REQUIRE(dtype == SIGE_F32 || dtype == SIGE_F16 || dtype == SIGE_BF16, "sige_spade_modulate: unsupported dtype %d", dtype);
    SIGE_REQUIRE(C % vec == 0 && x_pixel_stride % vec == 0 && gamma_pixel_stride % vec == 0 && beta_pixel_stride % vec == 0 && out_pixel_stride % vec == 0,
                 "sige_spade_modulate: C and the pixel strides must be multiples of %d elements (16-byte channel vectors)", vec);
    SIGE_REQUIRE(((uintptr_t)x | (uintptr_t)gamma | (uintptr_t)beta | (uintptr_t)out) % 16 == 0, "sige_spade_modulate: buffers must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case SIGE_F32: return launch_spade<float>(x, x_pixel_stride, gamma, gamma_pixel_stride, beta, beta_pixel_stride, out, out_pixel_stride, pixels, C, negative_slope, st);
        case SIGE_F16: return launch_spade<__half>(x, x_pixel_stride, gamma, gamma_pixel_stride, beta, beta_pixel_stride, out, out_pixel_stride, pixels, C, negative_slope, st);
        default: return launch_spade<__nv_bfloat16>(x, x_pixel_stride, gamma, gamma_pixel_stride, beta, beta_pixel_stride, out, out_pixel_stride, pixels, C, negative_slope, st);
    }
}
