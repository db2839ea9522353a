// common.cuh — shared device helpers for the sm_90a SIGE kernels.
//
// Replaces reference sige/common.cpp (enums, broadcastable) and
// sige/cuda/common_cuda.cu (binary_op_array_cuda, activation_cuda).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <utility>

#include "../../include/sige_b200.h"
#include "ptx.cuh"

namespace sige {

// Streaming multiprocessors of the current device, queried once per device; 132 (H100 SXM) where no device can be queried
// (host-only planning on a machine without a GPU).
constexpr int kDefaultSMs = 132;
inline int sm_count() {
    static int cache[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) {
        (void)cudaGetLastError();
        return kDefaultSMs;
    }
    if (cache[dev] == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
            (void)cudaGetLastError();
            return kDefaultSMs;
        }
        cache[dev] = n;
    }
    return cache[dev];
}

// ----------------------------------------------------------------------------
// error plumbing (host)
// ----------------------------------------------------------------------------
void set_error(const char *fmt, ...);
int check_launch(const char *what);

#define SIGE_REQUIRE(cond, ...)          \
    do {                                 \
        if (!(cond)) {                   \
            ::sige::set_error(__VA_ARGS__); \
            return 1;                    \
        }                                \
    } while (0)

// cudaLaunchKernelEx with a thread-block cluster (attribute added only when `cluster` is not 1x1x1) and programmatic
// dependent launch (attribute added only when `pdl` is set).  The caller reports a failure in its own words.
template <typename... KArgs, typename... Args>
cudaError_t launch_ex(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl, dim3 cluster,
                      Args &&...args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attrs[2];
    int na = 0;
    if (cluster.x * cluster.y * cluster.z > 1) {
        attrs[na].id = cudaLaunchAttributeClusterDimension;
        attrs[na].val.clusterDim.x = cluster.x;
        attrs[na].val.clusterDim.y = cluster.y;
        attrs[na].val.clusterDim.z = cluster.z;
        ++na;
    }
    if (pdl) {
        attrs[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attrs[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    cfg.attrs = attrs;
    cfg.numAttrs = na;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// ----------------------------------------------------------------------------
// dtype traits
// ----------------------------------------------------------------------------
template <typename T> struct DT;
template <> struct DT<float> {
    static constexpr int id = SIGE_F32;
    static constexpr int vec = 4;  // elements per 16 B
    __device__ __forceinline__ static float to_f(float v) { return v; }
    __device__ __forceinline__ static float from_f(float v) { return v; }
};
template <> struct DT<__half> {
    static constexpr int id = SIGE_F16;
    static constexpr int vec = 8;
    __device__ __forceinline__ static float to_f(__half v) { return __half2float(v); }
    __device__ __forceinline__ static __half from_f(float v) { return __float2half_rn(v); }
};
template <> struct DT<__nv_bfloat16> {
    static constexpr int id = SIGE_BF16;
    static constexpr int vec = 8;
    __device__ __forceinline__ static float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
    __device__ __forceinline__ static __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};

// 16-byte vector of T
template <typename T> struct alignas(16) Vec16 {
    T v[DT<T>::vec];
};

// ----------------------------------------------------------------------------
// activation   (reference sige/cuda/common_cuda.cu:32-38)
// The reference evaluates swish as z / (1.0 + exp(-z)): float expf, double add and
// divide.  For fp32 tensors we keep an accurate fp32 expf + IEEE division (<= 1 ulp
// from the reference's value); for fp16/bf16 storage the fast intrinsics are used
// (their error is far below the storage rounding).
// ----------------------------------------------------------------------------
template <bool kFast> __device__ __forceinline__ float swish(float z) {
    if (kFast) return __fdividef(z, 1.0f + __expf(-z));
    return z / (1.0f + expf(-z));
}
// SIGE_ACT_RELU is accepted only as the activation of a tile-conv aux destination (the fused ReLU epilogue).
template <bool kFast> __device__ __forceinline__ float activate(int act, float z) {
    return act == SIGE_ACT_SWISH ? swish<kFast>(z) : act == SIGE_ACT_RELU ? fmaxf(z, 0.f) : z;
}

// ----------------------------------------------------------------------------
// broadcast operand (device copy of sige_bcast_t with size-1 strides zeroed)
// reference sige/cuda/common_cuda.cu:15-30
// ----------------------------------------------------------------------------
struct Bcast {
    const void *ptr;   // nullptr = absent
    long long sb, sc, sh, sw;  // element strides, 0 where the dim has size 1
    int dtype;
    int c_contig;  // 1 if channel stride == 1 (vector loads along C allowed)
};

__device__ __forceinline__ float bcast_load(const Bcast &o, long long off) {
    if (o.dtype == SIGE_F32) return reinterpret_cast<const float *>(o.ptr)[off];
    if (o.dtype == SIGE_F16) return __half2float(reinterpret_cast<const __half *>(o.ptr)[off]);
    return __bfloat162float(reinterpret_cast<const __nv_bfloat16 *>(o.ptr)[off]);
}
__device__ __forceinline__ float bcast_at(const Bcast &o, int b, int c, int h, int w) {
    return bcast_load(o, b * o.sb + c * o.sc + h * o.sh + w * o.sw);
}

// order of operations: reference sige/cuda/gather_kernel.cu:45-65
template <bool kFast>
__device__ __forceinline__ float affine_act(float z, const Bcast &scale, const Bcast &shift, int act,
                                            bool act_first, int b, int c, int h, int w) {
    if (!act_first) {
        if (scale.ptr) z = bcast_at(scale, b, c, h, w) * z;
        if (shift.ptr) z = bcast_at(shift, b, c, h, w) + z;
    }
    z = activate<kFast>(act, z);
    if (act_first) {
        if (scale.ptr) z = bcast_at(scale, b, c, h, w) * z;
        if (shift.ptr) z = bcast_at(shift, b, c, h, w) + z;
    }
    return z;
}

// host: validate and convert a sige_bcast_t against the full extent (B,C,H,W)
int make_bcast(const sige_bcast_t *in, int B, int C, int H, int W, const char *name, Bcast *out);

inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

}  // namespace sige
