// ptx.cuh — inline-PTX wrappers used by more than one sm_90a kernel, each written once.
//
// Wrappers with a single user (wgmma, TMA, st.async, mapa, ...) live next to that user.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include <type_traits>

namespace sige {

// generic -> shared::cta address
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ----------------------------------------------------------------------------
// ldmatrix / mma.sync (legacy tensor-core path)
// ----------------------------------------------------------------------------
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t &r0, uint32_t &r1, uint32_t &r2, uint32_t &r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t addr, uint32_t &r0, uint32_t &r1, uint32_t &r2, uint32_t &r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
// D[16 x 8] += A[16 x 16] * B[16 x 8], T = __half or __nv_bfloat16, fp32 accumulator
template <typename T> __device__ __forceinline__ void mma_m16n8k16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    if constexpr (std::is_same<T, __half>::value)
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    else
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// two floats -> one 32-bit register of two T (round to nearest), the A-operand / store format
template <typename T> __device__ __forceinline__ uint32_t pack2(float a, float b) {
    if constexpr (std::is_same<T, __half>::value) {
        __half2 h = __floats2half2_rn(a, b);
        return *reinterpret_cast<uint32_t *>(&h);
    } else {
        __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
        return *reinterpret_cast<uint32_t *>(&h);
    }
}

// ----------------------------------------------------------------------------
// cp.async (LDGSTS), 16 bytes, bypassing L1; valid = false zero-fills the destination without reading
// ----------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void *src, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// ----------------------------------------------------------------------------
// mbarrier (shared::cta)
// ----------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}

// ----------------------------------------------------------------------------
// programmatic dependent launch
// ----------------------------------------------------------------------------
// let the next kernel of the stream start its prologue (no-op without a programmatic edge)
__device__ __forceinline__ void pdl_release() { asm volatile("griddepcontrol.launch_dependents;\n" ::); }
// wait until the previous kernel of the stream has completed and its writes are visible (no-op without a programmatic edge)
__device__ __forceinline__ void pdl_acquire() { asm volatile("griddepcontrol.wait;\n" ::: "memory"); }

}  // namespace sige
