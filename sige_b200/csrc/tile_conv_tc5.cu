// tile_conv_tc5.cu — Hopper-native fused gather -> (affine + SiLU) -> tile conv -> (+bias, +residual)
// -> scatter: wgmma with register accumulators, weights staged by TMA (cp.async.bulk.tensor, 128-byte
// swizzle), warp-specialised producer / MMA-consumer roles, mbarrier pipelines, split-K over a
// thread-block cluster with a distributed-shared-memory reduction.
//
// Same contract as tile_conv_mma.cu (one launch == the reference's Gather -> SIGEConv2d -> Scatter
// triple, reference sige/nn/gather.py:76-89, base.py:88-89, scatter.py:41-60); this file covers the
// geometries that make up >90 % of a DDPM step: 3x3 stride-1 on 6x6 halo tiles, 1x1 on 4x4 tiles and
// 3x3 stride-2 on 5x5 tiles.  Everything else stays on the mma.sync kernel.
//
// GEMM view per CTA: D[128 x BN] += A[128 x K] * B[K x BN], K = taps * Cin.  Two consumer warpgroups
// each own 64 rows and issue wgmma.m64nBNk16 with both operands in shared memory.
//   * 128 rows = 8 active tiles x 16 output pixels.  For the 3x3 case the row order is
//     m = oy*32 + tile*4 + ox and the A operand of tap (ky,kx) must be a plainly strided
//     [128 rows x 64 ch] K-major matrix (wgmma descriptors cannot express a gather).  Trick: keep
//     THREE column-shifted copies of the halo tiles in shared memory, copy kx laid out as
//     [y = 0..5][tile = 0..7][x' = 0..3] rows of 128 bytes holding halo pixel (y, kx + x').  Then
//     tap (ky,kx) is copy kx shifted by ky*32 rows: row m of the MMA reads row m + 32*ky — a pure
//     start-address offset of ky*4096 bytes, which is a multiple of the 1024-byte swizzle atom.
//     Cost: each gathered pixel is stored ~2x instead of the 9x of an im2col.
//   * B (weights, pre-packed [tap][Cin/64][Cout][64]) is a 2-D tensor map {64, taps*Cin/64*Cout}; one TMA
//     box {64, BN} (a contiguous BN*128-byte run) per (tap, 64-channel chunk) lands in a 128B-swizzled stage of an mbarrier ring.
//   * the consumers release weight stages and halo buffers once wgmma.wait_group has retired the MMAs that
//     read them; the fp32 accumulators are staged through shared memory so that the epilogue writes whole
//     16-byte runs of each NHWC pixel.
#include <cooperative_groups.h>
#include <cuda.h>

#include <type_traits>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace sige {
namespace tc5 {

constexpr int KC = 64;                 // channels per K chunk = one 128-byte swizzle row
constexpr int TILES = 8;               // tiles per CTA  (8 x 16 output pixels = 128 GEMM rows)
constexpr int NCONS_WARPS = 8;         // two MMA-consumer warpgroups (64 GEMM rows each; they also own the accumulators)
constexpr int NCONS = 32 * NCONS_WARPS;
constexpr int NPROD_WARPS = 8;         // A-operand producer warps
constexpr int NPROD = 32 * NPROD_WARPS;
constexpr int TMA_WARP = NCONS_WARPS + NPROD_WARPS;     // weight loads
constexpr int NTHREADS = 32 * (TMA_WARP + 1);
constexpr int A_COPY_BYTES = 6 * TILES * 4 * 128;        // one kx-copy: [6][8][4] rows x 128 B = 24576
constexpr int A_BUF_BYTES = 3 * A_COPY_BYTES;            // 73728 per 64-channel chunk
constexpr int EPI_PAD = 4;
// Stride-2 geometry (3x3 stride 2 on 5x5 halo tiles -> 2x2 outputs, the DDPM Downsample: reference
// diffusion/models/ddpm_arch/sige_fused_unet.py:212-221): 32 tiles x 4 outputs = 128 GEMM rows, row m = oy*64 + tile*2 + ox.
// Output (oy, ox) of tap (ky, kx) reads halo pixel (2*oy + ky, 2*ox + kx), so the halo rows are kept as five 64-row PLANES
// ordered y = 0, 2, 4, 1, 3 and copy kx holds pixel (y, 2*ox + kx) in row plane(y)*64 + tile*2 + ox: tap (ky, kx) is then
// copy kx starting at plane {0, 3, 1}[ky] — again ONE descriptor per tap, a start offset that is a multiple of 8192 bytes.
// A gathered pixel is stored 1.2 times (x = 2 feeds kx = 0 and kx = 2).
constexpr int S2_TILES = 32;
constexpr int S2_COPY_BYTES = 5 * 64 * 128;              // 40960
constexpr int S2_BUF_BYTES = 3 * S2_COPY_BYTES;          // 122880 per 64-channel chunk

struct Seg {
    const void *ptr;
    int pitch;   // elements from one pixel to the next (the segment's channel count, or more for a channel window, see ConvSeg)
    int up;
};

struct AuxDst {
    void *ptr;
    int C, c0;
    const float *scale, *shift;
    int act;
};

struct Params {
    Seg seg[2];
    int C0;
    int H, W;
    int src_is_stack;
    const int32_t *idx;
    int N, NT;
    const float *scale, *shift;
    int affine_bstride;
    int act;
    const float *bias;
    int Cin, Cout, taps;       // taps = 9 (3x3 on 6x6 tiles) or 1 (1x1 on 4x4 tiles)
    void *dst;
    int dst_is_stack;
    int dH, dW, dC, dst_c0;
    int offH, offW;
    const void *residual;
    int rC, res_c0;
    int n_aux;
    AuxDst aux[2];
    // optional second operand set: out += conv1x1(seg2) on tiles with sc_flags != 0 (the ResNet shortcut), see sige_tile_conv_t
    Seg seg2[2];
    int C0_2, Cin2;
    const float *bias2;
    const unsigned char *sc_flags;
    int padded;                // SIGE_CONV_PADDED: whole CTAs of SIGE_TILE_NONE padding may follow the real tiles (of each image)
    int idx_per_image;         // 1: idx / sc_flags hold B*N entries (row b*N + i = tile i of image b), else N shared by all images
    int ksplit;
    int pdl;                   // launched with programmatic dependent launch: the next layer is released at the epilogue
    int early_release;         // SIGE_CONV_EARLY_RELEASE: released right after this launch's own dependency has resolved instead
    int early;                 // SIGE_CONV_EARLY_* >> 4: source groups whose chunks are gathered before the dependency resolves (KOrder)
    int is_bf16;
    // SPADE modulation in the gather stage (MOD instantiations only, sige_tile_conv_t.modulation): gamma / beta are NHWC at the logical
    // source extent with gC / bC elements per pixel, each pointing at the first channel of its window (sige_conv_modulation_t's c0);
    // slope is the leaky-ReLU slope.  The fields take the padding before `trace` and the tail up to the tensor maps' 64-byte-aligned
    // parameter offset, so every other field and both tensor maps keep their offsets.
    float slope;
    long long *trace;          // development aid: per-CTA clock stamps (16 slots), or nullptr
    const void *gamma, *beta;
    int gC, bC;
};

template <int BN, int TAPS, bool DEEP = false, bool S2 = false, bool DB = false> struct Cfg {
    static_assert(!S2 || (BN == 64 && TAPS == 9 && !DEEP), "stride-2 geometry: narrow 3x3 only");
    static constexpr int CT = S2 ? S2_TILES : TILES;           // tiles per CTA
    static constexpr int A_COPY = S2 ? S2_COPY_BYTES : A_COPY_BYTES;
    static constexpr int A_BUF = S2 ? S2_BUF_BYTES : A_BUF_BYTES;
    // DEEP (split-K launches of the narrow 3x3 configuration, with the exchange slots) comes in two layouts of the same size:
    //  * single-buffered (K slices that need one halo fill): ONE halo buffer, and the other 72 KB go to the weight ring —
    //    5 stages = 120 KB in flight, so a slice's weights are on their way before the previous layer has finished;
    //  * double-buffered (DB: K slices that span several chunks): two halo buffers, so the gather of chunk c+1 overlaps
    //    the MMAs of chunk c, and a two-stage ring fed from L2 (the prologue prefetches the whole weight slice into L2).
    static_assert(!DEEP || (BN == 64 && TAPS == 9), "deep ring: narrow 3x3 only");
    static_assert(!DB || DEEP, "double-buffered halo: a split-K layout");
    static constexpr int NAB = ((DEEP && !DB) || S2) ? 1 : 2;
    // one weight-ring stage = TPS taps (a whole kernel row for the narrow 3x3 configuration): fewer barrier round
    // trips for the single MMA-issuing thread
    static constexpr int TPS = (TAPS == 9 && BN == 64) ? 3 : 1;
    static constexpr int SPC = TAPS / TPS;                     // ring steps per 64-channel chunk
    static constexpr int B_TILE_BYTES = BN * 128;              // one (tap, chunk) weight tile
    static constexpr int B_STAGE_BYTES = TPS * B_TILE_BYTES;
    // The narrow 3x3 configuration WITHOUT the deep ring is only launched un-split (decide() gives the deep ring to exactly the
    // split launches), so its split-K exchange slots are never used: their 30 KB hold a third weight stage instead (un-split launches are
    // the ones with long K loops per CTA, i.e. weight-ring bound: 72 KB in flight instead of 48).
    static constexpr bool kUnsplit39 = (BN == 64 && TAPS == 9 && !DEEP && !S2);
    static constexpr int NSTB = S2 ? 3 : DEEP ? (DB ? 2 : 5) : ((BN == 128) ? 4 : (TPS == 3 ? 3 : 4));   // weight ring depth (72 / 48 / 120 / 64 / 72 / 32 KB in flight per CTA)
    static constexpr int EPI_PITCH = BN + EPI_PAD;             // floats
    static constexpr int OFF_A = 0;
    static constexpr int OFF_B = NAB * A_BUF;
    // split-K (BN = 64 only): partial-tile rows pushed by the other ranks of the cluster land here — a region that no
    // mainloop touches, so a fast rank may push while this CTA is still multiplying.  <= 7 remote ranks x 16 rows.
    static constexpr int OFF_SLOT = OFF_B + NSTB * B_STAGE_BYTES;
    static constexpr int SLOT_BYTES = (BN == 64 && !kUnsplit39) ? 112 * EPI_PITCH * 4 : 0;
    static constexpr bool kSplitOk = (BN == 64 && !kUnsplit39);
    static constexpr int OFF_BAR = OFF_SLOT + SLOT_BYTES;
    static constexpr int OFF_CONST = OFF_BAR + 256;            // idx[CT][2] ints + CT shortcut flags, then bias | aux0 scale,shift | aux1 scale,shift | bias2
    static constexpr int OFF_FLAGS = OFF_CONST + CT * 8;
    static constexpr int OFF_VEC = OFF_FLAGS + (CT + 15) / 16 * 16;          // (80 bytes after OFF_CONST for the 8-tile geometries)
    static constexpr int SMEM_BYTES = OFF_VEC + 6 * BN * 4 + 1024;    // + slack for the 1024-byte alignment
    static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB shared-memory limit");
    static_assert(128 * EPI_PITCH * 4 <= NAB * A_BUF, "epilogue staging must fit in the halo buffers");
};

// ------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(bar) : "memory");
}
// wait with cluster-scope acquire: the phase is completed by remote st.async complete_tx operations
__device__ __forceinline__ void mbar_wait_cluster(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAITC_LOOP:\n"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAITC_DONE;\n"
        "bra WAITC_LOOP;\n"
        "WAITC_DONE:\n"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}
// shared::cta address -> the same offset in the shared memory of CTA `rank` of this cluster
__device__ __forceinline__ uint32_t map_rank(uint32_t addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;\n" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
// 8-byte store into a peer's shared memory that reports its bytes to an mbarrier of that peer: the receiver learns
// that the data has landed from its own barrier — no fence and no cluster-wide barrier on the sender's side
__device__ __forceinline__ void st_async8(uint32_t remote_addr, uint32_t a, uint32_t b, uint32_t remote_bar) {
    asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v2.b32 [%0], {%1, %2}, [%3];\n" ::"r"(remote_addr), "r"(a),
                 "r"(b), "r"(remote_bar)
                 : "memory");
}
// 16-byte asynchronous copy global -> shared (LDGSTS): no register staging, so several chunks can be in flight per CTA;
// src_bytes = 0 zero-fills the destination (outside the image / missing tile) without reading
__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src, uint32_t src_bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
// this thread's arrival on `bar` fires once all of its cp.async issued so far have landed (one of the barrier's expected arrivals)
__device__ __forceinline__ void cp_async_arrive(uint32_t bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];\n" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *tmap, int x, int y, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];\n" ::"r"(dst),
        "l"(tmap), "r"(x), "r"(y), "r"(bar)
        : "memory");
}
// pull one TMA box into L2 without a shared-memory destination or a barrier
__device__ __forceinline__ void tma_prefetch_l2_2d(const CUtensorMap *tmap, int x, int y) {
    asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];\n" ::"l"(tmap), "r"(x), "r"(y) : "memory");
}
// wgmma shared-memory descriptor, K-major, 128-byte swizzle (given as (lo, hi) words):
//   [0,14) start address >> 4 | [16,30) leading byte offset >> 4 (= 1, unused for swizzled K-major)
//   [32,46) stride byte offset >> 4 (= 1024 B between 8-row groups) | [49,52) base offset = 0 (all operand bases are
//   1024-byte aligned) | [62,64) layout = 1 (SWIZZLE_128B)
// The issuing warpgroup's instruction stream is the critical path of a latency-bound layer, so per-MMA descriptor
// arithmetic is one 32-bit add on the low word (start address in 16-byte units; every operand base is below 256 KB,
// so the 14-bit field never overflows into its neighbours).
constexpr uint32_t DESC_HI = (1024u >> 4) | (1u << 30);
__device__ __forceinline__ uint32_t desc_lo(uint32_t smem_addr) { return (smem_addr >> 4) | (1u << 16); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs that own those registers
template <int N> __device__ __forceinline__ void fence_acc(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x N] (+)= A[64 x 16] * B[16 x N]; fp32 accumulator fragment of thread t of the warpgroup: d[4i + {0,1}] =
// row 16*(t/32) + (t%32)/4, columns 8i + 2*(t%4) + {0,1}; d[4i + {2,3}] = the same columns, 8 rows further down.
__device__ __forceinline__ void wgmma_m64n64_f16(float (&d)[32], uint32_t a_lo, uint32_t b_lo, uint32_t hi, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        ".reg .b64 da, db;\n"
        "setp.ne.b32 p, %35, 0;\n"
        "mov.b64 da, {%32, %34};\n"
        "mov.b64 db, {%33, %34};\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{" 
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, da, db, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a_lo), "r"(b_lo), "r"(hi), "r"(scale_d)
        : "memory");
}
__device__ __forceinline__ void wgmma_m64n64_bf16(float (&d)[32], uint32_t a_lo, uint32_t b_lo, uint32_t hi, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        ".reg .b64 da, db;\n"
        "setp.ne.b32 p, %35, 0;\n"
        "mov.b64 da, {%32, %34};\n"
        "mov.b64 db, {%33, %34};\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{" 
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, da, db, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a_lo), "r"(b_lo), "r"(hi), "r"(scale_d)
        : "memory");
}
__device__ __forceinline__ void wgmma_m64n128_f16(float (&d)[64], uint32_t a_lo, uint32_t b_lo, uint32_t hi, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        ".reg .b64 da, db;\n"
        "setp.ne.b32 p, %67, 0;\n"
        "mov.b64 da, {%64, %66};\n"
        "mov.b64 db, {%65, %66};\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{" 
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, da, db, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a_lo), "r"(b_lo), "r"(hi), "r"(scale_d)
        : "memory");
}
__device__ __forceinline__ void wgmma_m64n128_bf16(float (&d)[64], uint32_t a_lo, uint32_t b_lo, uint32_t hi, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        ".reg .b64 da, db;\n"
        "setp.ne.b32 p, %67, 0;\n"
        "mov.b64 da, {%64, %66};\n"
        "mov.b64 db, {%65, %66};\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{" 
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, da, db, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a_lo), "r"(b_lo), "r"(hi), "r"(scale_d)
        : "memory");
}

template <typename T, int BN>
__device__ __forceinline__ void wgmma_step(float (&d)[BN / 2], uint32_t a_lo, uint32_t b_lo, uint32_t scale_d) {
    if constexpr (std::is_same<T, __half>::value) {
        if constexpr (BN == 64) wgmma_m64n64_f16(d, a_lo, b_lo, DESC_HI, scale_d); else wgmma_m64n128_f16(d, a_lo, b_lo, DESC_HI, scale_d);
    } else {
        if constexpr (BN == 64) wgmma_m64n64_bf16(d, a_lo, b_lo, DESC_HI, scale_d); else wgmma_m64n128_bf16(d, a_lo, b_lo, DESC_HI, scale_d);
    }
}

// ------------------------------------------------------------------------------------------
// kernel
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ long long gtime() {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;\n" : "=l"(t));
    return t;
}
#define SIGE_TRACE(slot)                                                                                          \
    do {                                                                                                          \
        if (p.trace) p.trace[((blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) * 16 + (slot)] = gtime(); \
    } while (0)

// even split of n ring steps over ks ranks: rank kr takes [k_slice(n, kr, ks), k_slice(n, kr + 1, ks))
__host__ __device__ __forceinline__ int k_slice(int J, int kr, int ks) { return (int)(((long long)J * kr) / ks); }

// K order and partition of a launch.  The ring steps fall into three source groups, each a run of whole 64-channel chunks in the
// natural order: main chunks of src[0], main chunks of src[1], fused-shortcut chunks (src2).  The groups whose bit is set in
// `early` (the SIGE_CONV_EARLY_* flags) come first, then the others, each group keeping its order; rank kr of a split takes an even
// share of the early steps followed by an even share of the late ones, so the work left after the dependency resolves is
// balanced.  early == 0 is the natural order and the even split of k_slice.  The kernel, the halo-layout choice
// (split_halo_fills) and decide() all use this one partition.
struct KOrder {
    int NC, spc, J_main, J;
    int b0, early, E;                                      // b0: ring steps of src[0] (the groups are [0, b0), [b0, J_main), [J_main, J))
    __host__ __device__ KOrder(int Cin, int C0, int Cin2, int spc_, int early_) {
        NC = Cin / KC;
        spc = spc_;
        J_main = NC * spc;
        J = J_main + Cin2 / KC;
        b0 = C0 < Cin ? C0 / KC * spc : J_main;
        early = early_ & 7;
        E = ((early & 1) ? b0 : 0) + ((early & 2) ? J_main - b0 : 0) + ((early & 4) ? J - J_main : 0);
    }
    // ring position q -> step j of the natural order
    __host__ __device__ int step(int q) const {
        const int want = q < E ? 1 : 0;                    // early groups first, then the others
        if (!want) q -= E;
        if (((early >> 0) & 1) == want) { if (q < b0) return q; q -= b0; }
        if (((early >> 1) & 1) == want) { if (q < J_main - b0) return b0 + q; q -= J_main - b0; }
        return J_main + q;
    }
    __host__ __device__ int chunk(int j) const { return j < J_main ? j / spc : NC + (j - J_main); }
};
// The K slice of rank kr: `ne` early ring positions from eb, then the late ones from lb; n in all.  Slice step i sits at ring
// position pos(i).  A chunk's steps are never split between the early and the late part.
struct KSlice {
    int eb, ne, lb, n;
    __host__ __device__ KSlice(const KOrder &o, int kr, int ks) {
        eb = k_slice(o.E, kr, ks);
        ne = k_slice(o.E, kr + 1, ks) - eb;
        lb = o.E + k_slice(o.J - o.E, kr, ks);
        n = ne + (o.E + k_slice(o.J - o.E, kr + 1, ks) - lb);
    }
    __host__ __device__ int pos(int i) const { return i < ne ? eb + i : lb + (i - ne); }
    // halo fills (distinct chunks) of the slice
    __host__ __device__ int fills(const KOrder &o) const {
        int f = 0, prev = -1;
        for (int i = 0; i < n; ++i) {
            const int c = o.chunk(o.step(pos(i)));
            if (c != prev) ++f;
            prev = c;
        }
        return f;
    }
};

// ASYNC: the gather is a pure copy (no pre-op: the producer of the source already applied it) and is done with cp.async.
// DB: the double-buffered split-K layout (Cfg).
// MOD: the register-staged gather applies SPADE's modulation after the pre-op (see Params::gamma); the source is a full tensor.
template <typename T, int BN, int TAPS, bool DEEP, bool ASYNC, bool S2 = false, bool DB = false, bool MOD = false>
__global__ void __launch_bounds__(NTHREADS, 1)
tile_conv_tc5_kernel(const __grid_constant__ Params p, const __grid_constant__ CUtensorMap wmap,
                     const __grid_constant__ CUtensorMap wmap2) {
    using C = Cfg<BN, TAPS, DEEP, S2, DB>;
    static_assert(!S2 || ASYNC, "stride-2 geometry: pure-copy (cp.async) gather only");
    static_assert(!MOD || !ASYNC, "modulated gather: register-staged only");
    constexpr int NSTB = C::NSTB, TPS = C::TPS, SPC = C::SPC, NAB = C::NAB;
    constexpr int TILES = C::CT;                      // (shadows the namespace constant: 32 for the stride-2 geometry)
    constexpr int A_COPY_BYTES = C::A_COPY, A_BUF_BYTES = C::A_BUF;
    constexpr int R = (TAPS == 9) ? (S2 ? 5 : 6) : 4; // halo tile extent
    constexpr int RS = R * R;
    constexpr int UNITS = TILES * RS * 8;             // 16-byte units gathered per chunk
    constexpr int LOADS = (UNITS + NPROD - 1) / NPROD;

    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const uint32_t sbase = smem_u32(smem);
    const uint32_t bar0 = sbase + C::OFF_BAR;
    // barrier layout (8 bytes each): b_full[NSTB] | b_empty[NSTB] | a_full[2] | a_empty[2] | red_full
    auto B_FULL = [&](int s) { return bar0 + 8 * s; };
    auto B_EMPTY = [&](int s) { return bar0 + 8 * (NSTB + s); };
    auto A_FULL = [&](int b) { return bar0 + 8 * (2 * NSTB + b); };
    auto A_EMPTY = [&](int b) { return bar0 + 8 * (2 * NSTB + 2 + b); };
    const uint32_t RED_FULL = bar0 + 8 * (2 * NSTB + 4);     // split-K: all partial rows of the other ranks have landed
    static_assert(8 * (2 * NSTB + 5) <= 256, "barrier block");

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tile0 = blockIdx.x * TILES;
    // fixed-capacity tile lists (one per image): real tiles are packed at the front, the rest are SIGE_TILE_NONE.  A CTA (and with it
    // its whole split-K cluster: same tile0) whose first tile is padding has nothing to read or write.
    // Early chunks (p.early) read buffers that the preceding launch does not write, before griddepcontrol.wait.  That is sound
    // because every CTA of every launch waits before it releases its dependents and before it exits (here, in the producers and
    // at the epilogue): when this launch starts, every CTA of the preceding launch has passed its wait, so the launch before that
    // has completed and its writes are visible — and no launch completes before its own predecessor, so all earlier ones have too.
    if (p.padded && __ldg(p.idx + 2 * tile0) <= SIGE_TILE_NONE) {
        if (p.pdl) pdl_acquire();
        return;
    }
    const int n0 = blockIdx.y * BN;
    const int ntile = min(TILES, p.NT - tile0);
    const int NC = p.Cin / KC;
    const int J_main = NC * SPC;                   // ring steps of the main conv (a step = TPS taps of one 64-channel chunk)
    const int kr = blockIdx.z;
    // halo-buffer chunks: main chunks 0..NC-1, then fused 1x1 shortcut chunks NC..NC+NC2-1 (one step, the centre tap, per chunk
    // of ITS input); this rank's steps in processing order: ko.step(ks.pos(i)), i < ks.n
    const KOrder ko(p.Cin, p.C0, (TAPS == 9 && !S2) ? p.Cin2 : 0, SPC, S2 ? 0 : p.early);
    const KSlice ks(ko, kr, p.ksplit);
    auto chunk_of = [&](int j) { return j < J_main ? j / SPC : NC + (j - J_main); };
    auto step_at = [&](int i) { return ko.step(ks.pos(i)); };
    // slice step i (step j) starts a chunk: the step after the last one of that chunk in this slice (or ks.n)
    auto chunk_end = [&](int i, int j) {
        const int rest = j < J_main ? SPC - (j - (j / SPC) * SPC) : 1;
        return min(i + rest, i < ks.ne ? ks.ne : ks.n);
    };
    if (tid == 0 && p.trace) p.trace[((blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) * 16 + 12] = ks.fills(ko);   // halo fills
    int32_t *s_idx = reinterpret_cast<int32_t *>(smem + C::OFF_CONST);          // [TILES][2] tile origins of this CTA
    unsigned char *s_flags = smem + C::OFF_FLAGS;                               // [TILES] 1 = evaluate the fused shortcut on this tile
    float *s_const = reinterpret_cast<float *>(smem + C::OFF_VEC);              // bias | aux0 scale | aux0 shift | aux1 scale | aux1 shift | bias2

    if (tid == 0) SIGE_TRACE(0);
    // ---------------- one-time setup ----------------
    if (warp == 0) {
        if (lane == 0) {
            asm volatile("prefetch.tensormap [%0];\n" ::"l"(&wmap) : "memory");
            for (int s = 0; s < NSTB; ++s) { mbar_init(B_FULL(s), 1); mbar_init(B_EMPTY(s), NCONS_WARPS); }
            for (int b = 0; b < 2; ++b) { mbar_init(A_FULL(b), NPROD); mbar_init(A_EMPTY(b), NCONS_WARPS); }
            mbar_init(RED_FULL, 1);
            fence_barrier_init();
        }
    } else if (warp == 2) {
        // this CTA's tile origins (constant since set_masks): one global round trip here instead of one per gather thread
        if (S2) {
            for (int e = lane; e < 2 * TILES; e += 32) {
                const int t = tile0 + (e >> 1);
                s_idx[e] = (t < p.NT && p.idx) ? __ldg(p.idx + 2 * (p.idx_per_image ? t : t % p.N) + (e & 1)) : 0;
            }
            s_flags[lane] = 0;                        // (no fused shortcut in this geometry)
        } else if (lane < 2 * TILES) {
            const int t = tile0 + (lane >> 1);
            int v = 0;
            if (t < p.NT && p.idx) v = __ldg(p.idx + 2 * (p.idx_per_image ? t : t % p.N) + (lane & 1));
            s_idx[lane] = v;
        } else if (lane < 2 * TILES + TILES) {
            const int tl = lane - 2 * TILES, t = tile0 + tl;
            s_flags[tl] = (p.Cin2 > 0 && t < p.NT && (p.sc_flags == nullptr || __ldg(p.sc_flags + (p.idx_per_image ? t : t % p.N)))) ? 1 : 0;
        }
    } else if (warp >= 3 && warp < 9) {
        // per-channel epilogue constants of this CTA's BN output channels
        const int which = warp - 3;                         // 0 bias, 1/2 aux0 scale/shift, 3/4 aux1 scale/shift, 5 bias2
        const float *src = which == 0 ? p.bias : (which == 1 ? p.aux[0].scale : which == 2 ? p.aux[0].shift : which == 3 ? p.aux[1].scale : which == 4 ? p.aux[1].shift : p.bias2);
        const bool on = which == 0 || which == 5 || (which <= 2 ? p.n_aux > 0 : p.n_aux > 1);
        const float dflt = (which == 1 || which == 3) ? 1.f : 0.f;
        for (int e = lane; e < BN; e += 32) s_const[which * BN + e] = (on && src && n0 + e < p.Cout) ? __ldg(src + n0 + e) : dflt;
    }
    __syncthreads();
    if (p.ksplit > 1) {
        // the receiver's side of the split-K exchange: (ksplit - 1) peers x its share of rows x BN floats will arrive
        if (tid == 0) mbar_expect_tx(RED_FULL, (uint32_t)(p.ksplit - 1) * (128 / p.ksplit) * BN * 4);
        cg::this_cluster().barrier_arrive();                 // every thread; matched by barrier_wait() before the first remote store
    }
    if (tid == 0) SIGE_TRACE(1);

    auto tl_of = [&](int m) { return S2 ? (m >> 1) & 31 : (TAPS == 9 ? (m >> 2) & 7 : m >> 4); };
    // GEMM row m -> destination pixel index, or -1 (row of a tile that does not exist / outside the image)
    auto pixel_of = [&](int m) -> long long {
        int tl, oy, ox;
        if (S2) { oy = m >> 6; tl = (m >> 1) & 31; ox = m & 1; }
        else if (TAPS == 9) { oy = m >> 5; tl = (m >> 2) & 7; ox = m & 3; } else { tl = m >> 4; oy = (m >> 2) & 3; ox = m & 3; }
        if (tl >= ntile) return -1;
        const int t = tile0 + tl;
        int hh = oy, ww = ox, img = t;
        if (!p.dst_is_stack) {
            img = 0;
            if (p.NT != p.N) img = t / p.N;
            if (S2) {       // output origin = (offset + tile origin) / stride, C division (reference sige/cuda/scatter_kernel.cu:24-25)
                hh += (p.offH + s_idx[2 * tl]) / 2;
                ww += (p.offW + s_idx[2 * tl + 1]) / 2;
            } else {
                hh += p.offH + s_idx[2 * tl];
                ww += p.offW + s_idx[2 * tl + 1];
            }
        } else if (p.idx && s_idx[2 * tl] <= SIGE_TILE_NONE) {
            return -1;                                 // a padding entry of the list writes nothing to its stack row
        }
        if (hh < 0 || hh >= p.dH || ww < 0 || ww >= p.dW) return -1;
        return ((long long)img * p.dH + hh) * p.dW + ww;
    };

    float acc[BN / 2];                                 // consumers: this thread's share of its warpgroup's 64 x BN accumulator
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;

    if (warp == TMA_WARP) {
        // ================= TMA producer: weights =================
        if (lane == 0) {
            int s = 0, k = 0;                                          // ring stage and lap
            for (int i = 0; i < ks.n; ++i) {
                const int j = step_at(i);
                if (DB && i == NSTB) {
                    // the ring is full: pull the rest of the slice into L2 now (this overlaps the previous layer under PDL),
                    // so that a two-stage ring refills from L2 rather than HBM
                    for (int ii = i; ii < ks.n; ++ii) {
                        const int jj = step_at(ii);
                        if (jj < J_main) {
                            const int cj = jj / SPC, row0 = ((jj - cj * SPC) * TPS * NC + cj) * p.Cout + n0;
#pragma unroll
                            for (int t = 0; t < TPS; ++t) tma_prefetch_l2_2d(&wmap, 0, row0 + t * NC * p.Cout);
                        } else {
                            tma_prefetch_l2_2d(&wmap2, 0, (jj - J_main) * p.Cout + n0);
                        }
                    }
                }
                mbar_wait(B_EMPTY(s), (k & 1) ^ 1);
                const uint32_t dst = sbase + C::OFF_B + s * C::B_STAGE_BYTES;
                if (j < J_main) {
                    mbar_expect_tx(B_FULL(s), C::B_STAGE_BYTES);
                    const int c = j / SPC, st = j - c * SPC;
                    const int row0 = (st * TPS * NC + c) * p.Cout + n0;      // weight rows of tap st*TPS, chunk c
#pragma unroll
                    for (int t = 0; t < TPS; ++t) tma_load_2d(dst + t * C::B_TILE_BYTES, &wmap, 0, row0 + t * NC * p.Cout, B_FULL(s));
                } else {                                               // shortcut weights [Cin2/64][Cout][64]
                    mbar_expect_tx(B_FULL(s), C::B_TILE_BYTES);
                    tma_load_2d(dst, &wmap2, 0, (j - J_main) * p.Cout + n0, B_FULL(s));
                }
                if (++s == NSTB) { s = 0; ++k; }
            }
        }
        __syncwarp();
    } else if (warp < NCONS_WARPS) {
        // ================= MMA consumers: warpgroup wg multiplies GEMM rows 64*wg .. 64*wg+63 =================
        // Descriptor low words are advanced by compile-time constants from per-step bases.  A step's MMAs are one
        // commit group; the weight stage of step j is released once step j+1 has been issued and step j has retired
        // (wait_group 1), so that the tensor core always has the next step queued.  At the end of a chunk everything
        // retires (wait_group 0) before its halo buffer is released: with a single halo buffer the producers cannot
        // start the next chunk earlier; with two they are already filling the other one.
        const int wg = warp >> 2;
        const uint32_t a_lo0 = desc_lo(sbase + C::OFF_A + wg * (64 * 128)), b_lo0 = desc_lo(sbase + C::OFF_B);
        uint32_t accum = 0;
        int ab = 0, ause = 0;             // halo buffer index and how many times it has been used
        int s = 0, k = 0;
        int pend = -1;                    // weight stage of the previous step, not yet released
        for (int i = 0; i < ks.n; ++i) {
            const int j = step_at(i);
            const bool is_sc = j >= J_main;
            const int st = is_sc ? 0 : j - (j / SPC) * SPC;
            if (i == 0 || i == ks.ne || st == 0) {                // a new chunk starts: wait for its halo buffer
                mbar_wait(A_FULL(ab), (ause / NAB) & 1);
                fence_proxy_async();          // gathered data (generic proxy writes) -> visible to the tensor core's async proxy
                if (i == 0 && tid == 0) SIGE_TRACE(5);
            }
            mbar_wait(B_FULL(s), k & 1);
            const uint32_t b_step = b_lo0 + s * (C::B_STAGE_BYTES >> 4);
            uint32_t a_step = a_lo0 + ab * (A_BUF_BYTES >> 4);
            if (S2) {
                a_step += (st == 0 ? 0 : (st == 1 ? 3 : 1)) * ((64 * 128) >> 4);               // ky = st: planes {0,2,4 | 1,3} start at {0, 3, 1}
            } else if (TAPS == 9) {
                if (is_sc) a_step += (A_COPY_BYTES + 32 * 128) >> 4;                           // tap (1,1)
                else if (TPS == 3) a_step += st * ((32 * 128) >> 4);                           // ky = st, kx = t
                else { const int ky = st / 3; a_step += ky * ((32 * 128) >> 4) + (st - 3 * ky) * (A_COPY_BYTES >> 4); }
            }
            const bool chunk_done = is_sc || st == SPC - 1 || i == ks.n - 1 || i == ks.ne - 1;
            fence_acc(acc);
            wgmma_fence();
#pragma unroll
            for (int t = 0; t < TPS; ++t) {
                if (is_sc && t > 0) break;                    // the shortcut is a single tap: the centre of the 3x3 frame
#pragma unroll
                for (int kk = 0; kk < KC / 16; ++kk)
                    wgmma_step<T, BN>(acc, a_step + t * (A_COPY_BYTES >> 4) + kk * 2, b_step + t * (C::B_TILE_BYTES >> 4) + kk * 2,
                                      (accum | t | kk) ? 1u : 0u);
            }
            wgmma_commit();
            if (chunk_done) {
                wgmma_wait<0>();
                if (lane == 0) {
                    if (pend >= 0) mbar_arrive(B_EMPTY(pend));
                    mbar_arrive(B_EMPTY(s));                          // weight stage free
                    mbar_arrive(A_EMPTY(ab));                         // halo buffer free
                }
                pend = -1;
            } else {
                wgmma_wait<1>();
                if (lane == 0 && pend >= 0) mbar_arrive(B_EMPTY(pend));
                pend = s;
            }
            fence_acc(acc);
            __syncwarp();
            accum = 1;
            if (chunk_done) { ++ause; ab = ause % NAB; }
            if (++s == NSTB) { s = 0; ++k; }
        }
        wgmma_wait<0>();
        fence_acc(acc);
        if (tid == 0) SIGE_TRACE(6);
    } else {
        // ================= A-operand producers: gather + pre-op + swizzled stores =================
        const int ptid = tid - NCONS;
        // griddepcontrol.wait right before the first late chunk's gather (slice step ks.ne), or after the last chunk when the whole
        // slice is early (see the invariant at the padding exit); slot 13 = the early chunks are gathered, slot 3 = the dependency
        // has resolved
        auto acquire = [&]() {
            if (ptid == 0 && ks.ne > 0) SIGE_TRACE(13);
            if (p.pdl) {
                pdl_acquire();
                if (p.early_release) pdl_release();
            }
            if (ptid == 0) SIGE_TRACE(3);
        };
        if constexpr (S2) {
            // ---- stride-2 geometry: 32 tiles x 5x5 halo pixels x 8 units = 6400 sixteen-byte copies per chunk, pure copy with
            //      cp.async straight into the plane layout described at S2_TILES.  Thread -> (tile = ptid / 8, unit = ptid % 8), and
            //      it walks the 25 pixels of ITS tile: pixel coordinates, planes and destination rows are compile-time constants of
            //      the unrolled loop, per-thread state is the tile origin and two swizzled row offsets.  (A first version kept 25
            //      resolved source offsets per thread: 92 bytes spilled, re-read through a ~20 KB L1 that the gather itself
            //      thrashes.)
            static_assert(NPROD == S2_TILES * 8 && UNITS == NPROD * RS, "one (tile, unit) per producer thread");
            const int tl = ptid >> 3, u = ptid & 7;
            const int t = tile0 + tl;
            const bool live = t < p.NT;
            int hh0 = 0, ww0 = 0, img = t;
            if (!p.src_is_stack) {
                hh0 = s_idx[2 * tl];
                ww0 = s_idx[2 * tl + 1];
                img = (p.NT != p.N) ? t / p.N : 0;
            }
            // destination of (plane 0, ox): row = tile*2 + ox, 16-byte chunk u XOR-swizzled by the row
            const uint32_t d_ox0 = sbase + C::OFF_A + (tl * 2) * 128 + ((u ^ ((tl * 2) & 7)) << 4);
            const uint32_t d_ox1 = sbase + C::OFF_A + (tl * 2 + 1) * 128 + ((u ^ ((tl * 2 + 1) & 7)) << 4);
            if (ptid == 0) SIGE_TRACE(2);
            int ause = 0;
            for (int i = 0, next; i < ks.n; i = next) {                   // (no fused shortcut, no early chunks: KOrder)
                const int j = step_at(i), c = chunk_of(j);
                next = chunk_end(i, j);
                if (i == 0) acquire();                                    // activations of the previous layer are complete
                mbar_wait(A_EMPTY(0), (ause & 1) ^ 1);                    // the MMAs that read the (single) halo buffer have retired
                const int cbase = c * KC;
                const int sg = cbase >= p.C0 ? 1 : 0;
                const Seg &seg = p.seg[sg];
                const int Hs = p.H >> seg.up, Ws = p.W >> seg.up;
                const T *sbase_p = reinterpret_cast<const T *>(seg.ptr) + (cbase - (sg ? p.C0 : 0)) + u * 8;
#pragma unroll
                for (int y = 0; y < R; ++y) {
                    const int hh = hh0 + y;
                    const bool row_ok = live && hh >= 0 && hh < p.H;
                    const long long rbase = ((long long)img * Hs + (hh >> seg.up)) * Ws;
                    const int plane = (y & 1) ? 3 + (y >> 1) : (y >> 1);
#pragma unroll
                    for (int x = 0; x < R; ++x) {
                        const int ww = ww0 + x;
                        const bool ok = row_ok && ww >= 0 && ww < p.W;
                        const T *src = ok ? sbase_p + (rbase + (ww >> seg.up)) * seg.pitch : reinterpret_cast<const T *>(seg.ptr);
                        const uint32_t nb = ok ? 16u : 0u;
#pragma unroll
                        for (int kx = 0; kx < 3; ++kx) {
                            const int xp = x - kx;
                            if (xp == 0 || xp == 2) cp_async16((xp == 0 ? d_ox0 : d_ox1) + kx * A_COPY_BYTES + plane * (64 * 128), src, nb);
                        }
                    }
                }
                cp_async_arrive(A_FULL(0));
                if (ptid == 0 && i == 0) SIGE_TRACE(4);
                ++ause;
            }
            if (ks.n == 0) acquire();
        } else {
        // per-thread gather list (fixed for the whole kernel)
        int g_xyt[LOADS];     // x | y << 4 | tile << 8 of the halo pixel this load feeds
        int g_off[LOADS];     // element offset of its 16-byte unit in the CURRENT source segment (channel-chunk offset
                              // excluded), -1 = zero fill (outside the image / missing tile), -2 = nothing to do.  The
                              // address arithmetic is done here, in the prologue that overlaps the previous layer, so that
                              // after griddepcontrol.wait a load is one add away; it is redone if the K slice crosses into
                              // the second (concatenated) source.
        int g_sg = -1;
        auto resolve = [&](int sg) {
            const Seg &seg = p.seg[sg];
            const int Hs = p.H >> seg.up, Ws = p.W >> seg.up;
#pragma unroll
            for (int k = 0; k < LOADS; ++k) {
                const int q = ptid + k * NPROD;
                g_off[k] = -2;
                if (q < UNITS) {
                    g_off[k] = -1;
                    const int x = g_xyt[k] & 15, y = (g_xyt[k] >> 4) & 15, tl = g_xyt[k] >> 8;
                    const int t = tile0 + tl;
                    if (t < p.NT) {
                        int hh = y, ww = x, img = t;
                        if (!p.src_is_stack) {
                            hh += s_idx[2 * tl];
                            ww += s_idx[2 * tl + 1];
                            img = (p.NT != p.N) ? t / p.N : 0;          // batch > 1 only (SD); DDPM is batch 1
                        }
                        if (hh >= 0 && hh < p.H && ww >= 0 && ww < p.W)
                            g_off[k] = ((img * Hs + (hh >> seg.up)) * Ws + (ww >> seg.up)) * seg.pitch + (q & 7) * 8;
                    }
                }
            }
            g_sg = sg;
        };
#pragma unroll
        for (int k = 0; k < LOADS; ++k) {
            const int pix = (ptid + k * NPROD) >> 3;
            const int tl = pix / RS, rem = pix - tl * RS;
            const int y = rem / R, x = rem - y * R;
            g_xyt[k] = x | (y << 4) | (tl << 8);
        }
        const int c_first = ks.n > 0 ? chunk_of(step_at(0)) : 0;
        resolve(c_first < NC && c_first * KC >= p.C0 ? 1 : 0);
        if (ptid == 0) SIGE_TRACE(2);   // bookkeeping (idx loads) done
        uint4 regs[LOADS];
        auto issue = [&](int c) {
            const int cbase = c * KC;
            const int sg = cbase >= p.C0 ? 1 : 0;
            const Seg &seg = p.seg[sg];
            const int cl = cbase - (sg ? p.C0 : 0);
            if (sg != g_sg) resolve(sg);
#pragma unroll
            for (int k = 0; k < LOADS; ++k) {
                regs[k] = make_uint4(0, 0, 0, 0);
                if (g_off[k] >= 0) {
                    const T *src = reinterpret_cast<const T *>(seg.ptr) + g_off[k] + cl;
                    regs[k] = __ldg(reinterpret_cast<const uint4 *>(src));
                }
            }
        };
        const bool pre = MOD || (p.scale != nullptr) || (p.shift != nullptr) || (p.act != SIGE_ACT_IDENTITY);
        auto store = [&](int c, unsigned char *abuf) {
#pragma unroll
            for (int k = 0; k < LOADS; ++k) {
                if (g_off[k] == -2) continue;
                uint4 v = regs[k];
                const int u = (ptid + k * NPROD) & 7;
                if (pre && g_off[k] >= 0) {
                    const int ab_k = (p.NT != p.N) ? (tile0 + (g_xyt[k] >> 8)) / p.N : 0;      // batch index (batch > 1: SD only)
                    const int ch = c * KC + u * 8;
                    T *e = reinterpret_cast<T *>(&v);
                    float sc[8], sh[8];
#pragma unroll
                    for (int z = 0; z < 8; ++z) { sc[z] = 1.f; sh[z] = 0.f; }
                    if (p.scale) {
                        const float4 *s4 = reinterpret_cast<const float4 *>(p.scale + (long long)ab_k * p.affine_bstride + ch);
                        const float4 a = __ldg(s4), b = __ldg(s4 + 1);
                        sc[0] = a.x; sc[1] = a.y; sc[2] = a.z; sc[3] = a.w; sc[4] = b.x; sc[5] = b.y; sc[6] = b.z; sc[7] = b.w;
                    }
                    if (p.shift) {
                        const float4 *s4 = reinterpret_cast<const float4 *>(p.shift + (long long)ab_k * p.affine_bstride + ch);
                        const float4 a = __ldg(s4), b = __ldg(s4 + 1);
                        sh[0] = a.x; sh[1] = a.y; sh[2] = a.z; sh[3] = a.w; sh[4] = b.x; sh[5] = b.y; sh[6] = b.z; sh[7] = b.w;
                    }
                    if constexpr (MOD) {
                        // leaky((x*scale + shift) * (1 + gamma) + beta) at the halo pixel's LOGICAL coordinates (the source may be read
                        // up-sampled), rounded once: the expression and order of the mma.sync MOD path, so the staged operand is the same
                        const int tl = g_xyt[k] >> 8;
                        const long long px = ((long long)ab_k * p.H + (((g_xyt[k] >> 4) & 15) + s_idx[2 * tl])) * p.W + ((g_xyt[k] & 15) + s_idx[2 * tl + 1]);
                        const uint4 gr = __ldg(reinterpret_cast<const uint4 *>(reinterpret_cast<const T *>(p.gamma) + px * p.gC + ch));
                        const uint4 br = __ldg(reinterpret_cast<const uint4 *>(reinterpret_cast<const T *>(p.beta) + px * p.bC + ch));
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
                const int x = g_xyt[k] & 15, y = (g_xyt[k] >> 4) & 15, tl = g_xyt[k] >> 8;
                if (TAPS == 9) {
#pragma unroll
                    for (int kx = 0; kx < 3; ++kx) {
                        const int xp = x - kx;
                        if (xp >= 0 && xp < 4) {
                            const int row = y * 32 + tl * 4 + xp;
                            *reinterpret_cast<uint4 *>(abuf + kx * A_COPY_BYTES + row * 128 + ((u ^ (row & 7)) << 4)) = v;
                        }
                    }
                } else {
                    const int row = tl * 16 + y * 4 + x;
                    *reinterpret_cast<uint4 *>(abuf + row * 128 + ((u ^ (row & 7)) << 4)) = v;
                }
            }
        };
        // fused shortcut chunks: only the 4x4 centre of each halo tile is needed (tap (1,1)), from the RAW block input,
        // into copy kx = 1 at rows y*32 + tile*4 + (x-1); tiles whose shortcut is not active contribute zeros
        constexpr int LOADS2 = (TILES * 16 * 8 + NPROD - 1) / NPROD;
        auto issue2 = [&](int c2) {
            const int cbase = c2 * KC;
            const int sg = cbase >= p.C0_2 ? 1 : 0;
            const Seg &seg = p.seg2[sg];
            const int cl = cbase - (sg ? p.C0_2 : 0);
            const int Hs = p.H >> seg.up, Ws = p.W >> seg.up;
#pragma unroll
            for (int k = 0; k < LOADS2; ++k) {
                const int q = ptid + k * NPROD;
                regs[k] = make_uint4(0, 0, 0, 0);
                const int pix = q >> 3, u = q & 7;
                const int tl = pix >> 4, rem = pix & 15;
                const int y = 1 + (rem >> 2), xx = 1 + (rem & 3);
                const int t = tile0 + tl;
                if (q < TILES * 16 * 8 && t < p.NT && s_flags[tl]) {
                    int b = 0;
                    if (p.NT != p.N) b = t / p.N;
                    const int hh = y + s_idx[2 * tl], ww = xx + s_idx[2 * tl + 1];
                    if (hh >= 0 && hh < p.H && ww >= 0 && ww < p.W) {
                        const T *src = reinterpret_cast<const T *>(seg.ptr) + (((long long)b * Hs + (hh >> seg.up)) * Ws + (ww >> seg.up)) * seg.pitch + cl + u * 8;
                        regs[k] = __ldg(reinterpret_cast<const uint4 *>(src));
                    }
                }
            }
        };
        auto store2 = [&](unsigned char *abuf) {
#pragma unroll
            for (int k = 0; k < LOADS2; ++k) {
                const int q = ptid + k * NPROD;
                if (q >= TILES * 16 * 8) continue;
                const int pix = q >> 3, u = q & 7;
                const int tl = pix >> 4, rem = pix & 15;
                const int row = (1 + (rem >> 2)) * 32 + tl * 4 + (rem & 3);
                *reinterpret_cast<uint4 *>(abuf + A_COPY_BYTES + row * 128 + ((u ^ (row & 7)) << 4)) = regs[k];
            }
        };
        auto issue_any = [&](int c) { if (c < NC) issue(c); else issue2(c - NC); };
        if (ASYNC) {
            // ---- pure-copy gather with cp.async: every unit goes straight from global/L2 to its (up to three) swizzled
            //      destinations; the thread's arrival on A_FULL fires when its copies have landed, so the producer never
            //      waits for data and keeps NAB chunks in flight (register staging kept exactly one in flight)
            auto copy_chunk = [&](int c, unsigned char *abuf, uint32_t full_bar) {
                const uint32_t abase = smem_u32(abuf);
                if (c < NC) {
                    const int cbase = c * KC;
                    const int sg = cbase >= p.C0 ? 1 : 0;
                    const Seg &seg = p.seg[sg];
                    const int cl = cbase - (sg ? p.C0 : 0);
                    if (sg != g_sg) resolve(sg);
#pragma unroll
                    for (int k = 0; k < LOADS; ++k) {
                        if (g_off[k] == -2) continue;
                        const bool ok = g_off[k] >= 0;
                        const T *src = reinterpret_cast<const T *>(seg.ptr) + (ok ? g_off[k] + cl : 0);
                        const uint32_t nb = ok ? 16u : 0u;
                        const int u = (ptid + k * NPROD) & 7;
                        const int x = g_xyt[k] & 15, y = (g_xyt[k] >> 4) & 15, tl = g_xyt[k] >> 8;
                        if (TAPS == 9) {
#pragma unroll
                            for (int kx = 0; kx < 3; ++kx) {
                                const int xp = x - kx;
                                if (xp >= 0 && xp < 4) {
                                    const int row = y * 32 + tl * 4 + xp;
                                    cp_async16(abase + kx * A_COPY_BYTES + row * 128 + ((u ^ (row & 7)) << 4), src, nb);
                                }
                            }
                        } else {
                            const int row = tl * 16 + y * 4 + x;
                            cp_async16(abase + row * 128 + ((u ^ (row & 7)) << 4), src, nb);
                        }
                    }
                } else {
                    // fused shortcut chunk: the 4x4 centre of each halo tile from the RAW block input into copy kx = 1
                    const int cbase = (c - NC) * KC;
                    const int sg = cbase >= p.C0_2 ? 1 : 0;
                    const Seg &seg = p.seg2[sg];
                    const int cl = cbase - (sg ? p.C0_2 : 0);
                    const int Hs = p.H >> seg.up, Ws = p.W >> seg.up;
#pragma unroll
                    for (int k = 0; k < LOADS2; ++k) {
                        const int q = ptid + k * NPROD;
                        if (q >= TILES * 16 * 8) continue;
                        const int pix = q >> 3, u = q & 7;
                        const int tl = pix >> 4, rem = pix & 15;
                        const int y = 1 + (rem >> 2), xx = 1 + (rem & 3);
                        const int t = tile0 + tl;
                        const T *src = reinterpret_cast<const T *>(seg.ptr);
                        uint32_t nb = 0;
                        if (t < p.NT && s_flags[tl]) {
                            int b = 0;
                            if (p.NT != p.N) b = t / p.N;
                            const int hh = y + s_idx[2 * tl], ww = xx + s_idx[2 * tl + 1];
                            if (hh >= 0 && hh < p.H && ww >= 0 && ww < p.W) {
                                src += (((long long)b * Hs + (hh >> seg.up)) * Ws + (ww >> seg.up)) * seg.pitch + cl + u * 8;
                                nb = 16;
                            }
                        }
                        const int row = (1 + (rem >> 2)) * 32 + tl * 4 + (rem & 3);
                        cp_async16(abase + A_COPY_BYTES + row * 128 + ((u ^ (row & 7)) << 4), src, nb);
                    }
                }
                cp_async_arrive(full_bar);
            };
            int ab = 0, ause = 0;
            for (int i = 0, next; i < ks.n; i = next) {
                const int j = step_at(i), c = chunk_of(j);
                next = chunk_end(i, j);
                if (i == ks.ne) acquire();                                // activations of the previous layer are complete
                mbar_wait(A_EMPTY(ab), ((ause / NAB) & 1) ^ 1);           // the MMAs that read this buffer have retired
                copy_chunk(c, smem + C::OFF_A + ab * A_BUF_BYTES, A_FULL(ab));
                if (ptid == 0 && i == 0) SIGE_TRACE(4);
                ++ause;
                ab = ause % NAB;
            }
            if (ks.ne == ks.n) acquire();
        } else {
        if (ks.n > 0) {
            if (ks.ne == 0) acquire();                                // activations of the previous layer are complete
            issue_any(c_first);
        }
        int ab = 0, ause = 0;
        for (int i = 0; i < ks.n;) {
            const int j = step_at(i), c = chunk_of(j), next = chunk_end(i, j);
            mbar_wait(A_EMPTY(ab), ((ause / NAB) & 1) ^ 1);           // the MMAs that read this buffer have retired
            if (c < NC) store(c, smem + C::OFF_A + ab * A_BUF_BYTES); else store2(smem + C::OFF_A + ab * A_BUF_BYTES);
            if (ptid == 0 && i == 0) SIGE_TRACE(4);
            fence_proxy_async();                                      // generic-proxy stores -> visible to the tensor core
            mbar_arrive(A_FULL(ab));
            if (next < ks.n) {
                if (next == ks.ne) acquire();
                issue_any(chunk_of(step_at(next)));
            }
            i = next;
            ++ause;
            ab = ause % NAB;
        }
        if (ks.ne == ks.n) acquire();
        }
        }   // !S2
    }

    // ---------------- epilogue ----------------
    // the next layer's prologue may overlap this epilogue.  A thread waits before it releases: the first release of a CTA is what
    // counts, and the weight-loading warp can get here before the producers' wait has returned.
    if (p.pdl) {
        pdl_acquire();
        pdl_release();
    }
    float *cst = reinterpret_cast<float *>(smem + C::OFF_A);
    // v[8] (fp32 conv result of 8 consecutive channels starting at n) -> +bias, +residual -> dst and aux destinations
    auto emit = [&](long long pixel, int tl, int n, float (&v)[8]) {
        const int nl = n - n0;
        {
            const float4 b0 = *reinterpret_cast<const float4 *>(s_const + nl), b1 = *reinterpret_cast<const float4 *>(s_const + nl + 4);
            v[0] += b0.x; v[1] += b0.y; v[2] += b0.z; v[3] += b0.w; v[4] += b1.x; v[5] += b1.y; v[6] += b1.z; v[7] += b1.w;
        }
        const bool fresh_sc = s_flags[tl] != 0;       // the fused 1x1 shortcut was evaluated on this tile
        if (fresh_sc) {
            const float4 b0 = *reinterpret_cast<const float4 *>(s_const + 5 * BN + nl), b1 = *reinterpret_cast<const float4 *>(s_const + 5 * BN + nl + 4);
            v[0] += b0.x; v[1] += b0.y; v[2] += b0.z; v[3] += b0.w; v[4] += b1.x; v[5] += b1.y; v[6] += b1.z; v[7] += b1.w;
        } else if (p.residual) {                       // plain residual, or the CACHED shortcut where the fused one is inactive
            const uint4 rr = __ldg(reinterpret_cast<const uint4 *>(reinterpret_cast<const T *>(p.residual) + pixel * p.rC + p.res_c0 + n));
            const T *re = reinterpret_cast<const T *>(&rr);
#pragma unroll
            for (int z = 0; z < 8; ++z) v[z] += DT<T>::to_f(re[z]);
        }
        if (p.dst) {
            uint4 o;
            T *oe = reinterpret_cast<T *>(&o);
#pragma unroll
            for (int z = 0; z < 8; ++z) oe[z] = DT<T>::from_f(v[z]);
            *reinterpret_cast<uint4 *>(reinterpret_cast<T *>(p.dst) + pixel * p.dC + p.dst_c0 + n) = o;
        }
        for (int ax = 0; ax < p.n_aux; ++ax) {   // extra destinations: the consumer's pre-op applied by the producer
            const AuxDst &A = p.aux[ax];
            const float *sc = s_const + (1 + 2 * ax) * BN + nl, *sh = sc + BN;      // staged (scale defaults to 1, shift to 0)
            uint4 oa;
            T *ae = reinterpret_cast<T *>(&oa);
#pragma unroll
            for (int z = 0; z < 8; ++z) ae[z] = DT<T>::from_f(activate<true>(A.act, fmaf(v[z], sc[z], sh[z])));
            *reinterpret_cast<uint4 *>(reinterpret_cast<T *>(A.ptr) + pixel * A.C + A.c0 + n) = oa;
        }
    };
    // accumulator fragment (see wgmma_m64n64_f16): element 4i + h of consumer thread `tid` is GEMM row frag_row(i, h),
    // columns frag_col(i) + {0, 1} (h = 0: d[4i], d[4i+1]; h = 1: d[4i+2], d[4i+3])
    const int frag_m = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2), frag_n = 2 * (lane & 3);
    // the staging area (the halo buffers) is free once both warpgroups' MMAs have retired
    if (warp < NCONS_WARPS) asm volatile("bar.sync 1, %0;\n" ::"n"(NCONS) : "memory");

    if (p.ksplit == 1) {
        // ---- no split-K: registers -> shared staging [128][EPI_PITCH] -> global, a thread per (row, 8 channels): one
        //      contiguous 16-byte run in NHWC, consecutive threads on consecutive runs of the same pixel.
        if (warp < NCONS_WARPS) {
#pragma unroll
            for (int i = 0; i < BN / 8; ++i)
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    *reinterpret_cast<float2 *>(cst + (frag_m + 8 * h) * C::EPI_PITCH + 8 * i + frag_n) = make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
        }
        __syncthreads();
        if (tid == 0) { SIGE_TRACE(7); SIGE_TRACE(8); SIGE_TRACE(9); }       // (no exchange: staged rows are complete)
        if (p.pdl) pdl_acquire();
        for (int q = tid; q < 128 * (BN / 8); q += NTHREADS) {
            const int m = q / (BN / 8), nv = q - m * (BN / 8);
            const int n = n0 + nv * 8;
            if (n >= p.Cout) continue;
            const long long pixel = pixel_of(m);
            if (pixel < 0) continue;
            float v[8];
            const float4 c0 = *reinterpret_cast<const float4 *>(cst + m * C::EPI_PITCH + nv * 8), c1 = *reinterpret_cast<const float4 *>(cst + m * C::EPI_PITCH + nv * 8 + 4);
            v[0] = c0.x; v[1] = c0.y; v[2] = c0.z; v[3] = c0.w; v[4] = c1.x; v[5] = c1.y; v[6] = c1.z; v[7] = c1.w;
            emit(pixel, tl_of(m), n, v);
        }
        if (tid == 0) SIGE_TRACE(10);
        if (p.trace) {                     // (uniform) CTA exit = every thread's stores issued
            __syncthreads();
            if (tid == 0) SIGE_TRACE(11);
        }
        return;
    }

    // ---- split-K: every CTA PUSHES the rows of its partial tile straight from registers into the shared memory of the
    //      rank that owns them (st.async, counted by the owner's RED_FULL barrier), then each rank sums the ks slots it received (local
    //      reads, fixed order -> deterministic) and stores.  Slot layout at the owner: [source rank][row within the owner's
    //      share][EPI_PITCH]; a rank's own rows go to its halo buffers.  Nobody reads remote memory after the exchange, so
    //      no exit barrier is needed.
    cg::cluster_group cluster = cg::this_cluster();
    const int per = 128 / p.ksplit;
    cluster.barrier_wait();                // (arrived during setup) every CTA of the cluster is running: remote stores are legal
    if (warp < NCONS_WARPS) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = frag_m + 8 * h;
            const int owner = m / per, lr = m - owner * per;
            const int row_off = ((kr < owner ? kr : kr - 1) * per + lr) * C::EPI_PITCH;      // in the owner's slot region
            if (owner != kr) {
                // st.async: the bytes are counted by an mbarrier of the OWNER, which then waits on its own barrier only
                const uint32_t remote = map_rank(sbase + C::OFF_SLOT + (uint32_t)(row_off + frag_n) * 4, owner);
                const uint32_t remote_bar = map_rank(RED_FULL, owner);
#pragma unroll
                for (int i = 0; i < BN / 8; ++i)
                    st_async8(remote + 32 * i, __float_as_uint(acc[4 * i + 2 * h]), __float_as_uint(acc[4 * i + 2 * h + 1]), remote_bar);
            } else {
                float *slot = cst + lr * C::EPI_PITCH;
#pragma unroll
                for (int i = 0; i < BN / 8; ++i)
                    *reinterpret_cast<float2 *>(slot + 8 * i + frag_n) = make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
            }
        }
    }
    if (tid == 0) SIGE_TRACE(7);
    if (p.pdl) pdl_acquire();
    __syncthreads();                       // own rows staged
    mbar_wait_cluster(RED_FULL, 0);        // the rows the other ranks pushed have landed
    if (tid == 0) { SIGE_TRACE(8); SIGE_TRACE(9); }
    const float *rslot = reinterpret_cast<const float *>(smem + C::OFF_SLOT);
    for (int q = tid; q < per * (BN / 8); q += NTHREADS) {
        const int lr = q / (BN / 8), nv = q - lr * (BN / 8);
        const int n = n0 + nv * 8;
        if (n >= p.Cout) continue;
        const long long pixel = pixel_of(kr * per + lr);
        if (pixel < 0) continue;
        float v[8];
#pragma unroll
        for (int z = 0; z < 8; ++z) v[z] = 0.f;
#pragma unroll
        for (int r = 0; r < 8; ++r) {       // fixed rank order: bitwise-deterministic sum
            if (r < p.ksplit) {
                const float *cs = (r == kr ? cst + lr * C::EPI_PITCH : rslot + ((r < kr ? r : r - 1) * per + lr) * C::EPI_PITCH) + nv * 8;
                const float4 c0 = *reinterpret_cast<const float4 *>(cs), c1 = *reinterpret_cast<const float4 *>(cs + 4);
                v[0] += c0.x; v[1] += c0.y; v[2] += c0.z; v[3] += c0.w; v[4] += c1.x; v[5] += c1.y; v[6] += c1.z; v[7] += c1.w;
            }
        }
        emit(pixel, tl_of(kr * per + lr), n, v);
    }
    if (tid == 0) SIGE_TRACE(10);
    if (p.trace) {                         // (uniform) CTA exit = every thread's stores issued
        __syncthreads();
        if (tid == 0) SIGE_TRACE(11);
    }
}

// ------------------------------------------------------------------------------------------
// host: tensor map + launch
// ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *sym = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(sym);
    }
    return fn;
}

// Launch plan of one layer: tile width, K split and ring flavour.  Pure host logic (exported as sige_tile_conv_plan so
// that it can be tested without a GPU).
struct Plan {
    int bn, ksplit, deep;
};

// What the plan needs to know about the device: SMs, and how many CTAs of this kernel (214 KB of shared memory, one CTA per
// SM) are co-resident for clusters of 1 / 2 / 4 / 8 — cudaOccupancyMaxActiveClusters x cluster size, queried once per device.
// Without a device (host-only planning) the values of an H100 80GB HBM3 SXM: 132 / 132 / 120 / 120 (66 x2, 30 x4, 15 x8).
struct Machine {
    int sms;
    int max_ctas[9];
};
static Machine machine() {
    static const Machine kH100 = {kDefaultSMs, {0, kDefaultSMs, kDefaultSMs, 0, 120, 0, 0, 0, 120}};
    static Machine cache[64];
    static bool done[64] = {false};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) {
        (void)cudaGetLastError();
        return kH100;
    }
    if (!done[dev]) {
        Machine m = kH100;
        m.sms = sm_count();
        for (int cs = 1; cs <= 8; cs *= 2) m.max_ctas[cs] = 0;
        m.max_ctas[1] = m.max_ctas[2] = m.sms;
        using C = Cfg<64, 9, true>;
        auto kern = tile_conv_tc5_kernel<__half, 64, 9, true, true>;
        bool ok = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES) == cudaSuccess;
        for (int cs = 2; ok && cs <= 8; cs *= 2) {
            cudaLaunchConfig_t cfg = {};
            cfg.gridDim = dim3(1, 1, cs);
            cfg.blockDim = dim3(NTHREADS);
            cfg.dynamicSmemBytes = C::SMEM_BYTES;
            cudaLaunchAttribute attr;
            attr.id = cudaLaunchAttributeClusterDimension;
            attr.val.clusterDim.x = 1;
            attr.val.clusterDim.y = 1;
            attr.val.clusterDim.z = cs;
            cfg.attrs = &attr;
            cfg.numAttrs = 1;
            int n = 0;
            ok = cudaOccupancyMaxActiveClusters(&n, kern, &cfg) == cudaSuccess && n > 0;
            if (ok) m.max_ctas[cs] = n * cs;
        }
        (void)cudaGetLastError();
        if (!ok) m = kH100;
        cache[dev] = m;
        done[dev] = true;
    }
    return cache[dev];
}

// C0, early: channels of src[0] and the SIGE_CONV_EARLY_* mask, for the K partition (KOrder)
static Plan decide(long long NT, int Cin, int C0, int Cout, int taps, int Cin2, int early, int ksplit_req, bool s2 = false) {
    Plan pl;
    const long long m_blocks = ceil_div(NT, s2 ? S2_TILES : TILES);
    // BN = 128 when that still fills the machine — or when the narrow tiling would need more waves of one-per-SM CTAs
    // than the wide one (a batch of edits: 64 row blocks x Cout 256 is 256 narrow CTAs = 2 waves, 128 wide CTAs = 1 wave,
    // and a CTA's gather — the long pole — is the same either way); small problems want more, narrower CTAs
    const long long narrow_ctas = m_blocks * (Cout / 64), wide_ctas = m_blocks * (Cout / 128);
    const Machine mc = machine();
    const long long sms = mc.sms;
    const bool wide = !s2 && (Cout % 128 == 0) && (wide_ctas >= sms || (narrow_ctas > sms && ceil_div(wide_ctas, sms) < ceil_div(narrow_ctas, sms)));
    pl.bn = wide ? 128 : 64;
    const bool split_ok = pl.bn == 64;                       // Cfg::kSplitOk
    const int tps = (taps == 9 && pl.bn == 64) ? 3 : 1;     // Cfg::TPS
    const KOrder ko(Cin, C0, (taps == 9 && !s2) ? Cin2 : 0, taps / tps, s2 ? 0 : early);
    const int J = ko.J;                                      // ring steps
    auto shortest = [&](int k) {                             // steps of the shortest K slice of a k-way split
        int m = J;
        for (int kr = 0; kr < k; ++kr) m = min(m, KSlice(ko, kr, k).n);
        return m;
    };
    const long long base = m_blocks * (Cout / pl.bn);
    int ks = ksplit_req;
    if (ks <= 0) {
        // never spill into a second wave of co-resident CTAs (machine()); splitting pays while every slice keeps >= kMinTaps taps
        constexpr int kMinTaps = 3;
        const int *kMaxCtas = mc.max_ctas;
        ks = 1;
        while (split_ok && ks < 8 && base * (ks * 2) <= kMaxCtas[ks * 2] && shortest(ks * 2) * tps >= kMinTaps) ks *= 2;
    }
    if (ks > J || !split_ok) ks = 1;
    pl.ksplit = ks;
    pl.deep = (!s2 && pl.bn == 64 && taps == 9 && ks > 1) ? 1 : 0;       // every split narrow 3x3 launch, and only those (Cfg::kUnsplit39)
    return pl;
}

template <typename T, int BN, int TAPS, bool DEEP, bool ASYNC, bool S2 = false, bool DB = false, bool MOD = false>
static int launch_v(Params &p, const void *w_packed, const void *w2_packed, cudaStream_t st) {
    using C = Cfg<BN, TAPS, DEEP, S2, DB>;
    EncodeTiledFn enc = encode_fn();
    if (!enc) {
        set_error("sige_tile_conv(wgmma): cuTensorMapEncodeTiled is not available from the driver");
        return 2;
    }
    CUtensorMap wmap;
    // packed weights [tap][Cin/64][Cout][64] seen as a 2-D tensor {64, taps * Cin/64 * Cout}: a box is contiguous
    const cuuint64_t gdim[2] = {(cuuint64_t)KC, (cuuint64_t)TAPS * (p.Cin / KC) * p.Cout};
    const cuuint64_t gstr[1] = {(cuuint64_t)KC * 2};
    const cuuint32_t box[2] = {KC, (cuuint32_t)BN};
    const cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(&wmap, p.is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void *>(w_packed),
                     gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("sige_tile_conv(wgmma): cuTensorMapEncodeTiled failed with %d", (int)r);
        return 2;
    }
    CUtensorMap wmap2 = wmap;
    if (p.Cin2 > 0) {
        const cuuint64_t gdim2[2] = {(cuuint64_t)KC, (cuuint64_t)(p.Cin2 / KC) * p.Cout};
        r = enc(&wmap2, p.is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void *>(w2_packed), gdim2, gstr, box,
                estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) {
            set_error("sige_tile_conv(wgmma): cuTensorMapEncodeTiled (shortcut weights) failed with %d", (int)r);
            return 2;
        }
    }
    auto kern = tile_conv_tc5_kernel<T, BN, TAPS, DEEP, ASYNC, S2, DB, MOD>;
    static int attr_dev = -1;
    int dev = 0;
    cudaGetDevice(&dev);
    if (attr_dev != dev) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
        if (e != cudaSuccess) {
            set_error("sige_tile_conv(wgmma): cannot reserve %d bytes of shared memory: %s", C::SMEM_BYTES, cudaGetErrorString(e));
            return 2;
        }
        attr_dev = dev;
    }
    const dim3 grid(ceil_div(p.NT, C::CT), p.Cout / BN, p.ksplit);
    const cudaError_t e = launch_ex(kern, grid, dim3(NTHREADS), C::SMEM_BYTES, st, p.pdl != 0, dim3(1, 1, p.ksplit), p, wmap, wmap2);
    if (e != cudaSuccess) {
        set_error("sige_tile_conv(wgmma): launch failed (grid %d x %d x %d): %s", grid.x, grid.y, grid.z, cudaGetErrorString(e));
        (void)cudaGetLastError();
        return 2;
    }
    return 0;
}

// pure-copy gathers (no pre-op in the gather stage) take the cp.async variant; modulated ones the register-staged MOD variant
template <typename T, int BN, int TAPS, bool DEEP = false, bool DB = false>
static int launch(Params &p, const void *w_packed, const void *w2_packed, cudaStream_t st) {
    if (p.gamma) return launch_v<T, BN, TAPS, DEEP, false, false, DB, true>(p, w_packed, w2_packed, st);
    const bool pure_copy = p.scale == nullptr && p.shift == nullptr && p.act == SIGE_ACT_IDENTITY;
    if (pure_copy) return launch_v<T, BN, TAPS, DEEP, true, false, DB>(p, w_packed, w2_packed, st);
    return launch_v<T, BN, TAPS, DEEP, false, false, DB>(p, w_packed, w2_packed, st);
}

// Halo fills of the longest K slice of a split narrow 3x3 launch (the kernel's partition: KOrder, KSlice).  One fill: the
// single-buffered layout (its deep weight ring has the whole slice in flight); more: the double-buffered one.
static int split_halo_fills(int Cin, int C0, int Cin2, int early, int ks) {
    const KOrder ko(Cin, C0, Cin2, 3, early);
    int most = 0;
    for (int kr = 0; kr < ks; ++kr) most = max(most, KSlice(ko, kr, ks).fills(ko));
    return most;
}
static int g_split_halo_buffers = 0;     // sige_debug_set_split_halo_buffers

}  // namespace tc5

static long long *g_trace = nullptr;
extern "C" int sige_debug_set_trace(void *buf) {
    g_trace = reinterpret_cast<long long *>(buf);
    return 0;
}
extern "C" int sige_debug_set_split_halo_buffers(int n) {
    SIGE_REQUIRE(n >= 0 && n <= 2, "sige_debug_set_split_halo_buffers: n must be 0, 1 or 2 (got %d)", n);
    tc5::g_split_halo_buffers = n;
    return 0;
}

// stride-2 geometry: 3x3 stride 2 on 5x5 tiles -> 2x2 outputs, pure-copy gather (no pre-op in the gather stage), no fused shortcut
static bool tc5_is_s2(const sige_tile_conv_t *a) {
    return a->kH == 3 && a->kW == 3 && a->stride == 2 && a->R == 5 && a->S == 5 && a->n_src2 == 0 && a->scale == nullptr &&
           a->shift == nullptr && a->act == SIGE_ACT_IDENTITY;
}

// Can the wgmma kernel take this layer?  (3x3 stride 1 on 6x6 tiles, 1x1 on 4x4 tiles, or 3x3 stride 2 on 5x5 tiles; Cout % 64 == 0)
// A modulated layer takes the stride-1 geometries only: the stride-2 one has no register-staged gather.
bool tc5_supported(const sige_tile_conv_t *a) {
    if (a->modulation && a->stride != 1) return false;
    const bool g3 = (a->kH == 3 && a->kW == 3 && a->stride == 1 && a->R == 6 && a->S == 6) || tc5_is_s2(a);
    const bool g1 = a->kH == 1 && a->kW == 1 && a->stride == 1 && a->R == 4 && a->S == 4;
    if (a->n_src2 > 0 && !g3) return false;
    // the kernel keeps 32-bit element offsets into its sources
    const long long px = a->src_is_stack ? (long long)a->B * a->N * a->R * a->S : (long long)a->B * a->H * a->W;
    long long cmax = 0;
    for (int i = 0; i < a->n_src; ++i) {
        const int pitch = (i == 0 && a->src_pixel_stride > 0) ? a->src_pixel_stride : a->src[i].C;
        cmax = pitch > cmax ? pitch : cmax;
    }
    if (px * cmax >= (1ll << 31)) return false;
    if ((a->dst_is_stack ? (long long)a->B * a->N * 16 : (long long)a->B * a->dH * a->dW) >= (1ll << 31)) return false;
    if (tc5_is_s2(a) && a->dst_is_stack) return false;          // (stack outputs of this geometry: mma.sync kernel)
    return (g3 || g1) && a->Cout % 64 == 0 && a->Cin % 64 == 0 && (a->ksplit == 0 || a->ksplit == 1 || a->ksplit == 2 || a->ksplit == 4 || a->ksplit == 8);
}

// Arguments were validated by sige_tile_conv (tile_conv_mma.cu) before this is called.
int tc5_launch(const sige_tile_conv_t *a, cudaStream_t st) {
    tc5::Params p;
    p.seg[0] = tc5::Seg{a->src[0].ptr, a->src_pixel_stride > 0 ? a->src_pixel_stride : a->src[0].C, a->src[0].up};
    p.seg[1] = a->n_src == 2 ? tc5::Seg{a->src[1].ptr, a->src[1].C, a->src[1].up} : p.seg[0];
    p.C0 = a->src[0].C;
    p.src_is_stack = a->src_is_stack;
    p.H = a->src_is_stack ? a->R : a->H;
    p.W = a->src_is_stack ? a->S : a->W;
    p.idx = a->idx;
    p.N = a->N;
    p.NT = a->B * a->N;
    p.scale = a->scale; p.shift = a->shift; p.affine_bstride = a->affine_bstride; p.act = a->act;
    p.bias = a->bias;
    p.Cin = a->Cin; p.Cout = a->Cout; p.taps = a->kH * a->kW;
    p.dst = a->dst; p.dst_is_stack = a->dst_is_stack;
    p.dH = a->dst_is_stack ? 4 : a->dH;
    p.dW = a->dst_is_stack ? 4 : a->dW;
    p.dC = a->dC; p.dst_c0 = a->dst_c0;
    p.offH = a->offH; p.offW = a->offW;
    p.residual = a->residual; p.rC = a->rC; p.res_c0 = a->res_c0;
    p.n_aux = a->n_aux;
    for (int i = 0; i < a->n_aux; ++i) p.aux[i] = tc5::AuxDst{a->aux[i].ptr, a->aux[i].C, a->aux[i].c0, a->aux[i].scale, a->aux[i].shift, a->aux[i].act};
    p.seg2[0] = a->n_src2 > 0 ? tc5::Seg{a->src2[0].ptr, a->src2[0].C, a->src2[0].up} : p.seg[0];
    p.seg2[1] = a->n_src2 == 2 ? tc5::Seg{a->src2[1].ptr, a->src2[1].C, a->src2[1].up} : p.seg2[0];
    p.C0_2 = a->n_src2 > 0 ? a->src2[0].C : 0;
    p.Cin2 = a->n_src2 > 0 ? a->Cin2 : 0;
    p.bias2 = a->n_src2 > 0 ? a->bias2 : nullptr;
    p.sc_flags = a->n_src2 > 0 ? a->sc_flags : nullptr;
    p.idx_per_image = a->idx_per_image ? 1 : 0;
    p.ksplit = a->ksplit;
    p.pdl = (a->flags & SIGE_CONV_PDL) ? 1 : 0;
    p.early_release = (a->flags & SIGE_CONV_EARLY_RELEASE) ? 1 : 0;
    p.early = (a->flags >> 4) & 7;                                      // SIGE_CONV_EARLY_SRC0 | _SRC1 | _SHORTCUT
    p.is_bf16 = a->dtype == SIGE_BF16;
    p.trace = g_trace;
    const sige_conv_modulation_t *m = a->modulation;
    const size_t esz = 2;                                                  // f16 / bf16
    p.gamma = m ? static_cast<const char *>(m->gamma) + (size_t)m->gamma_c0 * esz : nullptr;
    p.beta = m ? static_cast<const char *>(m->beta) + (size_t)m->beta_c0 * esz : nullptr;
    p.gC = m ? m->gamma_C : 0;
    p.bC = m ? m->beta_C : 0;
    p.slope = m ? m->negative_slope : 1.f;
    const bool s2 = !m && tc5_is_s2(a);
    // a CTA's first index row is row tile0 of `idx`: one list (B == 1), or per-image lists whose length is a whole number of CTAs
    // (no CTA then holds tiles of two images, so padding behind one image's tiles fills whole CTAs)
    // (per-image lists may have a stack on one side; the list's row tile0 is then also the CTA's first stack row)
    p.padded = ((a->flags & SIGE_CONV_PADDED) && a->idx && (a->idx_per_image || (!a->src_is_stack && !a->dst_is_stack)) &&
                (a->B == 1 || (a->idx_per_image && a->N % (s2 ? tc5::S2_TILES : tc5::TILES) == 0))) ? 1 : 0;
    const tc5::Plan pl = tc5::decide(p.NT, p.Cin, p.C0, p.Cout, p.taps, p.Cin2, p.early, a->ksplit, s2);
    p.ksplit = pl.ksplit;
    if (s2) {
        if (a->dtype == SIGE_F16) return tc5::launch_v<__half, 64, 9, false, true, true>(p, a->w_packed, a->w2_packed, st);
        return tc5::launch_v<__nv_bfloat16, 64, 9, false, true, true>(p, a->w_packed, a->w2_packed, st);
    }
    const bool wide = pl.bn == 128, three = p.taps == 9;
    const int nab = tc5::g_split_halo_buffers ? tc5::g_split_halo_buffers : (tc5::split_halo_fills(p.Cin, p.C0, p.Cin2, p.early, p.ksplit) > 1 ? 2 : 1);
    const bool db = pl.deep && nab == 2;
#define SIGE_TC5(T)                                                                              \
    (wide ? (three ? tc5::launch<T, 128, 9>(p, a->w_packed, a->w2_packed, st) : tc5::launch<T, 128, 1>(p, a->w_packed, a->w2_packed, st)) \
          : (three ? (pl.deep ? (db ? tc5::launch<T, 64, 9, true, true>(p, a->w_packed, a->w2_packed, st) : tc5::launch<T, 64, 9, true>(p, a->w_packed, a->w2_packed, st)) \
                            : tc5::launch<T, 64, 9>(p, a->w_packed, a->w2_packed, st)) \
                   : tc5::launch<T, 64, 1>(p, a->w_packed, a->w2_packed, st)))
    if (a->dtype == SIGE_F16) return SIGE_TC5(__half);
    return SIGE_TC5(__nv_bfloat16);
#undef SIGE_TC5
}

void mma_plan_of(const sige_tile_conv_t *a, sige_tile_conv_plan_t *out);   // tile_conv_mma.cu

}  // namespace sige

// The wgmma plan of a descriptor whose launch takes the wgmma kernel.
static void tc5_plan(const sige_tile_conv_t *a, sige_tile_conv_plan_t *out) {
    using namespace sige;
    const long long NT = (long long)a->B * a->N;
    const bool s2 = tc5_is_s2(a);
    const int Cin2 = a->n_src2 > 0 ? a->Cin2 : 0;
    const tc5::Plan pl = tc5::decide(NT, a->Cin, a->src[0].C, a->Cout, a->kH * a->kW, Cin2, (a->flags >> 4) & 7, a->ksplit, s2);
    out->path = 1;
    out->bn = pl.bn;
    out->ksplit = pl.ksplit;
    out->deep_ring = pl.deep;
    out->grid_x = ceil_div(NT, s2 ? tc5::S2_TILES : tc5::TILES);
    out->grid_y = a->Cout / pl.bn;
    out->grid_z = pl.ksplit;
}

// Which kernel and grid sige_tile_conv would use for this descriptor (no pointer is dereferenced, nothing is launched).
extern "C" int sige_tile_conv_plan(const sige_tile_conv_t *a, sige_tile_conv_plan_t *out) {
    using namespace sige;
    SIGE_REQUIRE(a && out, "sige_tile_conv_plan: null pointer");
    out->path = 0; out->bn = 0; out->ksplit = 0; out->deep_ring = 0; out->grid_x = out->grid_y = out->grid_z = 0;
    if ((a->flags & SIGE_CONV_TC5) && tc5_supported(a)) tc5_plan(a, out);
    else mma_plan_of(a, out);
    return 0;
}
