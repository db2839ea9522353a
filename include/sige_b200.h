/*
 * sige_b200.h — C-ABI of the H100-native SIGE tile-sparse hot path.
 *
 * This is the drop-in boundary: plain pointers, sizes and a cudaStream_t; no torch
 * types.  It replaces the reference's pybind surface `sige.cuda`
 * (reference sige/cuda/pybind_cuda.cpp:5-12) and the libtorch host wrappers
 * behind it.  INTEGRATION.md shows the binding a maintainer of the reference
 * would add (ctypes / pybind stub).
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on error; the message is
 *     available from sige_last_error() (thread-local).  N == 0 is a no-op.
 *   - all pointers are DEVICE pointers unless the name ends in _host.
 *   - the caller owns every buffer, including outputs (allocation stays with the
 *     caller's allocator); inputs are never modified.
 *   - all work is enqueued on `stream` (a cudaStream_t passed as void*); nothing
 *     synchronises the host, so every call is CUDA-graph capturable.
 *   - activations are 4-D, logical (B, C, H, W).  `layout` says how they sit in
 *     memory: SIGE_NCHW (the reference's layout) or SIGE_NHWC (channels-last, the
 *     layout the tensor-core path wants).  Tile stacks are logical
 *     (B*N, C, R, S), tile row b*N + i (reference sige/cuda/gather_kernel.cu:30),
 *     stored in the same layout family as the activations.
 *   - active index lists are int32 [N,2] = (h, w) tile origins in the frame of
 *     the gather input; may be negative (reference sige/utils.py:31-37).
 */
#ifndef SIGE_B200_H_
#define SIGE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SIGE_B200_ABI_VERSION 3

typedef enum { SIGE_F32 = 0, SIGE_F16 = 1, SIGE_BF16 = 2 } sige_dtype_t;
typedef enum { SIGE_NCHW = 0, SIGE_NHWC = 1 } sige_layout_t;
/* reference sige/common.cpp:11-23 (ActivationType, getActivationType).  SIGE_ACT_RELU = max(x, 0) is accepted only as the
 * activation of a sige_tile_conv aux destination (the fused ReLU epilogue); every other activation argument takes
 * identity / swish. */
typedef enum { SIGE_ACT_IDENTITY = 0, SIGE_ACT_SWISH = 1, SIGE_ACT_RELU = 2 } sige_act_t;

typedef void *sige_stream_t; /* cudaStream_t */

/*
 * Broadcast operand (scale / shift / residual): a 4-D tensor whose every dim is
 * either 1 or the full extent (reference sige/common.cpp:25-34 `broadcastable`,
 * sige/cuda/common_cuda.cu:15-30 `binary_op_array_cuda`).  Element strides are
 * explicit so that any memory layout can be passed; a size-1 dim is never
 * multiplied by its stride.  ptr == NULL means "operand absent".
 */
typedef struct {
    const void *ptr;
    int dims[4];       /* B, C, H, W — each 1 or full */
    int64_t stride[4]; /* element strides of B, C, H, W */
    int dtype;         /* sige_dtype_t */
} sige_bcast_t;

/* ------------------------------------------------------------------------- */
/* library                                                                    */
/* ------------------------------------------------------------------------- */
const char *sige_last_error(void);
int sige_abi_version(void);
/* "sm_90a" etc. — the architecture the kernels in this library were built for. */
const char *sige_built_arch(void);
/* reference sige/common.cpp:17-23: "identity" / "swish" -> sige_act_t, -1 if unknown
 * (the reference has undefined behaviour for unknown names). */
int sige_activation_from_name(const char *name);

/* ------------------------------------------------------------------------- */
/* a1: mask -> active tile origins      (reference sige/utils.py:8-37)        */
/* ------------------------------------------------------------------------- */
/*
 * mask: uint8 [H, W] (non-zero = edited).  Writes up to `capacity` (h, w) pairs
 * into idx_out in row-major order of the pooled grid and the total count into
 * *count_out (device int32).  Bit-exact with the reference's pad -> max_pool2d ->
 * nonzero chain.  The pooled grid has floor((H+padH)/strideH)+1 rows.
 */
int sige_reduce_mask(const uint8_t *mask, int H, int W, int R, int S, int strideH, int strideW,
                     int padH, int padW, int32_t *idx_out, int capacity, int32_t *count_out,
                     sige_stream_t stream);
/*
 * E masks of one geometry, uint8 [E, H, W], in ONE launch (one CTA per mask, each the
 * ordered compaction of sige_reduce_mask): image e's tiles go to rows e*cap + i of
 * idx_out [E*cap, 2] (the per-image layout of sige_tile_conv_t.idx_per_image) in the
 * same order as sige_reduce_mask, SIGE_TILE_NONE fills the rest of each image's rows.
 * counts_out[e] (device int32) = the number of active tiles of image e.  An image with
 * more than cap keeps its first cap tiles and bit 0 of *status (device int32) is set;
 * the word is only ever OR-ed, never cleared.  E == 0 is a no-op.
 */
int sige_reduce_mask_batched(const uint8_t *masks, int E, int H, int W, int R, int S, int strideH,
                             int strideW, int padH, int padW, int32_t *idx_out, int cap,
                             int32_t *counts_out, int32_t *status, sige_stream_t stream);
/* host helper: number of candidate tiles (upper bound for `capacity`).  A geometry of 2^31 or more candidates, which
 * sige_reduce_mask and sige_reduce_mask_batched refuse, returns -1 and sets the error. */
int sige_reduce_mask_capacity(int H, int W, int R, int S, int strideH, int strideW, int padH,
                              int padW);

/* ------------------------------------------------------------------------- */
/* a2: gather                 (reference sige/cuda/gather_kernel.cu:7-124)    */
/* ------------------------------------------------------------------------- */
/* out: tile stack (B*N, C, R, S).  Zero outside the image, applied AFTER the
 * affine/activation (gather_kernel.cu:33-42). */
int sige_gather(const void *x, int dtype, int layout, int B, int C, int H, int W, int R, int S,
                const int32_t *idx, int N, const sige_bcast_t *scale, const sige_bcast_t *shift,
                int act, int act_first, void *out, sige_stream_t stream);
/* The same gather from a source that holds (H/2, W/2) pixels, read through nearest-neighbour x2 up-sampling (up = 1): what
 * `Gather(F.interpolate(x, scale_factor=2))` produces (reference diffusion/models/ddpm_arch/sige_fused_unet.py:223,
 * gaugan/models/spade_generators/sige_fused_spade_generator.py:237-249) without materialising the up-sampled tensor.
 * H, W are the up-sampled extents the tile origins refer to; up = 0 is sige_gather. */
int sige_gather_upsampled(const void *x, int dtype, int layout, int B, int C, int H, int W, int up, int R, int S,
                          const int32_t *idx, int N, const sige_bcast_t *scale, const sige_bcast_t *shift,
                          int act, int act_first, void *out, sige_stream_t stream);

/* ------------------------------------------------------------------------- */
/* a6: scatter                (reference sige/cuda/scatter_kernel.cu:8-44,76-117) */
/* ------------------------------------------------------------------------- */
/*
 * x: stack (B*N, C, Ro, So).  y: cached full tensor (B, C, H, W) or NULL.
 * out: (B, C, H, W).  If y != NULL and y != out the function first copies y into
 * out (the reference's `y.clone()`, scatter_kernel.cu:89); with y == NULL (or
 * y == out) the tiles are pasted in place into `out`.
 * out[b,c,oy+r,ox+s] = x[...] (+ residual[b,c,oy+r,ox+s]), oy = (offH + iy)/strideH.
 */
int sige_scatter(const void *x, const void *y, void *out, int dtype, int layout, int B, int C,
                 int H, int W, int Ro, int So, int offH, int offW, int strideH, int strideW,
                 const int32_t *idx, int N, const sige_bcast_t *residual, sige_stream_t stream);

/* ------------------------------------------------------------------------- */
/* a7: scatter_with_block_residual (reference scatter_kernel.cu:46-74,119-146) */
/* ------------------------------------------------------------------------- */
/* out = scatter(x0 -> y0, residual = y1); then out += x1 - y1 on the shortcut tiles
 * idx1 (raw origins, no offset/stride).  Same in-place convention as sige_scatter. */
int sige_scatter_with_block_residual(const void *x0, const void *y0, const void *x1,
                                     const void *y1, void *out, int dtype, int layout, int B,
                                     int C, int H, int W, int R0, int S0, int R1, int S1, int offH,
                                     int offW, int strideH, int strideW, const int32_t *idx0,
                                     int N0, const int32_t *idx1, int N1, sige_stream_t stream);

/* ------------------------------------------------------------------------- */
/* a5: get_scatter_map   (reference sige/cuda/scatter_gather_kernel.cu:69-98,164-188) */
/* ------------------------------------------------------------------------- */
/* map_out: int32 [H, W, 3] = (tile id, r, s) or -1. Fills -1 itself. */
int sige_get_scatter_map(int H, int W, int R, int S, int kH, int kW, int offH, int offW,
                         int strideH, int strideW, const int32_t *idx, int N, int32_t *map_out,
                         sige_stream_t stream);

/* ------------------------------------------------------------------------- */
/* a4: scatter_gather    (reference sige/cuda/scatter_gather_kernel.cu:8-67,100-162) */
/* ------------------------------------------------------------------------- */
/* x: previous conv's output stack (B*N, C, Rx, Sx); y: cached (B, C, H, W);
 * out: stack (B*N, C, R, S) for the next conv. */
int sige_scatter_gather(const void *x, const void *y, int dtype, int layout, int B, int C, int H,
                        int W, int Rx, int Sx, int R, int S, const int32_t *idx, int N,
                        const int32_t *scatter_map, const sige_bcast_t *scale,
                        const sige_bcast_t *shift, int act, int act_first, void *out,
                        sige_stream_t stream);

/* ------------------------------------------------------------------------- */
/* a3 + fused forms: tile convolution                                         */
/*   (reference sige/nn/base.py:85-92 -> F.conv2d on the stack; the fused forms */
/*    replace the gather -> conv -> scatter call triple of                     */
/*    diffusion/models/ddpm_arch/sige_fused_unet.py:111-128)                   */
/* ------------------------------------------------------------------------- */

/* Weight repack for the tensor-core path: OIHW (any dtype) -> [kH*kW][Cin/64][Cout][64]
 * in `dst_dtype` (f16/bf16) — the slab of one (tap, 64-channel chunk, Cout block) is contiguous.
 * Run once per weight.  (Cin not a multiple of 64: plain [kH*kW][Cout][Cin].  A sige_tile_conv source of such a
 * width wants the weight zero-padded along Cin to round_up(Cin, 64) first, then packed.) */
int sige_pack_conv_weight(const void *w_oihw, int src_dtype, int Cout, int Cin, int kH, int kW,
                          void *w_packed, int dst_dtype, sige_stream_t stream);

/* One source segment of the (virtually concatenated) conv input: NHWC. */
typedef struct {
    const void *ptr; /* [B, H>>up, W>>up, C] */
    int C;           /* channels in this segment: a multiple of 64 on the tensor-core path, or a multiple of 8 for the
                        only segment of a launch (mma.sync kernel; no fused shortcut) */
    int up;          /* 0, or 1 = nearest-neighbour x2 upsample applied on read */
} sige_conv_src_t;

/* Extra destination of the fused epilogue: aux = act(out * scale[c] + shift[c]) written next to `dst` (same
 * geometry).  Lets the PRODUCER of an activation apply the consumer's GroupNorm affine + SiLU once per
 * element, so the consumer's gather stage is a pure copy (reference applies it in every gather,
 * sige/cuda/gather_kernel.cu:45-65). */
typedef struct {
    void *ptr;          /* NHWC, C channels per pixel, same B/H/W (or stack shape) as dst */
    int C, c0;          /* writes channels [c0, c0 + Cout) */
    const float *scale; /* fp32 [Cout] or NULL */
    const float *shift; /* fp32 [Cout] or NULL */
    int act;            /* sige_act_t; SIGE_ACT_RELU only on a sige_tile_conv aux (dst = NULL, one aux, no affine:
                           the launch writes relu(conv + bias [+ residual])) */
} sige_conv_aux_t;

/* SPADE's modulation applied in the gather stage of a tile conv (sige_tile_conv_t.modulation): for channel c < Cin of an in-image
 * halo pixel the conv reads
 *   a = leaky((x*scale[c] + shift[c]) * (1 + gamma[c]) + beta[c], negative_slope)      (fp32, rounded once to the dtype)
 * — reference gaugan/models/sige_normalization.py:84-86 plus the block's F.leaky_relu(., 0.2) on the three stacks its Gather /
 * ScatterGather modules cut, without materialising them.  gamma and beta are NHWC [B, H, W, C] at the source's LOGICAL extent
 * (B, H, W of the descriptor; the source itself may be read through x2 up-sampling), each read from channels
 * [c0, c0 + Cin) of its C.  Pixels outside the image and SIGE_TILE_NONE tiles read zero; on a narrow source gamma and beta are
 * never read at or past Cin. */
typedef struct {
    const void *gamma;
    int gamma_C, gamma_c0;
    const void *beta;
    int beta_C, beta_c0;
    float negative_slope;   /* 1 = no activation (the shortcut SPADE) */
} sige_conv_modulation_t;

typedef struct {
    int dtype; /* SIGE_F16 / SIGE_BF16 (tensor cores) */
    /* ---- source: where halo tiles are gathered from ----
     * Every segment's C is a multiple of 64, or n_src == 1 and C is a multiple of 8 (a narrow layer: the last K chunk is
     * partial and runs on the mma.sync kernel; w_packed is then the weight zero-padded to round_up(Cin, 64) input channels;
     * no fused shortcut). */
    int n_src;              /* 1 or 2 (channel concat of two tensors, torch.cat dim=1) */
    sige_conv_src_t src[2];
    int B, H, W;            /* logical input extent (after optional upsample) */
    int src_is_stack;       /* 1: src[0] is a tile stack (B*N, R, S, C); origins are (0,0) */
    const int32_t *idx;     /* [N,2] tile origins (input frame); unused for a stack source */
    int N;                  /* active tiles per batch element */
    int R, S;               /* halo tile extent */
    /* ---- fused pre-op: act(x*scale+shift), zero outside the image ---- */
    const float *scale;     /* fp32 [B or 1, Cin] or NULL */
    const float *shift;     /* fp32 [B or 1, Cin] or NULL */
    int affine_bstride;     /* 0 (shared) or Cin (per batch element) */
    int act;                /* sige_act_t */
    /* ---- conv ---- */
    const void *w_packed;   /* from sige_pack_conv_weight (of the Cin-padded weight on a narrow source) */
    const float *bias;      /* fp32 [Cout] or NULL */
    int Cin, Cout, kH, kW, stride;
    /* ---- destination ---- */
    void *dst;              /* NHWC [B, dH, dW, dC] or stack (B*N, Ro, So, dC) */
    int dst_is_stack;
    int dH, dW, dC, dst_c0; /* writes channels [dst_c0, dst_c0 + Cout) of dC */
    int offH, offW;         /* output origin = (off + idx) / stride  (scatter_kernel.cu:29,33) */
    const void *residual;   /* NHWC, same geometry as dst (rC channels), added in the epilogue; or NULL */
    int rC, res_c0;
    /* ---- scheduling ---- */
    int ksplit;             /* split-K factor = thread-block-cluster size (partials reduced over distributed
                               shared memory): 0 = auto, or 1 / 2 / 4 / 8 */
    int flags;              /* SIGE_CONV_* */
    /* ---- optional extra destinations ---- */
    int n_aux;              /* 0, 1 or 2 */
    sige_conv_aux_t aux[2];
    /* ---- optional fused 1x1 shortcut (wgmma path, 3x3 main conv only) ----
     * out += conv1x1(src2) + bias2 on the main tiles whose sc_flags byte is non-zero (sc_flags == NULL: all); on the
     * other tiles `residual` (the CACHED shortcut output) is added instead.  This is the reference's
     * ScatterWithBlockResidual (sige/cuda/scatter_kernel.cu:46-74,119-146) folded into conv2's launch: the shortcut's
     * own active tiles are a subset of the main conv's. */
    int n_src2;             /* 0, 1 or 2 channel-concatenated raw sources (same B/H/W as src) */
    sige_conv_src_t src2[2];
    int Cin2;               /* channels of the shortcut input (multiple of 64) */
    const void *w2_packed;  /* sige_pack_conv_weight of the 1x1 weights */
    const float *bias2;     /* fp32 [Cout] or NULL */
    const uint8_t *sc_flags;/* [N] per main tile, or NULL */
    /* ---- per-image tile lists: a batch of INDEPENDENT EDITS in one launch ----
     * 0 (the reference's layout, sige/cuda/gather_kernel.cu:30): every image of the batch uses the same N tile origins.
     * 1: `idx` (and `sc_flags`) hold B*N entries, row b*N + i = tile i of image b — each edit has its own mask; lists shorter
     * than N are padded with SIGE_TILE_NONE origins (such a tile reads zeros and writes nothing).  Weights are read once for
     * the whole batch.  Full-tensor source and destination only (no stacks).  A window source (src_pixel_stride) or a modulated
     * one (modulation) takes per-image lists only with SIGE_CONV_PER_IMAGE_OPERANDS in `flags`. */
    int idx_per_image;
    /* ---- single source read as a channel window of a wider NHWC buffer ----
     * 0: src[0] has src[0].C channels per pixel.  Otherwise src[0] is channels [c0, c0 + src[0].C) of a buffer with
     * src_pixel_stride channels per pixel, src[0].ptr pointing at channel c0 of pixel 0 — e.g. one torch.split part of a conv's
     * output (SPADE's actv_0 / actv_1 / actv_s, reference gaugan/models/spade_generators/sige_fused_spade_generator.py:160-167),
     * read in place.  The launch is the one of the compacted window (same kernel, plan and result); SIGE_CONV_TC5 is honoured.
     * Needs n_src == 1, a full-tensor source, no fused shortcut, idx_per_image == 0 (or 1 with SIGE_CONV_PER_IMAGE_OPERANDS), a
     * stride that is a multiple of 8 and at least src[0].C, a 16-byte aligned source, and no modulation. */
    int src_pixel_stride;
    /* ---- SPADE's modulation in the gather stage (sige_conv_modulation_t above), or NULL ----
     * The pre-op is followed by the modulation.  With SIGE_CONV_TC5, the stride-1 wgmma geometries (3x3 on 6x6 tiles, 1x1 on 4x4
     * tiles, Cin and Cout multiples of 64) run on the wgmma kernel with the plan of the unmodulated launch; everything else (narrow
     * Cin, other Cout, stride 2, no flag) runs on the mma.sync kernel.  Both stage the same operand.  Needs n_src == 1, a
     * full-tensor source, act == SIGE_ACT_IDENTITY (negative_slope is the activation), no fused shortcut, idx_per_image == 0 (or 1
     * with SIGE_CONV_PER_IMAGE_OPERANDS), a finite slope, non-null 16-byte aligned gamma / beta whose windows are multiples of 8 elements within their buffers, and
     * src_pixel_stride == 0. */
    const sige_conv_modulation_t *modulation;
} sige_tile_conv_t;

/* Launch with programmatic dependent launch: the kernel prefetches its weights while the previous kernel
 * of the stream drains, and waits (griddepcontrol.wait) before touching activations. */
#define SIGE_CONV_PDL 1
/* Use the wgmma / TMA kernel when the geometry allows (3x3 s1 on 6x6 tiles, 1x1 on 4x4 tiles,
 * Cout % 64 == 0); otherwise the mma.sync kernel runs. */
#define SIGE_CONV_TC5 2
/* `idx` is a fixed-capacity list (B == 1), or B of them (idx_per_image == 1): real tiles packed at the front of each list,
 * SIGE_TILE_NONE entries behind them, possibly whole CTAs' worth — CTAs made only of padding exit at once.  With per-image lists
 * the flag takes effect only when N is a multiple of the kernel's tiles per CTA (8 for the stride-1 geometries of either kernel,
 * 32 for the wgmma stride-2 one, the plan's tiles per CTA on the mma.sync kernel), so that no CTA holds tiles of two images.
 * (Without the flag padding entries are still harmless: they read zeros and write nothing; the flag only buys the early exit,
 * at the price of one index load on every CTA's prologue.) */
#define SIGE_CONV_PADDED 4
/* With SIGE_CONV_PDL on the wgmma kernel: release the next launch right after this launch's own dependency has resolved, instead
 * of at the epilogue, so that the next launch's CTAs take the SMs this one leaves idle and gather their early chunks (below)
 * during this launch's mainloop.  Meant for the predecessor of a launch with early source groups. */
#define SIGE_CONV_EARLY_RELEASE 8
/* Early source groups (wgmma kernel, with SIGE_CONV_PDL): source groups the launch may read before its dependency on the preceding
 * launch of the stream resolves — src[0], src[1], all of src2 (the fused shortcut).  Their K chunks are gathered and multiplied
 * while the preceding launch is still running; each rank of a split takes an even share of them, then an even share of the rest.
 * Set one only for a group that the preceding launch does not write (nor the pre-op's scale / shift, nor the modulation's gamma /
 * beta, for the src groups), and only when the preceding launch is a sige_tile_conv on the wgmma kernel: such a launch waits for
 * ITS predecessor before it releases its dependents, so every launch before it has completed.  None set = wait before the first
 * gather.  The sum is the same up to the order of the K chunks; the mma.sync kernel and the stride-2 geometry ignore them (they
 * wait first). */
#define SIGE_CONV_EARLY_SRC0 16
#define SIGE_CONV_EARLY_SRC1 32
#define SIGE_CONV_EARLY_SHORTCUT 64
/* A batch of INDEPENDENT EDITS (sige_tile_conv_t.flags and sige_separable_conv_t.flags): every operand of the launch holds B
 * images — the source or its window, gamma and beta of the modulation, the destinations — image b of each at b * H * W * (its
 * pixel stride), and the launch reads per-image tile lists: row b*N + i of `idx` is tile i of image b, a SIGE_TILE_NONE row reads
 * zeros and writes nothing.  sige_tile_conv: needs idx_per_image == 1 (and so full-tensor source and destination); it is what lets
 * a window or a modulated source take per-image lists.  sige_separable_conv: needs an NHWC buffer source and buffer destinations
 * (no stacks).  Both refuse the flag otherwise, before any CUDA call; SIGE_CONV_PADDED behaves as for per-image lists. */
#define SIGE_CONV_PER_IMAGE_OPERANDS 128
/* Origin of a padding entry of a per-image tile list (both coordinates). */
#define SIGE_TILE_NONE (-30000)

/* Fused gather -> (affine+SiLU) [-> SPADE modulation] -> conv (+bias) -> (+residual) -> scatter, one launch.  Every refusal
 * comes before any CUDA call: a null descriptor and one with both src_pixel_stride and modulation set first, then a window or a
 * modulation that lacks what its field needs, then whatever fails the checks every launch makes.  N == 0 is a no-op. */
int sige_tile_conv(const sige_tile_conv_t *p, sige_stream_t stream);

/* Residual block: conv1 -> conv2 of one block (reference diffusion/models/ddpm_arch/sige_fused_unet.py:100-131: main_gather ->
 * conv1 -> scatter_gather -> conv2 -> scatter[_with_block_residual]) as ONE call.  `conv2` gathers from the buffer `conv1`
 * scatters into (conv1->dst or one of its aux views must be conv2's source); its fused 1x1 shortcut / residual fields carry
 * the block's skip path.  The two launches are chained by programmatic dependent launch (SIGE_CONV_PDL is forced on the
 * second): conv2's prologue and weight prefetch overlap conv1, its gather waits for conv1's tiles.  Returns the first
 * non-zero status. */
int sige_resblock(const sige_tile_conv_t *conv1, const sige_tile_conv_t *conv2, sige_stream_t stream);

/* Generic (any dtype incl. fp32, any channel count, groups, dilation) tile convolution on a
 * stack: x (M, Cin, R, S) -> out (M, Cout, Ro, So); w OIHW in `dtype`; fp32 accumulate. */
int sige_tile_conv_generic(const void *x, const void *w, const void *bias, void *out, int dtype,
                           int layout, int M, int Cin, int R, int S, int Cout, int kH, int kW,
                           int strideH, int strideW, int dilH, int dilW, int groups,
                           sige_stream_t stream);

/* ------------------------------------------------------------------------- */
/* dense glue of a step (not tile-shaped), NHWC f16/bf16                      */
/*   reference diffusion/models/ddpm_arch/sige_fused_unet.py:395 (conv_in),    */
/*   :431-433 (norm_out -> swish -> conv_out), models/common.py:37-57 (fold)   */
/* ------------------------------------------------------------------------- */
/* Launch plan sige_tile_conv would use for a descriptor: pure host logic (no pointer is dereferenced, nothing is
 * launched) — exported so that the tile-width / split-K / ring heuristics can be tested without a GPU (which then plan
 * for 132 SMs).  A window is planned with its pixel stride and a modulated descriptor (modulation only tested against NULL) with
 * the kernels that take modulated launches, so the plan is the launch's.  path 0 with every other field 0: the mma.sync kernel
 * would not take the descriptor either (fp32, a tile that fits no CTA configuration, a ksplit that is not a cluster size, ...). */
typedef struct {
    int path;      /* 1 = wgmma kernel, 0 = mma.sync kernel */
    int bn;        /* output channels per CTA (64 or 128); mma.sync: 128 = the L configuration (128 GEMM rows), 64 = M (64
                      rows) or S (32 rows), each packing min(rows / (Ro*So), halo pixels / (R*S)) tiles per CTA, halo 288 /
                      144 / 72 pixels: grid_x = ceil(B*N / tiles per CTA) tells M from S */
    int ksplit;    /* K slices = thread-block cluster size (1, 2, 4, 8) */
    int deep_ring; /* 1 = the split-K layout of the narrow 3x3 configuration: one halo buffer + five weight stages when every
                      K slice needs one halo fill, else two halo buffers + two weight stages fed from L2 */
    int grid_x, grid_y, grid_z;   /* mma.sync: ceil(B*N / tiles per CTA), ceil(Cout / bn), ksplit; deep_ring 0 */
} sige_tile_conv_plan_t;
int sige_tile_conv_plan(const sige_tile_conv_t *desc, sige_tile_conv_plan_t *plan);

/* 3x3 / stride 1 / pad 1 convolution with Cin <= 4 (the RGB stem): x NHWC (B,H,W,Cin), w OIHW, out NHWC;
 * up to two extra outputs aux[i] = act(out*scale+shift) (NHWC, Cout channels). */
int sige_conv_in_nhwc(const void *x, const void *w, const void *bias, void *out, int dtype, int B,
                      int H, int W, int Cin, int Cout, int n_aux, const sige_conv_aux_t *aux,
                      sige_stream_t stream);
/* The same stem evaluated only inside a list of R x S pixel tiles (tile t = rows idx[2t] .. +R-1, columns idx[2t+1] ..
 * +S-1; pixels outside the image are skipped).  idx_per_image == 0: the same n_tiles tiles in every image of the batch;
 * 1: idx holds B*n_tiles entries, row b*n_tiles + i = tile i of image b (see sige_tile_conv_t.idx_per_image).  When every consumer
 * of the stem reads it through Gather with one index set (reference sige/nn/gather.py:76-89), nothing else is read. */
int sige_conv_in_nhwc_tiles(const void *x, const void *w, const void *bias, void *out, int dtype, int B,
                            int H, int W, int Cin, int Cout, const int32_t *idx, int n_tiles, int R, int S,
                            int idx_per_image, int n_aux, const sige_conv_aux_t *aux, sige_stream_t stream);
/* GroupNorm statistics folded to per-channel fp32 (scale, shift) [B, C]: GroupNorm(x) == x*scale + shift.
 * Deterministic two-stage reduction; `workspace` holds sige_group_norm_fold_workspace(B, C) floats, which is -1 (and the
 * error is set) when that count exceeds 2^31 - 1.  H * W < 2^31. */
int sige_group_norm_fold_workspace(int B, int C);
int sige_group_norm_fold(const void *x, int dtype, int B, int H, int W, int C, int groups, float eps,
                         const void *gamma, const void *beta, float *scale, float *shift,
                         float *workspace, int workspace_floats, sige_stream_t stream);
/* out(NCHW, B x Cout x H x W) = conv3x3_pad1( act(x*scale + shift) ), Cout <= 8, C % 16 == 0; scale/shift fp32 [B, C] or NULL. */
int sige_conv_out_nhwc(const void *x, const float *scale, const float *shift, int act, const void *w,
                       const void *bias, void *out, int dtype, int B, int H, int W, int C, int Cout,
                       sige_stream_t stream);
/* Dense single-head attention core of the DDPM AttnBlock (reference diffusion/models/ddpm_arch/sige_fused_unet.py:185-199,
 * the torch bmm / softmax / bmm between the qkv and proj_out 1x1 convolutions) on NHWC tokens:
 *   qkv [B][N][3C] = per pixel [q | k | v], q ALREADY multiplied by C^-0.5;  out [B][N][C] = softmax(q k^T) v.
 * N in {64, 128, 256} tokens, C in {256, 512}, f16 / bf16 (sige_attention_tokens_supported() tells).
 * flags: SIGE_CONV_PDL = programmatic dependent launch, as for sige_tile_conv. */
int sige_attention_tokens_supported(int N, int C, int dtype);
int sige_attention_tokens(const void *qkv, void *out, int B, int N, int C, int dtype, int flags,
                          sige_stream_t stream);

/* Multi-head attention core for SPARSE queries (Stable Diffusion's transformer blocks in sparse mode): the reference's
 * torch.bmm(q, k^T) * scale -> softmax(-1) -> torch.bmm(., v) of stable-diffusion/ldm/modules/attention.py:81-93 (attn1: queries =
 * tokens of the active tiles, keys / values = all tokens of the scattered tensor, sige_attention.py:79,153-160) and
 * sige_attention.py:44-58 (attn2: the same queries against the text keys / values cached by the dense pass), as one launch;
 * the [Nq x Nk] logits never reach HBM.
 *   out[b, h, i, :] = softmax_j(scale * q[b, h, i, :] . k[b, h, j, :]) v[b, h, j, :]
 * Element strides {batch, head, token} per operand, the head dim D contiguous — so both the reference's "(b h) n d" copies
 * (heads = 1, B = b*h) and the "b n (h d)" layout the Linear layers produce are addressable without a rearrange.
 * D in {32, 40, 64, 80, 128, 160, 512}, f16 / bf16 (sige_sparse_attention_supported() tells); strides multiples of 8 elements,
 * buffers 16-byte aligned; scale > 0; Nq == 0 is a no-op.  D = 512 (the single head of the Stable Diffusion VAE's mid-block
 * attention) splits the key range over a thread-block cluster and merges the partial softmax statistics in the same launch. */
typedef struct {
    const void *q;               /* Nq query tokens per (batch, head) */
    const void *k, *v;           /* Nk key / value tokens per (batch, head) */
    void *out;                   /* same shape as q */
    int B, heads, Nq, Nk, D;
    long long q_stride[3], k_stride[3], v_stride[3], out_stride[3];
    float scale;
    int dtype;
    int flags;                   /* reserved, 0 */
} sige_sparse_attention_t;
int sige_sparse_attention_supported(int D, int dtype);
int sige_sparse_attention(const sige_sparse_attention_t *p, sige_stream_t stream);

/* SPADE's modulation of a tile stack (or any channels-innermost tensor of `pixels` pixels), one launch:
 *   out = act(x * (1 + gamma) + beta),  act = leaky_relu(negative_slope)  (negative_slope = 1: identity)
 * — the four pointwise torch calls of reference gaugan/models/sige_normalization.py:84-86 plus the block's F.leaky_relu(., 0.2)
 * (gaugan/models/spade_generators/sige_fused_spade_generator.py:200-201) on the gathered tiles.  Every operand has its own pixel
 * stride in elements (gamma and beta are the channel halves of one [pixels, 2C] tensor); C and the strides multiples of one
 * 16-byte vector, buffers 16-byte aligned; f32 / f16 / bf16; fp32 arithmetic. */
int sige_spade_modulate(const void *x, long long x_pixel_stride, const void *gamma, long long gamma_pixel_stride,
                        const void *beta, long long beta_pixel_stride, void *out, long long out_pixel_stride,
                        long long pixels, int C, float negative_slope, int dtype, sige_stream_t stream);

/* Separable convolution of GAN Compression's sub-mobile SPADE on the active tiles, one launch per SPADE layer:
 *   out_b = conv1x1_b( dwconv3x3_b(x) * scale_b + shift_b ),   b < nbranch (gamma and beta read the same input)
 * — per branch the depthwise SIGEConv2d (groups = Cin), the folded instance norm and the 1x1 SIGEConv2d of reference
 * gaugan/models/mobile_modules.py:108-112, and the Scatter / ScatterGather behind them (gaugan/models/sige_normalization.py:157-165):
 * the 4x4 outputs of every 6x6 halo tile are pasted IN PLACE into the branch's destination.  The affine is folded by the caller:
 * dw_weight = scale * w, dw_bias = scale * b + shift.
 * Source: a channel window [src_c0, src_c0 + Cin) of an NHWC buffer [B, H, W, src_C] read through `idx` (zero outside the image;
 * SIGE_TILE_NONE tiles read zeros and write nothing), or of a tile stack [B*N, 6, 6, src_C] (row b*N + i).  Destination: channels
 * [dst_c0, dst_c0 + Cout) of an NHWC buffer [B, dH, dW, dst_C] at (idx + off), or a stack [B*N, 4, 4, dst_C].  With a tile list, a
 * SIGE_TILE_NONE entry writes nothing to either kind of destination: its stack row keeps its contents (whatever a stack source
 * holds in that row is read and discarded).  A stack-to-stack launch may pass idx = NULL: every row is then a tile.
 * Cin a multiple of 16 in [16, 256], Cout a multiple of 8 in [8, 1024], f16 / bf16 (sige_separable_conv_supported() tells, k = 3);
 * channel counts and offsets multiples of 8; buffers 16-byte aligned.  flags: SIGE_CONV_PDL, SIGE_CONV_PER_IMAGE_OPERANDS (a batch of
 * independent edits: `idx` holds B*N rows, row b*N + i = tile i of image b, for a buffer source and buffer destinations); other
 * bits are ignored. */
typedef struct {
    const float *dw_weight; /* fp32 [Cin][3][3], affine folded */
    const float *dw_bias;   /* fp32 [Cin] or NULL */
    const void *pw_weight;  /* [Cout][Cin] in dtype */
    const float *pw_bias;   /* fp32 [Cout] or NULL */
    void *dst;
    int dst_is_stack;
    int dH, dW, dst_C, dst_c0;
} sige_separable_branch_t;
typedef struct {
    int dtype;
    const void *src;
    int src_is_stack;
    int src_C, src_c0;
    int B, H, W;            /* source extent (NHWC buffer source) */
    const int32_t *idx;     /* [N,2] halo-tile origins in the source frame */
    int N;                  /* tiles per image */
    int Cin, Cout;
    int offH, offW;         /* output origin = idx + off */
    int nbranch;            /* 1 or 2 */
    sige_separable_branch_t branch[2];
    int flags;
} sige_separable_conv_t;
int sige_separable_conv_supported(int Cin, int Cout, int k, int dtype);
int sige_separable_conv(const sige_separable_conv_t *p, sige_stream_t stream);

/* ------------------------------------------------------------------------- */
/* a8: sparse_update write-back (reference sige/nn/scatter.py:59-60,114-129,  */
/*     sige/nn/scatter_gather.py:65-77)                                        */
/* ------------------------------------------------------------------------- */
/* Copies the output tiles of many NHWC buffers into their caches, one launch.  Entry e: tile i of image b (b < B) writes rows
 * [(idx_h + offH) / strideH, + Ro) and columns [(idx_w + offW) / strideW, + So) — sige_scatter's paste rule, C division —
 * clipped to the image, every channel, from `src` (NHWC [B, H, W, C], f16 / bf16) into `dst` (the same logical [B, C, H, W] in
 * dst_layout; dst_dtype SIGE_F32 or src_dtype, so every conversion is exact).  SIGE_TILE_NONE entries write nothing, so a
 * fixed-capacity list may be passed whole.  An entry with N == 0 is skipped and its pointers are not looked at.  C a multiple
 * of 8, Ro and So in [1, 8], buffers 16-byte aligned.  At most SIGE_WRITEBACK_MAX_ENTRIES entries per call (the table travels
 * in the launch's parameters); every entry is validated before any device call. */
#define SIGE_WRITEBACK_MAX_ENTRIES 64
typedef struct {
    const void *src;
    void *dst;
    const int32_t *idx;     /* [N,2] tile origins */
    int N, B, C, H, W;
    int src_dtype, dst_dtype, dst_layout;
    int offH, offW, strideH, strideW, Ro, So;
} sige_writeback_entry_t;
int sige_tile_writeback(const sige_writeback_entry_t *entries, int n_entries, sige_stream_t stream);

/* ------------------------------------------------------------------------- */
/* cache load: the cached buffers of a fused step from the module caches     */
/* ------------------------------------------------------------------------- */
/* Entry e reads `src`, a cache [src_batch, C, H, W] (dense in src_layout, f32 / f16 / bf16), once, and writes
 *   raw          NHWC [E, H, W, C] in `dtype`: the cache rounded to nearest (NULL: none);
 *   view[k].dst  NHWC [E, H, W, C] in `dtype`: act(cache * scale[c] + shift[c]) for k < n_views, scale / shift fp32 [C] or NULL,
 *                act SIGE_ACT_IDENTITY or SIGE_ACT_SWISH.
 * A source of one image (src_batch == 1) is written to all E images; otherwise src_batch == E and image i goes to image i.
 * Arithmetic in fp32, each operation rounded (no contraction): z * scale, then + shift, then swish as z * (1 / (1 + expf(-z))).
 * C a multiple of 8, destinations 16-byte aligned and not overlapping any source.  At most SIGE_CACHE_LOAD_MAX_ENTRIES entries
 * per call (the table travels in the launch's parameters); every entry is validated before any device call; n_entries == 0
 * does nothing. */
#define SIGE_CACHE_LOAD_MAX_ENTRIES 64
typedef struct {
    void *dst;
    const float *scale, *shift;
    int act;
} sige_cache_view_t;
typedef struct {
    const void *src;
    int src_dtype, src_layout, src_batch;
    int C, H, W, E;
    void *raw;
    int n_views;
    sige_cache_view_t view[2];
} sige_cache_load_entry_t;
int sige_cache_load(const sige_cache_load_entry_t *entries, int n_entries, int dtype, sige_stream_t stream);

/* ------------------------------------------------------------------------- */
/* diagnostics                                                                */
/* ------------------------------------------------------------------------- */
/* In-kernel timeline: while `buf` (device int64, 16 slots per CTA of the NEXT sige_tile_conv launch that takes the wgmma
 * path) is set, that launch stamps %globaltimer per CTA — slot 0 entry, 3 dependency resolved (griddepcontrol.wait returned), 4 halo stored,
 * 5/6 MMA issue begin/end, 7 accumulators out of registers, 8/9 every partial row present (split-K: exchange landed),
 * 10 stores of thread 0 issued, 11 exit (every thread's stores issued); slot 12 holds the number of halo fills of the
 * CTA's K slice (a count, not a time); slot 13 the early chunks of the slice gathered (SIGE_CONV_EARLY_*; 0 without any).  The pointer is baked into the launch's
 * kernel parameters (so it survives CUDA-graph capture); call again (NULL to stop) before the next launch.  bench.py derives
 * the in-step roofline from these stamps; returns 0. */
int sige_debug_set_trace(void *buf);

/* Halo buffers of split-K narrow 3x3 wgmma launches from now on: 0 = chosen per launch from its K slices (default), 1 = the
 * single-buffered layout, 2 = the double-buffered one.  Both compute the same sums in the same order, so the outputs are
 * bitwise equal; for tests.  Returns 0, or non-zero for any other n. */
int sige_debug_set_split_halo_buffers(int n);

#ifdef __cplusplus
}
#endif
#endif /* SIGE_B200_H_ */
