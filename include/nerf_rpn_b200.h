/*
 * nerf_rpn_b200.h -- C ABI of the NeRF-RPN hot path (libnerf_rpn_b200.so).
 *
 * The reference (lyclyc52/NeRF_RPN) has no FFI registry: its drop-in surface is Python module paths plus
 * ONE native pybind module, `sort_vertices` (nerf_rpn/model/rotated_iou/cuda_op/sort_vert.cpp:6-34).
 * This header is what a binding for the hot path links against.  Every entry point
 *   - takes plain device pointers / sizes and a CUDA stream (no torch types),
 *   - is stream-ordered and never synchronises the device or the host,
 *   - owns no caller memory (the caller allocates inputs, outputs and workspaces),
 *   - returns 0 on success or a negative nrpn_status; it never calls exit() (the reference's
 *     CUDA_CHECK_ERRORS does, cuda_utils.h:26-35).
 * All pointers are device pointers unless marked "host".  Kernels are compiled for sm_90a (H100) only.
 */
#ifndef NERF_RPN_B200_H
#define NERF_RPN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void *nrpn_stream_t; /* cudaStream_t */

typedef enum {
    NRPN_OK = 0,
    NRPN_ERR_INVALID = -1,      /* bad argument (null pointer, negative size, unsupported box_dim ...) */
    NRPN_ERR_UNSUPPORTED = -2,  /* shape outside what the kernels were built for */
    NRPN_ERR_WORKSPACE = -3,    /* workspace too small */
    NRPN_ERR_CUDA = -4,         /* CUDA runtime / driver error (see nrpn_last_cuda_error) */
    NRPN_ERR_NO_DEVICE = -5     /* no sm_90 device or driver entry point unavailable */
} nrpn_status;

int nrpn_version(void);
const char *nrpn_status_string(int status);
/* last cudaError_t observed by this library on the calling thread (0 if none). */
int nrpn_last_cuda_error(void);
/* Number of kernels this library has launched since load (bench.py's gpu_launches). */
unsigned long long nrpn_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * Box overlap.  Boxes are fp32 rows of box_dim floats:
 *   box_dim == 6: axis-aligned (x1,y1,z1,x2,y2,z2)        -- nerf_rpn/model/utils.py:418-458
 *   box_dim == 7: yaw-oriented (x,y,z,w,h,d,theta)        -- nerf_rpn/model/rotated_iou/oriented_iou_loss.py:82-107
 * ---------------------------------------------------------------------------------------------- */

/* iou[i] = IoU3D(a[i], b[i]).  Replaces cal_iou_3d on (1,n,7)x(1,n,7) (oriented_iou_loss.py:82) and the
 * element-wise AABB case. */
int nrpn_iou3d_pairs(const float *a, const float *b, int n, int box_dim, float *iou, nrpn_stream_t stream);

/* cal_iou_3d(box3d1, box3d2, verbose=True) (oriented_iou_loss.py:82-107) for n pairs of oriented boxes: IoU, the two corner sets
 * (n, 4, 2), z_range = extent of the union of the z ranges, u3d = V1 + V2 - intersection -- the inputs of the IoU-type regression losses
 * (rpn.py:133-165, fcos/loss.py). */
int nrpn_iou3d_pairs_verbose(const float *a, const float *b, int n, float *iou, float *corners1, float *corners2, float *z_range,
                             float *u3d, nrpn_stream_t stream);
/* Backward of (iou, u3d) w.r.t. both boxes (the reference differentiates its torch chain with autograd; the vertex order is not
 * differentiated there either, cuda_ext.py:10): grad_a / grad_b (n, 7) = grad_iou * d iou + grad_u3d * d u3d; either upstream gradient
 * may be NULL.  The intersection volume is differentiated by central differences in fp64 (piecewise smooth; DESIGN.md 3.3). */
int nrpn_iou3d_pairs_backward(const float *a, const float *b, int n, const float *grad_iou, const float *grad_u3d, float *grad_a,
                              float *grad_b, nrpn_stream_t stream);

/* out[i*m + j] = IoU3D(a[i], b[j]).  Replaces box_iou_3d (utils.py:387-415), which tiles both sets to
 * (n,m,7) in HBM and runs ~40 ATen kernels plus the native sort. */
int nrpn_iou3d_matrix(const float *a, int n, const float *b, int m, int box_dim, float *out, nrpn_stream_t stream);

/* Drop-in for the reference's only native op on the path:
 *   sort_vertices.sort_vertices_forward(vertices (b,n,m,2) f32, mask (b,n,m) bool, num_valid (b,n) i32)
 *       -> idx (b,n,9) i32                                   -- cuda_op/sort_vert.cpp:6-34
 * m must be <= 32 (the reference always passes 24). */
int nrpn_sort_vertices(const float *vertices, const uint8_t *mask, const int32_t *num_valid, int b, int n, int m,
                       int32_t *idx, nrpn_stream_t stream);

/* Rounding order of the oriented-IoU chain (csrc/box_iou.cuh).  The reference runs it as ~40 ATen kernels whose libm and reduction
 * orders differ between its CPU and CUDA builds: bit 0 = operation order of the torch-CUDA kernels (bmm as fma, 4-accumulator /
 * tree sums), bit 1 = CUDA sinf / cosf instead of fp64-rounded sin / cos.  Default 3: bit-identical to the reference running on
 * the same GPU (tests/test_gpu_reference.py); 0: bit-identical to oracle/box_oracle.c's default (the reference's CPU build).
 * Process-wide; takes effect for launches issued after the call (synchronous 4-byte copy to the device). */
int nrpn_set_iou_mode(int mode);
int nrpn_get_iou_mode(void);

/* Greedy NMS, per group, fully on device (no host round trip per kept box as in utils.py:215-230).
 *   boxes  (n, box_dim) f32, scores (n) f32, group (n) i32 in [0,255] or NULL (single group)
 *   keep   (n) i64 out: indices kept, sorted by score descending (ties: lower index first)
 *   n_keep (1) i32 out (device)
 * A pair (i,j) with score_i >= score_j of the same group suppresses j when !(IoU(box_i, box_j) <= thr)
 * (utils.py:228).  Equivalent to batched_nms (utils.py:233-265); with group == NULL, to nms().
 * n <= nrpn_nms_max_boxes().  workspace: nrpn_nms_workspace_bytes(n) bytes, 256-byte aligned. */
int nrpn_nms_max_boxes(void);
size_t nrpn_nms_workspace_bytes(int n);
int nrpn_nms(const float *boxes, int box_dim, const float *scores, const int32_t *group, int n, float thr,
             int64_t *keep, int32_t *n_keep, void *workspace, size_t workspace_bytes, nrpn_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * 3-D convolution as an implicit GEMM on wgmma tensor cores (replaces every nn.Conv3d (+BatchNorm3d
 * +ReLU +residual / FPN top-down add) on the path: feature_extractor.py:31-68,145-235, anchor.py:177-213).
 *
 * Layouts (all bf16 unless stated):
 *   x  : (N, X, Y, Z, Cin)   channels-last, Cin % 64 == 0; the reference's NCDHW (N,C,W,L,H) permuted
 *   w  : (taps, CoutPad, Cin) one K-major (Cout x Cin) matrix per filter tap, BN scale pre-multiplied,
 *        CoutPad = Cout rounded up to the kernel's N tile (nrpn_conv3d_block_n)
 *   shift : (CoutPad) fp32   bias or folded BN shift
 *   y  : (N, Xo, Yo, Zo, ldy) bf16 or fp32 (out_fp32), first Cout channels of each row written
 *   res: optional (N, Xr, Yr, Zr, ldr) bf16 added before the activation; when its extent differs from
 *        the output it is read through nearest-neighbour up-sampling (F.interpolate(size=..), fpn top-down)
 * Output voxel o takes input voxel  o * stride + tap_offset[t] (zero outside the grid), so padding and
 * dilation are expressed by the tap table.  Up to NRPN_CONV_MAX_LEVELS problems that share w/shift
 * (the RPN head applied to P2..P5) are executed by ONE persistent launch.
 * ---------------------------------------------------------------------------------------------- */
#define NRPN_CONV_MAX_LEVELS 4
#define NRPN_CONV_MAX_TAPS 64

typedef struct {
    const void *x;      /* bf16 */
    void *y;            /* bf16 or fp32 */
    const void *res;    /* bf16 or NULL */
    int32_t n;          /* batch */
    int32_t xi, yi, zi; /* input extent */
    int32_t xo, yo, zo; /* output extent */
    int32_t xr, yr, zr; /* residual extent (ignored when res == NULL) */
    int32_t ldy;        /* output row pitch in elements */
    int32_t ldr;        /* residual row pitch in elements */
} nrpn_conv_level;

typedef struct {
    int32_t cin, cout;              /* cin % 64 == 0 */
    int32_t n_taps;                 /* 1 .. NRPN_CONV_MAX_TAPS */
    int8_t tap_off[NRPN_CONV_MAX_TAPS][3]; /* per tap (dx,dy,dz) input offset */
    int32_t stride;                 /* 1 or 2 (same on all axes) */
    int32_t relu;                   /* final activation: 0 none, 1 ReLU, 2 exact (erf) GELU */
    int32_t out_fp32;               /* y is fp32 */
    const void *w;                  /* bf16 (taps, CoutPad, cin) */
    const float *shift;             /* fp32 (CoutPad) */
    int32_t n_levels;
    nrpn_conv_level level[NRPN_CONV_MAX_LEVELS];
    void *workspace;                /* optional split-K scratch (see nrpn_conv3d_workspace_bytes) or NULL */
    size_t workspace_bytes;
    int32_t act_fp16;               /* 16-bit format of x / w / res / 16-bit y: 0 = bf16, 1 = fp16 (IEEE half) */
    int32_t wsplit;                 /* 1: w is (taps, 2, CoutPad, cin) = every weight as the sum hi + lo of two 16-bit numbers (both
                                     * planes are multiplied with the same activation tile into one fp32 accumulator): the weights
                                     * then contribute no 16-bit rounding error -- the <= 1e-3 feature-map parity mode */
} nrpn_conv_desc;

/* Padding granularity of the output-channel axis for this cout (64, 128 or 256): w / shift must be padded to a multiple. */
int nrpn_conv3d_block_n(int cout);
/* Name of the kernel variant nrpn_conv3d_fprop would launch for this descriptor ("slab<4x16x8,N64>", "igemm<256,4,1>", ...;
 * "invalid" / "unsupported" when it would be rejected).  Pure host logic: pointers inside the descriptor are not dereferenced. */
const char *nrpn_conv3d_variant(const nrpn_conv_desc *desc);
/* Layers with few output tiles and a long reduction are split along K over several CTAs; each stores its partial tile
 * into its own fp32 slab and the last CTA to arrive sums the slabs in a fixed order (bit-reproducible).  Returns the
 * bytes such a layer wants (0: the layer is not split).  The first 256-byte-aligned counters region must be zero-filled
 * ONCE by the caller (simplest: zero the whole buffer); every launch leaves the counters at zero, so one buffer can serve
 * all layers of a stream.  Passing workspace == NULL (or too small) is legal: the layer then runs unsplit. */
size_t nrpn_conv3d_workspace_bytes(const nrpn_conv_desc *desc /*host*/);
int nrpn_conv3d_fprop(const nrpn_conv_desc *desc /*host*/, nrpn_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Bandwidth-bound helpers around the convolutions.
 * ---------------------------------------------------------------------------------------------- */

/* Stem input packing: fp32 NCDHW grid (4, X, Y, Z) as the reference feeds the backbone (datasets.py:55-57,
 * nerf_rpn.py:210) -> bf16 (ceil(X/2), ceil(Y/2), ceil(Z/2)+1, 64): a 2x2x2 space-to-depth block (32 ch)
 * of voxel (i,j,k-1) followed by the block of voxel (i,j,k), k in [0, ceil(Z/2)] (so the packed Z extent is
 * ceil(Z/2)+1); turns the 7^3 stride-2 stem conv (feature_extractor.py:163) into a 4x4x2-tap stride-1
 * implicit GEMM with K = 64 per tap. */
int nrpn_pack_stem_input(const float *grid, int n, int x, int y, int z, void *packed, int act_fp16,
                         int channels_last /* 0: grid is (N,4,X,Y,Z); 1: (N,X,Y,Z,4) as stored on disk, datasets.py:49-57 */,
                         nrpn_stream_t stream);

/* Same, with density_to_alpha = 1 applying the reference dataset's --normalize_density map to the last channel on the device:
 * alpha = clip(1 - exp(-exp(sigma) / 100), 0, 1) (datasets.py:50-52,165-167), fused into the read of the grid. */
int nrpn_pack_stem_input_ex(const float *grid, int n, int x, int y, int z, void *packed, int act_fp16, int channels_last,
                            int density_to_alpha, nrpn_stream_t stream);

/* Same packing from a raw uint8 grid in its on-disk order (N,X,Y,Z,4): bytes are normalised by / 255 on the device, as
 * datasets.py:59-61 does on the host (.float() / 255.0); a quarter of the fp32 host-to-device traffic. */
int nrpn_pack_stem_input_u8(const uint8_t *grid_xyzc, int n, int x, int y, int z, void *packed, int act_fp16, nrpn_stream_t stream);

/* F.max_pool3d(kernel 3, stride 2, padding 1) on (N,X,Y,Z,C) bf16, C % 8 == 0 (feature_extractor.py:219). */
int nrpn_maxpool3d_k3s2(const void *in, int n, int x, int y, int z, int c, void *out, int act_fp16, nrpn_stream_t stream);

/* nn.MaxPool3d(kernel 2, stride 2, ceil_mode=True) (VGG stages, feature_extractor.py:347): output extent ceil(in/2). */
int nrpn_maxpool3d_k2s2_ceil(const void *in, int n, int x, int y, int z, int c, void *out, int act_fp16, nrpn_stream_t stream);

/* Stride-1 stem packing for VGG_FPN on grids smaller than 160 (Conv3d(4,64,kernel 7,stride 1,padding 3),
 * feature_extractor.py:341): fp32 NCDHW (4,X,Y,Z) -> bf16 (X, Y+1, Z, 64); row (x,yp,z) = the 7 z-neighbours of the two
 * input rows y = yp-1, yp (56 channels + 8 zero), so that the conv is a 7x4-tap implicit GEMM with K = 64 per tap. */
int nrpn_pack_stem_input_s1(const float *grid, int n, int x, int y, int z, void *packed, int act_fp16, nrpn_stream_t stream);

/* GroupNorm(32 groups, 256 channels) + optional ReLU, in place, on up to NRPN_CONV_MAX_LEVELS channels-last bf16 tensors
 * (N, voxels, 256) that share gamma/beta (FCOS towers: Conv3d -> GroupNorm -> ReLU, fcos/fcos.py:43-69).  Statistics are
 * per (sample, level, group); reductions run in a fixed order (bit-reproducible). */
typedef struct {
    void *x;          /* bf16 (N, voxels, 256), normalised in place */
    int32_t voxels;
} nrpn_gn_level;
size_t nrpn_groupnorm_workspace_bytes(int n_levels, int n);
int nrpn_groupnorm_relu(const nrpn_gn_level *levels /*host*/, int n_levels, int n, int c, int groups, const float *gamma,
                        const float *beta, float eps, int relu, int act_fp16, void *workspace, size_t workspace_bytes,
                        nrpn_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * RPN post-processing (rpn.py:292-370, anchor.py:51-122, coder/AABB_coder.py:86-137,
 * coder/midpoint_offset_coder.py:160-223, utils.py:268-367) for ONE scene, fully on device.
 * ---------------------------------------------------------------------------------------------- */
#define NRPN_RPN_MAX_LEVELS 4

typedef struct {
    const float *pred;   /* (X*Y*Z, ld) fp32 rows: [A logits | A*code deltas | pad], anchor-major deltas */
    int32_t ld;
    int32_t gx, gy, gz;  /* feature grid */
    int32_t sx, sy, sz;  /* anchor stride = mesh // grid (anchor.py:160-162) */
} nrpn_rpn_level;

typedef struct {
    int32_t n_levels;
    nrpn_rpn_level level[NRPN_RPN_MAX_LEVELS];
    int32_t num_anchors;              /* A, anchors per location (<= 16) */
    float cell_anchors[NRPN_RPN_MAX_LEVELS][16][6]; /* rounded half extents, anchor.py:51-82 */
    int32_t rotated;                  /* 0: 6 deltas -> AABB, 1: 8 deltas -> OBB */
    int32_t pre_nms_top_n;            /* per level */
    int32_t post_nms_top_n;
    float nms_thresh, score_thresh, min_size;
    int32_t mesh[3];                  /* (padded) mesh extent used for clipping */
    int32_t valid[3];                 /* original extent (padding mask, anchor.py:124-152); == mesh if unpadded */
} nrpn_rpn_desc;

size_t nrpn_rpn_workspace_bytes(const nrpn_rpn_desc *desc /*host*/);
/* Outputs: boxes (post_nms_top_n, 6|7) f32, scores (post_nms_top_n) f32, levels (post_nms_top_n) f32
 * (the reference returns the level id as a float column), count (1) i32. */
int nrpn_rpn_proposals(const nrpn_rpn_desc *desc /*host*/, float *boxes, float *scores, float *levels,
                       int32_t *count, void *workspace, size_t workspace_bytes, nrpn_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Swin-3D support (SwinTransformer_FPN, feature_extractor.py:382-789). Token grids are channels-last bf16 (N,H,W,D,ld) with
 * C real channels, ld >= C; the Linear layers run through nrpn_conv3d_fprop as 1x1x1 convolutions.
 * ---------------------------------------------------------------------------------------------- */
/* fp32 NCDHW grid (N,4,X,Y,Z) -> bf16 (N, X/4, Y/4, Z/4, 256) patch rows, channel ((c*4+px)*4+py)*4+pz: the patch embedding
 * Conv3d(4, C, kernel 4, stride 4) becomes a 256 -> C GEMM. */
int nrpn_patch_embed_pack(const float *grid, int n, int x, int y, int z, void *out, int act_fp16, nrpn_stream_t stream);
/* per-token LayerNorm over the first c channels of each row; rows are ld_in / ld_out elements apart. */
int nrpn_layernorm(const void *in, int ld_in, void *out, int ld_out, long tokens, int c, const float *gamma, const float *beta,
                   float eps, int act_fp16, nrpn_stream_t stream);
/* PatchMerging front half: 2x2x2 gather (zero past odd extents) + LayerNorm(8c) -> (N, ceil(h/2), ceil(w/2), ceil(d/2), 8c). */
int nrpn_patch_merge_ln(const void *in, int ld_in, int n, int h, int w, int d, int c, void *out, const float *gamma,
                        const float *beta, float eps, int act_fp16, nrpn_stream_t stream);
/* 4x4x4 (shifted) window multi-head attention, head_dim 32: qkv (N,h,w,d, 3c) -> out (N,h,w,d, ld_out). shift in {0, 2};
 * table = (343, heads) relative position bias table; qkv_bias (3c) stands in for zero-padded tokens. */
int nrpn_window_attention(const void *qkv, int ld_qkv, void *out, int ld_out, const float *qkv_bias, const float *table, int n,
                          int h, int w, int d, int c, int heads, int shift, int act_fp16, nrpn_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * FCOS (anchor-free) post-processing for ONE scene (fcos/fcos.py:116-126,221-250; fcos/inference.py:48-195;
 * fcos/utils.py:12-61), fully on device: head transform (Scale, ReLU, x stride), sigmoid, candidate selection, centerness
 * weighting, per-level top-k, AABB / midpoint-offset OBB decode, clip, min-size, one NMS over all levels, k-th value cap.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    const float *cls;    /* (X*Y*Z, ld_cls) fp32 rows, channel 0 = raw class logit */
    const float *reg;    /* (X*Y*Z, ld_reg) fp32 rows, channels [0,6|8) = raw distances (+ alpha, beta), next = raw centerness */
    int32_t ld_cls, ld_reg;
    int32_t gx, gy, gz;
    int32_t stride;      /* FPN stride of the level: locations = idx*stride + stride/2 */
    float scale;         /* the level's learnable Scale */
} nrpn_fcos_level;

typedef struct {
    int32_t n_levels;
    nrpn_fcos_level level[NRPN_RPN_MAX_LEVELS];
    int32_t use_obb;
    int32_t pre_nms_top_n, post_nms_top_n;
    float pre_nms_thresh, nms_thresh, min_size;
    int32_t grid_size[3];     /* the scene's own extent (clipping, padding mask) */
    int32_t padded;           /* 1: batch > 1, mask locations outside grid_size (fcos.py:252-266) */
} nrpn_fcos_desc;

/* capacity (rows) the outputs must have: sum over levels of min(pre_nms_top_n, locations) -- the k-th value cut keeps ties,
 * so more than post_nms_top_n rows can come back. */
int nrpn_fcos_max_proposals(const nrpn_fcos_desc *desc /*host*/);
size_t nrpn_fcos_workspace_bytes(const nrpn_fcos_desc *desc /*host*/);
/* boxes (cap, 1+6|7) f32 with the level id in column 0, scores (cap) f32, count (1) i32. */
int nrpn_fcos_proposals(const nrpn_fcos_desc *desc /*host*/, float *boxes, float *scores, int32_t *count, void *workspace,
                        size_t workspace_bytes, nrpn_stream_t stream);

/* ------------------------------------------------------------------------------------------------ recall metric
 * Greedy proposal <-> ground-truth matching of evaluate_box_proposals_recall (eval.py:33-52) on device.
 * overlaps: (n_proposals, n_gt) fp32 IoU matrix (nrpn_iou3d_matrix of the score-sorted, limit-truncated proposals against the
 * ground truth); gt_overlaps: min(n_proposals, n_gt) fp32, the IoU recorded at each step of the reference loop (the rest of
 * the reference's zero-initialised vector is left to the caller).  Ties: lowest ground-truth index, then lowest proposal
 * index, as torch.max on CPU.  n_proposals <= 262 144, n_gt <= 4 096. */
int nrpn_recall_match(const float *overlaps, int n_proposals, int n_gt, float *gt_overlaps, nrpn_stream_t stream);
/* Row-wise maximum and first arg-max of a (rows, cols) fp32 matrix (torch.max(dim=1) tie rule): the per-detection step of
 * evaluate_box_proposals_ap (eval.py:355-358) for a whole scene's IoU matrix. */
int nrpn_rowmax_f32(const float *m, int rows, int cols, float *maxv, int32_t *argmax, nrpn_stream_t stream);

/* ------------------------------------------------------------------------------------------------ training targets
 * RegionProposalNetwork.assign_targets_to_anchors (rpn.py:240-290): IoU of every anchor with every (rectified, obb2hbb_3d)
 * ground-truth box, Matcher(high, low, allow_low_quality_matches) (utils.py:98-212) and the label mapping, without the
 * (G, N) matrix.  anchors (N,6) f32 [x1,y1,z1,x2,y2,z2]; gt (G,6) AABB or (G,7) OBB; valid: optional (N) u8 padding mask
 * (0 = anchor in a padded voxel: enters the matcher as -1.0, label -1).  labels (N) f32 in {1, 0, -1}; matched_idxs (N) i64:
 * the matcher's output (GT index, -1 below low, -2 between thresholds); gather gt[clamp(idx, 0)] for the matched boxes.
 * Any G (ground truth streamed through shared memory in chunks of 1 024).  G == 0 is the caller's "background mesh" case (rpn.py:246-250) and is rejected here. */
size_t nrpn_assign_targets_workspace_bytes(int n_anchors, int n_gt);
int nrpn_assign_targets(const float *anchors, int n_anchors, const float *gt, int n_gt, int gt_dim, const uint8_t *valid,
                        float high_threshold, float low_threshold, int allow_low_quality_matches, float *labels,
                        int64_t *matched_idxs, void *workspace, size_t workspace_bytes, nrpn_stream_t stream);

/* ------------------------------------------------------------------------------------------------ weight gradient
 * dW[tap][co][ci] = sum_v dY[v][co] * X[v + tap_off][ci] of a stride-1 convolution (training, SURVEY.md 8(a) a18) on wgmma.
 * operand_layout 1 (what the training engine uses): both operands are read channels-last where they live (MN-major wgmma operands).
 * operand_layout 0: both operands in PLANAR layout (N, C, X, Y, z_pitch), 16-bit (nrpn_transpose_to_planar converts a channels-last tensor);
 * levels that share the weights (RPN head on P2..P5) accumulate into the same dW.  dw: fp32 (taps, cout, cin), overwritten.
 * cout % 128 == 0; cin % 32 == 0, cin <= 256; tap z offsets in {-1, 0, +1}.  Deterministic (fixed-order reduction of the K-split partial tiles). */
typedef struct {
    const void *dy_planar;   /* (N, cout, X, Y, z_pitch) bf16 / fp16 */
    const void *x_planar[3]; /* (N, cin,  X, Y, z_pitch): copies shifted along z, [k][z] = x[z + (k - 1)], zero outside; NULL if no tap has dz = k - 1 */
    int32_t n, x, y, z;
    int32_t z_pitch;         /* >= z + 1, multiple of 8; positions without a source MUST be zero (pre-zeroed buffers) */
    /* operand_layout == 1: the operands where they live, channels-last 16-bit (N, X, Y, Z, ld); no copies, no staging buffers */
    const void *dy_cl;       /* (N, x, y, z, ld_dy >= cout) */
    const void *x_cl;        /* (N, xx, xy, xz, ld_x >= cin): the layer input, same grid as dY unless xx / xy / xz say otherwise */
    int32_t ld_dy, ld_x;     /* row pitches in elements, multiples of 8 */
    int32_t xx, xy, xz;      /* extents of X when they differ from (x, y, z); 0 = same */
} nrpn_wgrad_level;

typedef struct {
    int32_t cin, cout, n_taps;
    int8_t tap_off[NRPN_CONV_MAX_TAPS][3];
    int32_t n_levels;
    nrpn_wgrad_level level[NRPN_CONV_MAX_LEVELS];
    float *dw;
    void *workspace;
    size_t workspace_bytes;
    int32_t act_fp16;
    int32_t dw_layout;       /* 0: dw is (taps, Cout, Cin); 1: dw is (Cout, Cin, taps) = nn.Conv3d.weight's own memory order */
    int32_t accumulate;      /* 1: dw += result (a weight shared by several launches) */
    int32_t operand_layout;  /* 0: planar copies (dy_planar / x_planar); 1: channels-last tensors (dy_cl / x_cl) read through MN-major descriptors */
} nrpn_wgrad_desc;

size_t nrpn_conv3d_wgrad_workspace_bytes(const nrpn_wgrad_desc *desc /*host*/);
int nrpn_conv3d_wgrad(const nrpn_wgrad_desc *desc /*host*/, nrpn_stream_t stream);
/* channels-last (N, X, Y, Z, ld >= c) 16-bit -> planar (N, c, X, Y, z_pitch >= Z); columns [Z, z_pitch) are left untouched
 * (pre-zero the buffer once) */
int nrpn_transpose_to_planar(const void *in_cl, int n, int x, int y, int z, int c, int ld, void *out_planar, int z_pitch,
                             int z_shift /* out[z'] = in[z' + z_shift] */, nrpn_stream_t stream);

/* Pointwise pieces of a conv + bias + ReLU layer's backward pass (training building blocks):
 * db[c] = sum over rows of dY[row][c] (fixed-order two-stage reduction, bit-reproducible); dY *= (act > 0) in place. */
size_t nrpn_bias_grad_workspace_bytes(int c);
int nrpn_bias_grad(const void *dy_cl /* (rows, ld >= c) 16-bit */, long rows, int c, int ld, int act_fp16, float *db, void *workspace,
                   size_t workspace_bytes, nrpn_stream_t stream);
int nrpn_relu_backward(void *dy_cl, const void *act_cl, size_t elements /* % 8 == 0 */, int act_fp16, nrpn_stream_t stream);


/* ------------------------------------------------------------------------------------------------
 * Training step (row a18, BASELINE config 4): everything of the reference's `loss.backward(); clip_grad_norm_; optimizer.step()`
 * (run_rpn.py:384-395) that is not one of the three GEMMs above.  Channels-last 16-bit activations / gradients (rows, c),
 * c % 8 == 0; all reductions run in a fixed order (bit-reproducible).
 * ---------------------------------------------------------------------------------------------- */
size_t nrpn_chan_reduce_workspace_bytes(int c);
/* nn.BatchNorm3d in train mode, statistics half (feature_extractor.py:38-43 under model.train()): stats = {mean[c], rstd[c],
 * biased var[c]} over `rows`; when running_mean/var are given they are updated with `momentum` (unbiased variance) like torch. */
int nrpn_bn_stats(const void *y, long rows, int c, int act_fp16, float eps, float *stats /*3c*/, float *running_mean,
                  float *running_var, float momentum, void *workspace, size_t workspace_bytes, nrpn_stream_t stream);
/* out = act(gamma * (y - mean) * rstd + beta (+ res)): normalise (+ residual, Bottleneck.forward :61-66) (+ ReLU) */
int nrpn_bn_apply(const void *y, const void *res, void *out, long rows, int c, const float *stats, const float *gamma,
                  const float *beta, int relu, int act_fp16, nrpn_stream_t stream);
/* Backward of [BatchNorm (+ residual) (+ ReLU)]: g = dout * (act > 0 when relu); sums = {sum g * xhat = dgamma [c], sum g = dbeta [c]};
 * dy = gamma * rstd * (g - sum g / rows - xhat * sum(g xhat) / rows); dres (optional) = g, the gradient of the skip branch. */
int nrpn_bn_backward(const void *dout, const void *act, const void *y, void *dy, void *dres, long rows, int c, const float *stats,
                     const float *gamma, float *sums /*2c*/, int relu, int act_fp16, void *workspace, size_t workspace_bytes,
                     nrpn_stream_t stream);
/* F.max_pool3d(3, 2, 1) with the recorded argmax (one byte per output element: window position of the first maximum) and its
 * backward as a deterministic gather over the <= 8 windows that contain an input voxel (feature_extractor.py:219). */
int nrpn_maxpool3d_k3s2_argmax(const void *in, int n, int x, int y, int z, int c, void *out, uint8_t *idx, int act_fp16, nrpn_stream_t stream);
int nrpn_maxpool3d_k3s2_backward(const void *dy, const uint8_t *idx, int n, int x, int y, int z, int c, void *dx, int act_fp16, nrpn_stream_t stream);
/* Backward of the FPN top-down merge fine += nearest_upsample(coarse) (feature_extractor.py:211-213): dcoarse (+)= sum of dfine over
 * the fine voxels whose source index floor(f * coarse / fine) is the coarse voxel (same float expression as the forward epilogue). */
int nrpn_upsample_nearest_backward(const void *dfine, int n, int xf, int yf, int zf, int xc, int yc, int zc, int c, void *dcoarse,
                                   int accumulate, int act_fp16, nrpn_stream_t stream);
/* Stride-2 1^3 convolutions (first block of ResNet stages 2-4): scatter = 0: dst (ceil/2 extents) = src sub-sampled at even
 * voxels (the wgrad operand); scatter = 1: dst (x,y,z) = src (ceil/2 extents) zero-stuffed (the data gradient). */
int nrpn_stride2(const void *src, void *dst, int n, int x, int y, int z, int c, int scatter, nrpn_stream_t stream);
int nrpn_add_inplace(void *a, const void *b, size_t elements, int act_fp16, nrpn_stream_t stream);
/* RPN losses of one mesh on its sampled anchors (rpn.py:372-417, smooth-L1 branch) and their gradient w.r.t. the predictor output.
 * desc: level geometry as for nrpn_rpn_proposals (pred = fp32 (voxels, 128) rows [A logits | A*code deltas]); dpred[l]: 16-bit
 * (voxels, 128) tensors, ZERO-FILLED by the caller; pos_idx / neg_idx: flat anchor indices (rpn.py:20-27 order) of the sampled
 * positives / negatives; gt_pos (n_pos, 6|7): their matched ground-truth boxes (encoded on the fly: AABB_coder.py:14-56 /
 * midpoint_offset_coder.py:106-158); norm = sampled anchors of the whole batch.  losses[0] += BCE sum / norm, losses[1] +=
 * smooth-L1(beta 1/9) sum / norm; dpred = grad_scale * d(w_obj * L_obj + w_reg * L_reg)/dpred.  targets_out (optional, (n_pos,
 * code)): the encoded regression targets (for tests). */
int nrpn_rpn_loss(const nrpn_rpn_desc *desc /*host*/, void *const *dpred /*host array*/, const int64_t *pos_idx, int n_pos,
                  const int64_t *neg_idx, int n_neg, const float *gt_pos, float norm, float w_obj, float w_reg, float grad_scale,
                  float *losses /*2, accumulated*/, float *targets_out, int act_fp16, nrpn_stream_t stream);
/* fp32 master weights (Cout, Cin, taps) -> 16-bit GEMM operands: fwd (taps, fwd_rows >= Cout, fwd_cols >= Cin) and, optionally,
 * the data-gradient operand with mirrored taps and transposed matrices (taps, bwd_rows >= Cin, bwd_cols >= Cout).  Pad regions are
 * not written (zero-fill the buffers once). */
int nrpn_pack_weights(const float *w, int cout, int cin, int taps, void *fwd, int fwd_rows, int fwd_cols, void *bwd, int bwd_rows,
                      int bwd_cols, int act_fp16, nrpn_stream_t stream);
/* out[i] = idx[i] >= 0 ? src[idx[i]] * scale : 0 -- 16-bit (out16) or fp32 (out32): layouts given by a host-built index table
 * (the space-to-depth stem weights and their gradient). */
int nrpn_gather_pack(const float *src, const int32_t *idx, size_t n, void *out16, float *out32, float scale, int act_fp16, nrpn_stream_t stream);
/* norm_out[0] = ||g||_2 * inv_scale (fp64 two-stage reduction) */
size_t nrpn_grad_norm_workspace_bytes(void);
int nrpn_grad_norm(const float *g, size_t n, float inv_scale, float *norm_out, void *workspace, size_t workspace_bytes, nrpn_stream_t stream);
/* torch.nn.utils.clip_grad_norm_(max_norm) (coefficient read from the device: no host sync) fused with torch.optim.AdamW's update
 * on flat fp32 buffers; gradients are multiplied by inv_scale first (loss scaling / world size). */
int nrpn_adamw_step(float *p, const float *g, float *m, float *v, size_t n, const float *norm, float max_norm, float inv_scale, float lr,
                    float beta1, float beta2, float eps, float weight_decay, int step, nrpn_stream_t stream);

/* ------------------------------------------------------------------------------------------------ FCOS training loss
 * FCOSLossComputation (fcos/loss.py:185-591) on the device, in two calls.
 *
 * nrpn_fcos_targets = prepare_targets / compute_targets_for_locations[_obb] / get_sample_region (loss.py:213-441) for ONE scene: every
 * location of every level against every ground-truth box (AABB (G,6) or OBB (G,7): encode_fcos_obb, fcos/utils.py:64-108), centre
 * sampling, the level's object-size range, smallest box wins (first minimum), without the (locations, G, 8) tensors.  locations (P,3)
 * f32 = the levels' compute_locations (fcos.py:221-250) concatenated, P = sum n_points.  labels (P) f32 in {0, 1}; reg_targets
 * (P, 6|8) f32: l, t, f, r, b, ba (divided by the level's stride when norm_reg_targets) + alpha, beta.  n_gt == 0: zeros (loss.py:324-328).
 * Any G (ground truth is streamed through shared memory in chunks). */
typedef struct {
    int32_t n_levels;
    int32_t n_points[NRPN_RPN_MAX_LEVELS];
    int32_t stride[NRPN_RPN_MAX_LEVELS];
    float size_lo[NRPN_RPN_MAX_LEVELS], size_hi[NRPN_RPN_MAX_LEVELS]; /* object_sizes_of_interest (loss.py:263-268): -1,16 / 16,32 / 32,64 / 64,1e8 */
    float center_sampling_radius;                                      /* <= 0: every location strictly inside a box is a candidate */
    int32_t norm_reg_targets;
} nrpn_fcos_target_desc;
int nrpn_fcos_targets(const nrpn_fcos_target_desc *desc /*host*/, const float *locations, const float *gt, int n_gt, int gt_dim,
                      float *labels, float *reg_targets, nrpn_stream_t stream);

/* nrpn_fcos_loss = FCOSLossComputation.__call__ (loss.py:487-591) up to the two normalisers: sigmoid focal loss over every (unmasked)
 * location, and on the positives the centerness target, BCE-with-logits of the centerness branch, the box regression loss weighted by
 * the centerness target (loss_type 0: smooth-L1 on all 6|8 channels; AABB head: 1 -log(iou), 2 1 - iou, 3 1 - giou of IOULoss :78-131)
 * and, for the OBB head with additional_l1, the smooth-L1 of alpha / beta.  For use_obb with loss_type >= 1 the rotated-IoU term itself
 * (RotatedIOULoss :134-181) is NOT computed here: the caller adds it on the gathered positives (cal_iou_3d & co. with their own backward).
 * Per level the head's NCDHW outputs are read where they are: cls (N,1,P_l), reg (N,6|8,P_l), ctr (N,1,P_l) fp32; d* (same shapes,
 * all three NULL for a forward-only call) receive the UN-normalised gradients of sums[0], sums[3] + sums[5], sums[4] (zeros where none).
 * labels (N,P) / reg_targets (N,P,6|8): nrpn_fcos_targets per scene; mask (N,P) u8 or NULL: compute_padding_masks (0 = dropped).
 * centerness_targets (N,P) f32 or NULL: the positives' centerness target (0 elsewhere).
 * sums[8] (device, fp64, fixed-order reduction): 0 focal sum, 1 positives, 2 sum of centerness targets, 3 weighted regression sum,
 * 4 centerness BCE sum, 5 weighted alpha/beta smooth-L1 sum, 6-7 zero.  The caller all-reduces [1], [2] over the ranks and divides
 * (loss.py:541-576): loss_cls = [0] / max([1]/W, 1), loss_reg = ([3] + [5]) / ([2]/W), loss_centerness = [4] / max([1]/W, 1). */
typedef struct {
    const float *cls, *reg, *ctr;
    float *dcls, *dreg, *dctr;
    int32_t n_points;
} nrpn_fcos_loss_level;
typedef struct {
    int32_t n_levels;
    nrpn_fcos_loss_level level[NRPN_RPN_MAX_LEVELS];
    int32_t n_images, use_obb, loss_type, additional_l1;
} nrpn_fcos_loss_desc;
size_t nrpn_fcos_loss_workspace_bytes(void);
int nrpn_fcos_loss(const nrpn_fcos_loss_desc *desc /*host*/, const float *labels, const float *reg_targets, const uint8_t *mask,
                   float *centerness_targets, double *sums, void *workspace, size_t workspace_bytes, nrpn_stream_t stream);

/* Which necessary-condition tests may skip the exact polygon clip inside NMS (process-wide; initial value from NRPN_NMS_CULL_MODE, default 0):
 *   0  exact-zero culls only (bounding circles / z ranges disjoint: the reference computes exactly 0) -- the keep set is provably the reference's;
 *   1  + volume-ratio and z-overlap-ratio culls, 3  + footprint-lens cull: geometric bounds, applied from 16 384 boxes up only.  The reference's
 *      vertex sort can report MORE than the geometric IoU in rare degenerate cases (DESIGN.md 3.3), so these modes may differ from it in about
 *      1e-5 of the boxes; they make the 1 M-box sweep 4-5x faster. */
void nrpn_set_nms_cull_mode(int mode);
int nrpn_get_nms_cull_mode(void);

/* Diagnostics of the cell-list NMS path (n >= 16 384 boxes): cumulative counters since the last reset -- out16[0..4] for the cross passes
 * (records streamed, record x query pair slots, exact IoU evaluations, hits, work items), out16[8..12] the same for the adjacency passes.  Synchronises. */
int nrpn_nms_cells_stats(unsigned long long *out16, int reset);

/* Training-time augmentation of one scene on the device (BaseDataset.augment_rpn_inputs + rotate_and_scale_scene, datasets.py:109-163,
 * 290-329, z-up): fp32 grid in its on-disk channels-last order (X, Y, Z, 4) -> out (Xo, Yo, Z, 4), Xo/Yo = Y/X when rot90 else X/Y.
 * rot90: transpose(x, y) + flip(x); flip_x / flip_y; resample: F.grid_sample(trilinear, zero padding, align_corners=True) of the
 * scene rotated by `angle` about z and scaled by `scale` exactly as the reference builds its sampling grid.  The box transforms are a
 * few scalars per box and stay on the host side (nerf_rpn_b200/augment.py). */
int nrpn_augment_scene(const float *grid_xyzc, int x, int y, int z, float *out_xyzc, int rot90, int flip_x, int flip_y, int resample,
                       float angle, float scale, nrpn_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* NERF_RPN_B200_H */
