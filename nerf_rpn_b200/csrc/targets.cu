// Anchor <-> ground-truth assignment for training (SURVEY.md 8(a) a18 / 8(f) rank 3): the fused replacement of
//   RegionProposalNetwork.assign_targets_to_anchors (rpn.py:240-290) = obb2hbb_3d (coder/misc.py:85-93) +
//   batched_box_iou in chunks of 16 GT (utils.py:371-384, the (G, 2.43 M) fp32 matrix) + Matcher with
//   allow_low_quality_matches (utils.py:98-212) + label mapping.
// The (G, N) match-quality matrix is never materialised: pass 1 keeps, per anchor, the best IoU and its (first) GT index in
// registers and folds the per-GT maxima through shared memory into G global atomics per CTA; pass 2 recomputes the IoUs with
// the same code (bit-identical) to find the anchors that tie a GT's maximum ("low-quality matches", ties included) and
// writes labels {1, 0, -1} and the matcher's index {>= 0, -1 below, -2 between}.
// IoU arithmetic = iou3d_aabb (utils.py:418-458 order: boxes1 = GT, boxes2 = anchor), anchors outside the padding mask
// enter the matcher as -1.0 and end with label -1 (rpn.py:260-263, 284-286).
#include "box_iou.cuh"
#include "anchor_mask.cuh"

namespace nrpn {

constexpr int kTgtThreads = 256;
constexpr int kTgtPerThread = 4;
constexpr int kTgtMaxGt = 1024;

struct TgtDev {
    const float* anchors; int n;
    const float* gt6; int g;                  // rectified ground truth (G, 6), device
    const uint8_t* valid;                     // per-anchor padding mask (1 = real) or null
    float high, low; int allow_low;
    float* best_val; int* best_idx; unsigned* gmax;
    float* labels; long long* matched;
};

// obb2hbb_3d: smallest AABB containing the OBB (cos / sin through fp64, rounded once).
__global__ void tgt_rectify_kernel(const float* __restrict__ gt, int g, int dim, float* __restrict__ out, unsigned* __restrict__ gmax) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= g) return;
    gmax[i] = 0u;                             // below every ordered float
    if (dim == 6) {
#pragma unroll
        for (int k = 0; k < 6; ++k) out[i * 6 + k] = gt[i * 6 + k];
        return;
    }
    const float* b = gt + (size_t)i * 7;
    const float x = b[0], y = b[1], z = b[2], w = b[3], h = b[4], d = b[5], th = b[6];
    const float co = (float)cos((double)th), si = (float)sin((double)th);
    const float hw = __fdiv_rn(w, 2.0f), hh = __fdiv_rn(h, 2.0f);
    const float xb = __fadd_rn(fabsf(__fmul_rn(hw, co)), fabsf(__fmul_rn(hh, si)));
    const float yb = __fadd_rn(fabsf(__fmul_rn(hw, si)), fabsf(__fmul_rn(hh, co)));
    const float zb = __fdiv_rn(d, 2.0f);
    out[i * 6 + 0] = __fsub_rn(x, xb); out[i * 6 + 1] = __fsub_rn(y, yb); out[i * 6 + 2] = __fsub_rn(z, zb);
    out[i * 6 + 3] = __fadd_rn(x, xb); out[i * 6 + 4] = __fadd_rn(y, yb); out[i * 6 + 5] = __fadd_rn(z, zb);
}

template <int PASS>
__global__ void __launch_bounds__(kTgtThreads) tgt_match_kernel(TgtDev P) {
    __shared__ float sgt[kTgtMaxGt][6];
    __shared__ unsigned smax[kTgtMaxGt];          // pass 1: CTA-local per-GT maxima; pass 2: the global maxima
    const int t = threadIdx.x, lane = t & 31;
    const long base = ((long)blockIdx.x * kTgtThreads) * kTgtPerThread;
    float a[kTgtPerThread][6];
    bool live[kTgtPerThread], masked[kTgtPerThread];
    float best[kTgtPerThread]; int arg[kTgtPerThread]; bool tie[kTgtPerThread];
#pragma unroll
    for (int u = 0; u < kTgtPerThread; ++u) {
        const long i = base + (long)u * kTgtThreads + t;           // coalesced: consecutive threads, consecutive anchors
        live[u] = i < P.n;
        masked[u] = live[u] && P.valid != nullptr && P.valid[i] == 0;
#pragma unroll
        for (int k = 0; k < 6; ++k) a[u][k] = live[u] ? P.anchors[i * 6 + k] : 0.0f;
        best[u] = -INFINITY; arg[u] = 0; tie[u] = false;
    }
    // the ground truth goes through shared memory in chunks of kTgtMaxGt boxes (one chunk for every scene of the reference's datasets)
    for (int g0 = 0; g0 < P.g; g0 += kTgtMaxGt) {
        const int gc = min(kTgtMaxGt, P.g - g0);
        if (g0 > 0) __syncthreads();
        for (int i = t; i < gc * 6; i += kTgtThreads) sgt[i / 6][i % 6] = P.gt6[(size_t)g0 * 6 + i];
        for (int i = t; i < gc; i += kTgtThreads) smax[i] = (PASS == 1) ? 0u : P.gmax[g0 + i];
        __syncthreads();
        for (int g = 0; g < gc; ++g) {
            float m = -INFINITY;
#pragma unroll
            for (int u = 0; u < kTgtPerThread; ++u) {
                if (!live[u]) continue;
                const float iou = masked[u] ? -1.0f : iou3d_aabb(sgt[g], a[u]);
                if (PASS == 1) {
                    if (iou > best[u]) { best[u] = iou; arg[u] = g0 + g; }     // first maximum, like torch.max on CPU
                    m = fmaxf(m, iou);
                } else {
                    tie[u] = tie[u] || (float_to_ordered(iou) == smax[g]);
                }
            }
            if (PASS == 1) {
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
                if (lane == 0 && m > -INFINITY) atomicMax(&smax[g], float_to_ordered(m));
            }
        }
        if (PASS == 1) {
            __syncthreads();
            for (int i = t; i < gc; i += kTgtThreads) if (smax[i]) atomicMax(&P.gmax[g0 + i], smax[i]);
        }
    }
    if (PASS == 1) {
#pragma unroll
        for (int u = 0; u < kTgtPerThread; ++u) {
            const long i = base + (long)u * kTgtThreads + t;
            if (live[u]) { P.best_val[i] = best[u]; P.best_idx[i] = arg[u]; }
        }
    } else {
#pragma unroll
        for (int u = 0; u < kTgtPerThread; ++u) {
            const long i = base + (long)u * kTgtThreads + t;
            if (!live[u]) continue;
            const float v = P.best_val[i];
            const int idx = P.best_idx[i];
            long long mt = idx;
            if (v < P.low) mt = -1;
            else if (v < P.high) mt = -2;
            if (P.allow_low && tie[u]) mt = idx;
            float lab = mt >= 0 ? 1.0f : (mt == -1 ? 0.0f : -1.0f);
            if (masked[u]) lab = -1.0f;
            P.labels[i] = lab;
            P.matched[i] = mt;
        }
    }
}

// One byte per (scene, flat anchor); the level geometry is shared, the limits are per scene.
struct MaskParams {
    AnchorMaskLevel lv[kMaskMaxLevels];
    int lim[NRPN_STEM_MAX_SCENES][kMaskMaxLevels][3];
    int n_levels, num_anchors;
    long long total;
};

__global__ void anchor_padding_mask_kernel(const __grid_constant__ MaskParams P, int n, uint8_t* __restrict__ mask) {
    const long long all = (long long)n * P.total;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < all; e += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(e / P.total);
        mask[e] = anchor_mask_value(P.lv, P.lim[b], P.n_levels, P.num_anchors, e - (long long)b * P.total);
    }
}

}  // namespace nrpn

using namespace nrpn;

extern "C" {
#pragma GCC visibility push(default)

size_t nrpn_assign_targets_workspace_bytes(int n_anchors, int n_gt) {
    if (n_anchors < 0 || n_gt < 0) return 0;
    return align_up((size_t)n_anchors * 4, 256) * 2 + align_up((size_t)n_gt * 4, 256) + align_up((size_t)n_gt * 24, 256) + 256;
}

int nrpn_assign_targets(const float* anchors, int n_anchors, const float* gt, int n_gt, int gt_dim, const uint8_t* valid, float high,
                        float low, int allow_low_quality, float* labels, int64_t* matched_idxs, void* workspace, size_t workspace_bytes,
                        nrpn_stream_t stream) {
    if (n_anchors < 0 || n_gt < 0 || (gt_dim != 6 && gt_dim != 7) || !(low <= high)) return NRPN_ERR_INVALID;
    if (n_anchors == 0) return NRPN_OK;
    if (n_gt == 0) return NRPN_ERR_INVALID;          // the reference handles empty targets before the matcher (rpn.py:246-250)
    if (!anchors || !gt || !labels || !matched_idxs || !workspace) return NRPN_ERR_INVALID;
    if (workspace_bytes < nrpn_assign_targets_workspace_bytes(n_anchors, n_gt)) return NRPN_ERR_WORKSPACE;
    char* b = reinterpret_cast<char*>(align_up((size_t)workspace, 256));
    TgtDev P;
    P.anchors = anchors; P.n = n_anchors; P.g = n_gt; P.valid = valid; P.high = high; P.low = low; P.allow_low = allow_low_quality;
    P.best_val = reinterpret_cast<float*>(b); b += align_up((size_t)n_anchors * 4, 256);
    P.best_idx = reinterpret_cast<int*>(b); b += align_up((size_t)n_anchors * 4, 256);
    P.gmax = reinterpret_cast<unsigned*>(b); b += align_up((size_t)n_gt * 4, 256);
    float* gt6 = reinterpret_cast<float*>(b);
    P.gt6 = gt6; P.labels = labels; P.matched = reinterpret_cast<long long*>(matched_idxs);
    cudaStream_t st = (cudaStream_t)stream;
    tgt_rectify_kernel<<<ceil_div(n_gt, 128), 128, 0, st>>>(gt, n_gt, gt_dim, gt6, P.gmax);
    NRPN_LAUNCH_CHECK();
    const int blocks = ceil_div(n_anchors, kTgtThreads * kTgtPerThread);
    tgt_match_kernel<1><<<blocks, kTgtThreads, 0, st>>>(P);
    NRPN_LAUNCH_CHECK();
    tgt_match_kernel<2><<<blocks, kTgtThreads, 0, st>>>(P);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

int nrpn_anchor_padding_mask(const int32_t* ori_sizes, int n, int px, int py, int pz, const int32_t* grid_dims, int n_levels, int num_anchors,
                             uint8_t* mask, nrpn_stream_t stream) {
    if (!ori_sizes || !grid_dims || !mask || n < 1 || n > NRPN_STEM_MAX_SCENES || n_levels < 1 || n_levels > kMaskMaxLevels || num_anchors < 1)
        return NRPN_ERR_INVALID;
    const int pad[3] = {px, py, pz};
    MaskParams P;
    P.n_levels = n_levels; P.num_anchors = num_anchors;
    long long begin = 0;
    for (int l = 0; l < n_levels; ++l) {
        P.lv[l].begin = begin;
        for (int a = 0; a < 3; ++a) {
            const int g = grid_dims[3 * l + a];
            if (g < 1 || pad[a] < g) return NRPN_ERR_INVALID;
            P.lv[l].grid[a] = g;
        }
        begin += (long long)num_anchors * P.lv[l].grid[0] * P.lv[l].grid[1] * P.lv[l].grid[2];
    }
    P.total = begin;
    for (int i = 0; i < n; ++i)
        for (int l = 0; l < n_levels; ++l)
            for (int a = 0; a < 3; ++a) {
                const int o = ori_sizes[3 * i + a];
                if (o < 1 || o > pad[a]) return NRPN_ERR_INVALID;
                P.lim[i][l][a] = anchor_mask_limit(o, pad[a], P.lv[l].grid[a]);
            }
    const long long all = (long long)n * P.total;
    const long long blocks = (all + 255) / 256;
    const int cap = num_sms() * 16;
    anchor_padding_mask_kernel<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, (cudaStream_t)stream>>>(P, n, mask);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

#pragma GCC visibility pop
}  // extern "C"
