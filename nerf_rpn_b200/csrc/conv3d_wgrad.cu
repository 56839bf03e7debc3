// Weight gradient of a stride-1 'same' 3-D convolution on wgmma (training, SURVEY.md 8(a) a18):
//     dW[tap][co][ci] = sum over voxels v   dY[v][co] * X[v + tap_offset][ci]
// The contraction runs over VOXELS, for which channels-last activations (a voxel's channels are contiguous) are MN-major operands:
// both tensors are read where they live, channels-last (N, X, Y, Z, ld), through MN-major shared-memory descriptors.  A TMA box
// {64 channels, bz, by, bx} of 64 voxels lands in shared memory as 64 rows of 128 bytes (128B swizzle) -- which IS the canonical MN-major
// operand layout of wgmma (SWIZZLE_128B: 64 channels contiguous per voxel row, 8 rows per 1024-byte swizzle atom, SBO = 1024 bytes between
// groups of 8 voxels, LBO = the distance between two 64-channel boxes), selected by the instruction's transpose flags.  No transposed copies,
// no zero-filled staging buffers: the tap offset is a plain coordinate shift of the X box and TMA's out-of-bounds zero fill is the convolution
// padding.
// D (128 x NT, fp32 in registers of two warpgroups) += A * B^T with A = dY box pair (128 output channels x 64 voxels), B = X boxes shifted by the tap
// (n_t input channels x 64 voxels).  Work item = (tap group, Cout slice(s), Cin slice, K-split); every item streams its share of the voxel bricks
// of all pyramid levels that share the weights (the RPN head on P2..P5) and writes fp32 partial tiles; a second kernel sums them in a fixed order
// (bit-reproducible) into dW (taps, Cout, Cin) or nn.Conv3d.weight's own (Cout, Cin, taps) order.
#include <cstdio>
#include <cstring>
#include <type_traits>
#include "common.cuh"
#include "wgmma.cuh"
#include "conv_internal.cuh"

namespace nrpn {

constexpr int kWgConsumers = 256;               // two warpgroups: output channels 0-63 / 64-127 of the slice
constexpr int kWgThreads = kWgConsumers + 32;   // + the TMA producer warp

// Stores the consumer warpgroup's rows of an accumulator (128 x NT, columns >= n_t are padding) as one fp32 partial tile.
template <int NT>
__device__ __forceinline__ void store_partial(float* tile, int n_t, int wg, int t, const float (&acc)[NT / 2], bool empty) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float* out = tile + (size_t)(wg * 64 + ptx::frag_row(t, h)) * n_t;
#pragma unroll
        for (int j = 0; j < NT / 8; ++j) {
            const int col = ptx::frag_col(t, j);
            if (col < n_t)
                *reinterpret_cast<float2*>(out + col) = empty ? make_float2(0.f, 0.f) : make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
    }
}

// dW[tap][co][ci] = sum over splits (fixed order) of the partial tiles
// layout 0: dw (taps, Cout, Cin);  layout 1: dw (Cout, Cin, taps) = nn.Conv3d.weight's own memory order (taps = kx*ky*kz row-major)
__global__ void wgrad_reduce_kernel(const float* __restrict__ partial, int n_taps, int m_tiles, int n_tiles, int splits, int n_t, int cout, int cin,
                                    float* __restrict__ dw, int layout) {
    const size_t total = (size_t)n_taps * cout * cin;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
        const int ci = (int)(t % cin); size_t v = t / cin;
        const int co = (int)(v % cout); const int tap = (int)(v / cout);
        const int mt = co >> 7, row = co & 127, nt = ci / n_t, col = ci - nt * n_t;
        const float* p = partial + (((((size_t)tap * m_tiles + mt) * n_tiles + nt) * splits) * 128 + row) * n_t + col;
        float s = 0.f;
        for (int sp = 0; sp < splits; ++sp) s += p[(size_t)sp * 128 * n_t];
        const size_t o = layout ? ((size_t)co * cin + ci) * n_taps + tap : t;
        dw[o] = s;
    }
}

struct WgLevel { int n, nxb, nyb, nzb, bx, by, bz, brick_begin; };
struct WgDev {
    int n_levels, n_taps, cin, cout, n_t, m_tiles, n_tiles, splits, total_bricks, fp16, b_boxes;
    int m_pair, m_items, stages;           // Cout slices per work item (1 or 2: two accumulators share one X tile), items along Cout, ring depth
    int t_group, n_groups;                 // taps per work item (their accumulators share one dY tile), tap groups
    signed char tap[NRPN_CONV_MAX_TAPS][4];
    WgLevel lv[NRPN_CONV_MAX_LEVELS];
    float* partial;                        // [tap][m_tile][n_tile][split][128][n_t]
};
struct WgMaps { CUtensorMap dy[NRPN_CONV_MAX_LEVELS]; CUtensorMap x[NRPN_CONV_MAX_LEVELS]; };
constexpr int kWgBox = 64 * 128;               // one {64 channels x 64 voxels} box, 16-bit
constexpr int kWgMaxStages = 4;
constexpr int kWgAccRegs = 128;                // accumulator registers per consumer thread: m_pair * t_group * NT / 2 <= this

// NT = 64 * b_boxes input channels per accumulator (columns >= n_t are TMA zero fill), NACC >= m_pair * t_group accumulators per work item
// (accumulator m * t_group + i = Cout slice m of the pair x tap i of the group).  With Cout >= 256 two 128-channel slices of Cout share the
// same X tile and a tap group shares one dY tile: the kernel is bound by the shared-memory fill rate out of L2, and sharing cuts it.
template <int NT, int NACC>
__global__ void __launch_bounds__(kWgThreads, 1) conv3d_wgrad_cl_kernel(const __grid_constant__ WgMaps maps, const WgDev P) {
    static_assert(NT * NACC / 2 <= kWgAccRegs, "accumulator registers");
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int a_boxes = 2 * P.m_pair;
    const int stage_bytes = (a_boxes + P.t_group * P.b_boxes) * kWgBox;
    const int stages = P.stages;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + stages * stage_bytes);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + kWgMaxStages;
    const int warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) {
        for (int s = 0; s < stages; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], 2); }
        ptx::fence_barrier_init();
        for (int l = 0; l < P.n_levels; ++l) { ptx::prefetch_tmap(&maps.dy[l]); ptx::prefetch_tmap(&maps.x[l]); }
    }
    __syncthreads();
    const int items = P.n_groups * P.m_items * P.n_tiles * P.splits;

    if (warp == kWgConsumers / 32) {
        const bool leader = ptx::elect_one();
        int stage = 0; uint32_t phase = 0;
        for (int item = blockIdx.x; item < items; item += gridDim.x) {
            const int split = item % P.splits;
            const int nt = (item / P.splits) % P.n_tiles;
            const int mi = (item / (P.splits * P.n_tiles)) % P.m_items;
            const int tap0 = (item / (P.splits * P.n_tiles * P.m_items)) * P.t_group;
            const int ntap = P.n_taps - tap0 < P.t_group ? P.n_taps - tap0 : P.t_group;        // taps of this item: tap0 .. tap0 + ntap - 1
            const int b0 = (int)(((long)P.total_bricks * split) / P.splits), b1 = (int)(((long)P.total_bricks * (split + 1)) / P.splits);
            for (int b = b0; b < b1; ++b) {
                int l = 0;
#pragma unroll
                for (int i = 1; i < NRPN_CONV_MAX_LEVELS; ++i) if (i < P.n_levels && b >= P.lv[i].brick_begin) l = i;
                const WgLevel& L = P.lv[l];
                int t = b - L.brick_begin;
                const int zb = t % L.nzb; t /= L.nzb;
                const int yb = t % L.nyb; t /= L.nyb;
                const int xb = t % L.nxb; const int nb = t / L.nxb;
                const int z0 = zb * L.bz, y0 = yb * L.by, x0 = xb * L.bx;
                ptx::mbar_wait(&empty_bar[stage], phase ^ 1u);
                if (leader) {
                    uint8_t* sa = smem + stage * stage_bytes;
                    ptx::mbar_expect_tx(&full_bar[stage], (uint32_t)((a_boxes + ntap * P.b_boxes) * kWgBox));
                    for (int j = 0; j < a_boxes; ++j)          // Cout slice (mi * m_pair + j / 2), 64-channel half j % 2 (beyond Cout: zero-filled)
                        ptx::tma_load_5d(sa + j * kWgBox, &maps.dy[l], &full_bar[stage], (mi * P.m_pair) * 128 + 64 * j, z0, y0, x0, nb);
                    for (int ti = 0; ti < ntap; ++ti) {        // one X tile per tap of the group: the tap is a coordinate shift
                        const int dx = P.tap[tap0 + ti][0], dy = P.tap[tap0 + ti][1], dz = P.tap[tap0 + ti][2];
                        for (int j = 0; j < P.b_boxes; ++j)
                            ptx::tma_load_5d(sa + (a_boxes + ti * P.b_boxes + j) * kWgBox, &maps.x[l], &full_bar[stage], nt * P.n_t + 64 * j, z0 + dz, y0 + dy,
                                             x0 + dx, nb);
                    }
                }
                __syncwarp();
                if (++stage == stages) { stage = 0; phase ^= 1u; }
            }
        }
        return;
    }

    const int t = threadIdx.x & 127, wg = threadIdx.x >> 7;       // warpgroup wg: output channels 64 wg .. 64 wg + 63 of each slice
    int stage = 0; uint32_t phase = 0;
    float acc[NACC][NT / 2];
    for (int item = blockIdx.x; item < items; item += gridDim.x) {
        const int split = item % P.splits;
        const int nt = (item / P.splits) % P.n_tiles;
        const int mi = (item / (P.splits * P.n_tiles)) % P.m_items;
        const int tap0 = (item / (P.splits * P.n_tiles * P.m_items)) * P.t_group;
        const int ntap = P.n_taps - tap0 < P.t_group ? P.n_taps - tap0 : P.t_group;
        const int b0 = (int)(((long)P.total_bricks * split) / P.splits), b1 = (int)(((long)P.total_bricks * (split + 1)) / P.splits);
#pragma unroll
        for (int am = 0; am < NACC; ++am) ptx::reg_fence(acc[am]);
        for (int b = b0; b < b1; ++b) {
            ptx::mbar_wait(&full_bar[stage], phase);
            const uint32_t sa = ptx::smem_u32(smem + stage * stage_bytes);
            auto issue = [&](auto f16) {
                ptx::wgmma_fence();
#pragma unroll
                for (int am = 0; am < NACC; ++am) {
                    // NACC == m_pair * t_group, so mp < m_pair always.  In a last tap group with ntap < t_group the surplus accumulators
                    // repeat tap ntap - 1 and are never stored: every MMA is issued, no branch around them (a divergent-looking path
                    // around wgmma makes ptxas serialise the whole chain)
                    const int mp = am / P.t_group, ti = min(am - mp * P.t_group, ntap - 1);
                    const uint64_t da = ptx::make_desc_mn_sw128(sa + (uint32_t)((2 * mp + wg) * kWgBox), kWgBox);
                    const uint64_t db = ptx::make_desc_mn_sw128(sa + (uint32_t)((a_boxes + ti * P.b_boxes) * kWgBox), kWgBox);
#pragma unroll
                    for (int k = 0; k < 4; ++k)      // 16 voxels per MMA = two 1024-byte atoms further along K
                        ptx::Wgmma<NT, decltype(f16)::value>::template ss<1, 1>(acc[am], da + (uint64_t)(128 * k), db + (uint64_t)(128 * k),
                                                                                 ((b - b0) | k) ? 1u : 0u);
                }
                ptx::wgmma_commit();
            };
            if (P.fp16) issue(std::true_type{}); else issue(std::false_type{});
            ptx::wgmma_wait<0>();
            if (t == 0) ptx::mbar_arrive(&empty_bar[stage]);
            if (++stage == stages) { stage = 0; phase ^= 1u; }
        }
#pragma unroll
        for (int am = 0; am < NACC; ++am) {
            ptx::reg_fence(acc[am]);
            const int mp = am / P.t_group, ti = am - mp * P.t_group;
            const int mt = mi * P.m_pair + mp, tap = tap0 + ti;
            if (mp >= P.m_pair || ti >= ntap || mt >= P.m_tiles) continue;
            float* tile = P.partial + ((((size_t)tap * P.m_tiles + mt) * P.n_tiles + nt) * P.splits + split) * 128 * P.n_t;
            store_partial<NT>(tile, P.n_t, wg, t, acc[am], b1 <= b0);
        }
    }
}

template <int NT, int NACC>
int launch_wgrad(const WgMaps& maps, const WgDev& P, int grid, int smem, cudaStream_t st) {
    static int smem_set = 0;
    if (smem > smem_set) {
        NRPN_CUDA_TRY(cudaFuncSetAttribute(conv3d_wgrad_cl_kernel<NT, NACC>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        smem_set = smem;
    }
    conv3d_wgrad_cl_kernel<NT, NACC><<<grid, kWgThreads, smem, st>>>(maps, P);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

}  // namespace nrpn

using namespace nrpn;

extern "C" {
#pragma GCC visibility push(default)

// K-splits of a wgrad launch: the work items (taps x Cout slices x Cin slices x splits) run on a persistent grid of one CTA per SM, so the split count
// is chosen for the fullest last wave (3^3 256->256 on 132 SMs: 54 base items; 2 splits = 108 items fill 82 % of one wave, 7 splits = 378 items
// fill 95 % of three waves), smallest count on ties, and at least 8 voxel bricks per split.
static int wgrad_pick_splits(int base, int bricks) {
    const int sms = num_sms();
    int best = 1; double best_util = 0.0;
    const int sp_max = 2 * sms / base + 1 > 32 ? 2 * sms / base + 1 : 32;
    for (int sp = 1; sp <= sp_max; ++sp) {
        if (sp > 1 && bricks / sp < 8) break;
        const long items = (long)base * sp;
        const long waves = (items + sms - 1) / sms;
        const double util = (double)items / (double)(waves * sms);
        if (util > best_util + 0.08) { best_util = util; best = sp; }        // every extra split is another 128 x N fp32 partial tile to write and reduce
    }
    return best;
}

static int pick_box(int extent, int cap) {           // power of two in [1, cap] with the least overhang over `extent`, the larger one on ties
    int best = 1; long waste = -1;
    for (int b = 1; b <= cap; b <<= 1) {
        const long w = (long)ceil_div(extent, b) * b;
        if (waste < 0 || w <= waste) { waste = w; best = b; }
    }
    return best;
}

static int wgrad_plan(const nrpn_wgrad_desc* d, WgDev& P) {
    if (!d || d->n_levels < 1 || d->n_levels > NRPN_CONV_MAX_LEVELS || d->n_taps < 1 || d->n_taps > NRPN_CONV_MAX_TAPS) return NRPN_ERR_INVALID;
    if (d->cout < 8 || d->cout % 8 != 0 || d->cin < 32 || d->cin % 32 != 0 || (d->cin > 256 && d->cin % 256 != 0)) return NRPN_ERR_UNSUPPORTED;
    memset(&P, 0, sizeof(P));
    P.n_levels = d->n_levels; P.n_taps = d->n_taps; P.cin = d->cin; P.cout = d->cout;
    P.n_t = d->cin > 256 ? 256 : d->cin; P.n_tiles = d->cin / P.n_t; P.m_tiles = ceil_div(d->cout, 128);
    P.b_boxes = ceil_div(P.n_t, 64);
    P.m_pair = (P.m_tiles >= 2 && 2 * P.b_boxes * 64 / 2 <= kWgAccRegs) ? 2 : 1;
    P.m_items = ceil_div(P.m_tiles, P.m_pair);
    {
        // taps per work item: their accumulators share one dY tile (the fill rate out of L2 bounds this kernel: 24 KB per four MMAs at N = 64 with one
        // tap, 12 KB with four); as many as the accumulator registers (kWgAccRegs per thread) and a ring of >= 3 stages allow, at most 4
        P.t_group = 1;
        for (int t = 2; t <= 4; t <<= 1) {
            if (t > d->n_taps || P.m_pair * t * P.b_boxes * 64 / 2 > kWgAccRegs) break;
            if ((227 * 1024 - 2048) / ((2 * P.m_pair + t * P.b_boxes) * kWgBox) < 3) break;
            P.t_group = t;
        }
        P.n_groups = ceil_div(d->n_taps, P.t_group);
        const int stage = (2 * P.m_pair + P.t_group * P.b_boxes) * kWgBox;
        int st = (227 * 1024 - 2048) / stage;
        P.stages = st > kWgMaxStages ? kWgMaxStages : st;
        if (P.stages < 2) return NRPN_ERR_UNSUPPORTED;
    }
    P.fp16 = d->act_fp16 ? 1 : 0;
    for (int t = 0; t < d->n_taps; ++t) { P.tap[t][0] = d->tap_off[t][0]; P.tap[t][1] = d->tap_off[t][1]; P.tap[t][2] = d->tap_off[t][2]; P.tap[t][3] = 0; }
    int bricks = 0;
    for (int l = 0; l < d->n_levels; ++l) {
        const nrpn_wgrad_level& S = d->level[l];
        if (S.n < 1 || S.x < 1 || S.y < 1 || S.z < 1 || !S.dy_cl || !S.x_cl || S.ld_dy < d->cout || S.ld_x < d->cin || S.ld_dy % 8 != 0 || S.ld_x % 8 != 0)
            return NRPN_ERR_INVALID;
        WgLevel& L = P.lv[l];
        L.n = S.n;
        L.bz = pick_box(S.z, 64); L.by = pick_box(S.y, 64 / L.bz); L.bx = 64 / (L.bz * L.by);
        L.nzb = ceil_div(S.z, L.bz); L.nyb = ceil_div(S.y, L.by); L.nxb = ceil_div(S.x, L.bx);
        L.brick_begin = bricks;
        bricks += S.n * L.nxb * L.nyb * L.nzb;
    }
    P.total_bricks = bricks;
    const int base = P.n_groups * P.m_items * P.n_tiles;
    P.splits = wgrad_pick_splits(base, bricks);
    return NRPN_OK;
}

static int wgrad_run(const nrpn_wgrad_desc* d, cudaStream_t st) {
    WgDev P;
    { const int rc = wgrad_plan(d, P); if (rc) return rc; }
    WgMaps maps;
    const CUtensorMapDataType dt = d->act_fp16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    for (int l = 0; l < d->n_levels; ++l) {
        const nrpn_wgrad_level& S = d->level[l];
        const WgLevel& L = P.lv[l];
        cuuint32_t box[5] = {64, (cuuint32_t)L.bz, (cuuint32_t)L.by, (cuuint32_t)L.bx, 1};
        // dY: (cout, Z, Y, X, N) with the extents of the OUTPUT grid; X: the input grid (its own extents when they differ)
        const int xz = S.xz > 0 ? S.xz : S.z, xy = S.xy > 0 ? S.xy : S.y, xx = S.xx > 0 ? S.xx : S.x;
        {
            cuuint64_t gdim[5] = {(cuuint64_t)d->cout, (cuuint64_t)S.z, (cuuint64_t)S.y, (cuuint64_t)S.x, (cuuint64_t)S.n};
            const cuuint64_t e = (cuuint64_t)S.ld_dy * 2;
            cuuint64_t gstr[4] = {e, e * S.z, e * S.z * S.y, e * S.z * S.y * S.x};
            const int rc = encode_tmap(&maps.dy[l], S.dy_cl, gdim, gstr, box, dt);
            if (rc) return rc;
        }
        {
            cuuint64_t gdim[5] = {(cuuint64_t)d->cin, (cuuint64_t)xz, (cuuint64_t)xy, (cuuint64_t)xx, (cuuint64_t)S.n};
            const cuuint64_t e = (cuuint64_t)S.ld_x * 2;
            cuuint64_t gstr[4] = {e, e * xz, e * xz * xy, e * xz * xy * xx};
            const int rc = encode_tmap(&maps.x[l], S.x_cl, gdim, gstr, box, dt);
            if (rc) return rc;
        }
    }
    for (int l = d->n_levels; l < NRPN_CONV_MAX_LEVELS; ++l) { maps.dy[l] = maps.dy[0]; maps.x[l] = maps.x[0]; }
    P.partial = reinterpret_cast<float*>(align_up((size_t)d->workspace, 256));
    const int smem = P.stages * (2 * P.m_pair + P.t_group * P.b_boxes) * kWgBox + 1024 + 256;
    const int items = P.n_groups * P.m_items * P.n_tiles * P.splits;
    const int grid = items < num_sms() ? items : num_sms();
    const int nacc = P.m_pair * P.t_group;
    int rc;
    switch (P.b_boxes) {
        case 1: rc = nacc == 1 ? launch_wgrad<64, 1>(maps, P, grid, smem, st) : nacc == 2 ? launch_wgrad<64, 2>(maps, P, grid, smem, st)
                                                                                          : launch_wgrad<64, 4>(maps, P, grid, smem, st); break;
        case 2: rc = nacc == 1 ? launch_wgrad<128, 1>(maps, P, grid, smem, st) : launch_wgrad<128, 2>(maps, P, grid, smem, st); break;
        case 3: rc = launch_wgrad<192, 1>(maps, P, grid, smem, st); break;
        default: rc = launch_wgrad<256, 1>(maps, P, grid, smem, st); break;
    }
    if (rc) return rc;
    const size_t total = (size_t)P.n_taps * P.cout * P.cin;
    size_t blocks = ceil_div(total, (size_t)256);
    if (blocks > (size_t)num_sms() * 8) blocks = (size_t)num_sms() * 8;
    wgrad_reduce_kernel<<<(unsigned)blocks, 256, 0, st>>>(P.partial, P.n_taps, P.m_tiles, P.n_tiles, P.splits, P.n_t, P.cout, P.cin, d->dw,
                                                        d->dw_layout ? 1 : 0);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

size_t nrpn_conv3d_wgrad_workspace_bytes(const nrpn_wgrad_desc* d) {
    WgDev P;
    if (wgrad_plan(d, P) != NRPN_OK) return 0;
    return (size_t)P.n_taps * P.m_tiles * P.n_tiles * P.splits * 128 * P.n_t * sizeof(float) + 256;
}

// "wgrad<NT,NACC>/m<m_pair>/t<t_group>/s<splits>": the instance wgrad_run's switch launches (NT = 64 b_boxes, NACC = m_pair t_group)
// and the plan it runs with.  Pure host logic; the name lives in a per-thread buffer until this thread's next call.
const char* nrpn_conv3d_wgrad_variant(const nrpn_wgrad_desc* d) {
    static thread_local char name[64];
    WgDev P;
    const int rc = wgrad_plan(d, P);
    if (rc == NRPN_ERR_UNSUPPORTED) return "unsupported";
    if (rc != NRPN_OK) return "invalid";
    snprintf(name, sizeof(name), "wgrad<%d,%d>/m%d/t%d/s%d", 64 * P.b_boxes, P.m_pair * P.t_group, P.m_pair, P.t_group, P.splits);
    return name;
}

int nrpn_conv3d_wgrad(const nrpn_wgrad_desc* d, nrpn_stream_t stream) {
    if (!d) return NRPN_ERR_INVALID;
    if (!d->dw || !d->workspace || d->workspace_bytes < nrpn_conv3d_wgrad_workspace_bytes(d)) return NRPN_ERR_WORKSPACE;
    return wgrad_run(d, (cudaStream_t)stream);
}

#pragma GCC visibility pop
}  // extern "C"

// ------------------------------------------------------------------------------------------------ bias gradient, ReLU backward
// The two pointwise pieces of a conv + bias + ReLU layer's backward pass (training building blocks next to dgrad / wgrad):
//   db[c]  = sum over voxels of dY[v][c]           (two-stage, fixed-order reduction: bit-reproducible)
//   dY[v][c] *= (act[v][c] > 0)                     (in place, 16-bit channels-last tensors)
namespace nrpn {

constexpr int kBgBlocks = 256;

__global__ void __launch_bounds__(256) bias_grad_partial_kernel(const __nv_bfloat16* __restrict__ dy, long rows, int c, int ld, int fp16,
                                                                float* __restrict__ partial) {
    // block b sums rows b, b + gridDim.x, ...; thread t owns channels t, t + 256, ...  (any c / ld: the general form)
    for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
        float s = 0.f;
        for (long r = blockIdx.x; r < rows; r += gridDim.x) s += load_act(dy + (size_t)r * ld + ch, fp16);
        partial[(size_t)blockIdx.x * c + ch] = s;
    }
}

// c % 8 == 0, c <= 2048, 16-byte aligned rows: a thread owns 8 channels (one 128-bit load per row) and one of 256 / (c / 8) row lanes; the lanes of a
// block are added in a fixed order through shared memory (bit-reproducible).  (The general form above reads 2 bytes per thread and row: 66 us per
// call on the 187 k x 256 head gradients.)
__global__ void __launch_bounds__(256) bias_grad_partial_vec_kernel(const __nv_bfloat16* __restrict__ dy, long rows, int c, int ld, int fp16,
                                                                    float* __restrict__ partial) {
    extern __shared__ float sm[];                            // [c]
    const int cgs = c >> 3, lanes = 256 / cgs;
    const int cg = threadIdx.x % cgs, lane = threadIdx.x / cgs;
    float s[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) s[k] = 0.f;
    if (lane < lanes) {
        for (long r = (long)blockIdx.x * lanes + lane; r < rows; r += (long)gridDim.x * lanes) {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(dy + (size_t)r * ld + cg * 8));
            const uint32_t* w = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
            for (int k = 0; k < 4; ++k) { const float2 f = unpack_act2(w[k], fp16); s[2 * k] += f.x; s[2 * k + 1] += f.y; }
        }
    }
    for (int i = threadIdx.x; i < c; i += blockDim.x) sm[i] = 0.f;
    __syncthreads();
    for (int l = 0; l < lanes; ++l) {
        if (lane == l) {
#pragma unroll
            for (int k = 0; k < 8; ++k) sm[cg * 8 + k] += s[k];
        }
        __syncthreads();
    }
    for (int i = threadIdx.x; i < c; i += blockDim.x) partial[(size_t)blockIdx.x * c + i] = sm[i];
}

__global__ void __launch_bounds__(256) bias_grad_final_kernel(const float* __restrict__ partial, int blocks, int c, float* __restrict__ db) {
    // 8 channels per CTA, 32 threads per channel (partials b, b + 32, ...), the 32 sums added in a fixed order: bit-reproducible
    __shared__ float red[32][8];
    const int cl = threadIdx.x & 7, kl = threadIdx.x >> 3;
    const int ch = blockIdx.x * 8 + cl;
    float s = 0.f;
    if (ch < c) for (int b = kl; b < blocks; b += 32) s += partial[(size_t)b * c + ch];
    red[kl][cl] = s;
    __syncthreads();
    if (kl != 0 || ch >= c) return;
    s = 0.f;
#pragma unroll
    for (int k = 0; k < 32; ++k) s += red[k][cl];
    db[ch] = s;
}

__global__ void relu_backward_kernel(__nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ act, size_t chunks, int fp16) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < chunks; i += (size_t)gridDim.x * blockDim.x) {
        uint4 g = reinterpret_cast<const uint4*>(dy)[i];
        const uint4 a = __ldg(reinterpret_cast<const uint4*>(act) + i);
        uint32_t* gw = reinterpret_cast<uint32_t*>(&g);
        const uint32_t* aw = reinterpret_cast<const uint32_t*>(&a);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 av = unpack_act2(aw[k], fp16);
            if (!(av.x > 0.f)) gw[k] &= 0xFFFF0000u;
            if (!(av.y > 0.f)) gw[k] &= 0x0000FFFFu;
        }
        reinterpret_cast<uint4*>(dy)[i] = g;
    }
}

}  // namespace nrpn

extern "C" {
#pragma GCC visibility push(default)

size_t nrpn_bias_grad_workspace_bytes(int c) { return c < 1 ? 0 : (size_t)nrpn::kBgBlocks * c * sizeof(float) + 256; }

int nrpn_bias_grad(const void* dy_cl, long rows, int c, int ld, int act_fp16, float* db, void* workspace, size_t workspace_bytes,
                   nrpn_stream_t stream) {
    if (!dy_cl || !db || !workspace || rows < 1 || c < 1 || ld < c) return NRPN_ERR_INVALID;
    if (workspace_bytes < nrpn_bias_grad_workspace_bytes(c)) return NRPN_ERR_WORKSPACE;
    float* partial = reinterpret_cast<float*>(nrpn::align_up((size_t)workspace, 256));
    const int blocks = rows < nrpn::kBgBlocks ? (int)rows : nrpn::kBgBlocks;
    if (c % 8 == 0 && c <= 2048 && ld % 8 == 0 && reinterpret_cast<uintptr_t>(dy_cl) % 16 == 0)
        nrpn::bias_grad_partial_vec_kernel<<<blocks, 256, c * sizeof(float), (cudaStream_t)stream>>>(reinterpret_cast<const __nv_bfloat16*>(dy_cl), rows, c, ld,
                                                                                                  act_fp16 ? 1 : 0, partial);
    else
        nrpn::bias_grad_partial_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const __nv_bfloat16*>(dy_cl), rows, c, ld,
                                                                              act_fp16 ? 1 : 0, partial);
    NRPN_LAUNCH_CHECK();
    nrpn::bias_grad_final_kernel<<<nrpn::ceil_div(c, 8), 256, 0, (cudaStream_t)stream>>>(partial, blocks, c, db);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

int nrpn_relu_backward(void* dy_cl, const void* act_cl, size_t elements, int act_fp16, nrpn_stream_t stream) {
    if (!dy_cl || !act_cl || elements < 8 || elements % 8 != 0) return NRPN_ERR_INVALID;
    if (reinterpret_cast<uintptr_t>(dy_cl) % 16 != 0 || reinterpret_cast<uintptr_t>(act_cl) % 16 != 0) return NRPN_ERR_INVALID;
    const size_t chunks = elements / 8;
    size_t blocks = nrpn::ceil_div(chunks, (size_t)256);
    if (blocks > (size_t)nrpn::num_sms() * 16) blocks = (size_t)nrpn::num_sms() * 16;
    nrpn::relu_backward_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<__nv_bfloat16*>(dy_cl),
                                                                                  reinterpret_cast<const __nv_bfloat16*>(act_cl), chunks,
                                                                                  act_fp16 ? 1 : 0);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

#pragma GCC visibility pop
}  // extern "C"
