// 3-D convolution as an implicit GEMM on Hopper warpgroup MMA (wgmma, sm_90a).
//
// Replaces every nn.Conv3d (+ BatchNorm3d + ReLU + residual / FPN top-down add) of the reference path
// (feature_extractor.py:31-68,145-235; anchor.py:177-213), which runs them as separate cuDNN / ATen kernels on
// fp32 NCDHW tensors.
//
// GEMM view:  D[M = voxels, N = Cout] = sum over (tap, Cin)  A[voxel + tap_offset, Cin] * W[tap][Cout, Cin]
//   - M tile  = a brick of bx*by*bz = 128 output voxels.  The A operand of one (tap, 64-channel) k-block is the
//     same brick shifted by the tap offset: ONE 5-D TMA box load {64 ch, bz, by, bx, 1} from the channels-last
//     activation tensor, out-of-bounds voxels zero-filled by TMA (= the convolution's zero padding).  The box
//     lands in shared memory as 128 rows x 128 bytes in the 128B-swizzled K-major layout wgmma consumes:
//     no im2col buffer, no index arithmetic on the SM.
//   - N tile  = 64 / 128 / 256 output channels; W is pre-packed (tap, Cout, Cin) so a k-block of weights is a
//     3-D TMA box {64, N, 1}.
//   - warps 0-7 = two consumer warpgroups (rows 0-63 / 64-127 of the tile: m64nNk16 wgmma into register accumulators,
//     then the epilogue straight from those registers), warp 8 = TMA producer (one elect.sync lane issues the loads).  smem
//     ring of 2-8 stages (full/empty mbarriers); a stage is released once the MMAs that read it have retired (wait_group 1),
//     so the producer streams the next tile's operands while the consumers run the epilogue.  Persistent CTAs (grid = min(tiles,
//     resident slots)) take tiles from a list that may span up to 4 pyramid levels sharing the same weights (the RPN head on
//     P2..P5 is ONE launch per layer).  Tiles are handed out dynamically: CTA b starts with tile b, then its producer claims the
//     next one from a per-launch counter (g_conv_sched) and passes each index to both consumer warpgroups through a 4-deep
//     shared-memory ring with its own full/empty mbarriers; an index past the last tile ends the loop.  A CTA that starts late
//     (its SM still busy with other streams' kernels) or runs slow thus does fewer tiles instead of setting the layer's end.
//     Every tile runs all its k-blocks in the same order on whichever CTA claims it: results do not depend on the schedule.
//     Prologue (barriers, tensor-map prefetch) runs ahead of griddepcontrol.wait (programmatic dependent launch, every launch).
//   - epilogue (fused): + shift (bias / folded BN), + residual (same shape, or nearest-upsampled coarser level for the FPN
//     top-down path), ReLU / GELU, convert to bf16 / fp16 / fp32.  TMA_EPI variants (16-bit output) stage the tile in shared
//     memory as 128 x 64 sub-tiles and store each with cp.async.bulk.tensor; the short reductions also prefetch a same-shape
//     residual by TMA.
//   - instances (kConvInstances, which also holds the names nrpn_conv3d_variant reports): <256,4,1> <128,6,1> <64,8,1> (long
//     reductions, each with and without TMA_EPI; <64,8,1> also for layers with fewer tiles than SMs), <64,2,3> /
//     <64,2,2,TMA_EPI> (reductions of at most 8 k-blocks); with WS the long ones are <256,2,1> <128,4,1> <64,6,1>.
#include <atomic>
#include <cstdlib>
#include <type_traits>
#include "common.cuh"
#include "wgmma.cuh"
#include "conv_internal.cuh"

namespace nrpn {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr int kUmmaK = 16;
constexpr int kABytes = kBlockM * kBlockK * 2;       // 16 KB
constexpr int kConsumerThreads = 256;                // two warpgroups of 64 accumulator rows each
constexpr int kConvThreads = kConsumerThreads + 32;  // + the TMA producer warp

struct ConvLevelDev {
    int n, xo, yo, zo;
    int bx, by, bz;          // brick (product 128)
    int tx, ty, tz;          // bricks per axis
    int tile_begin;          // first m-tile of this level
    int xr, yr, zr;          // residual extent
    float rsx, rsy, rsz;     // nearest-neighbour scale = in / out
    int ldy, ldr;
    int res_tma;             // TMA-epilogue variant: the residual has the output's extent and arrives through maps.r
    void* y;
    const __nv_bfloat16* res;
};

struct ConvDev {
    int n_levels, n_taps, kc_blocks, n_tiles_n, cout, relu, out_fp32, fp16;
    int total_m_tiles;
    int sched_slot;          // g_conv_sched pair of this launch
    signed char tap[NRPN_CONV_MAX_TAPS][4];
    const float* shift;
    ConvLevelDev lv[NRPN_CONV_MAX_LEVELS];
};

struct ConvMaps {
    CUtensorMap x[NRPN_CONV_MAX_LEVELS];
    CUtensorMap w;
    CUtensorMap y[NRPN_CONV_MAX_LEVELS];      // TMA-epilogue variant only: output tiles are stored with cp.async.bulk.tensor
    CUtensorMap r[NRPN_CONV_MAX_LEVELS];      // ... and same-shape residual tiles are prefetched by the producer warp
};

constexpr int kEpiTileBytes = kBlockM * 64 * 2;      // one 128 x 64 bf16 tile (residual in / output out of the TMA epilogue)
constexpr int kTileRing = 4;                         // tile indices handed from the producer warp to the consumers

// Dynamic tile scheduler: {claim, done} counter pairs, one pair per launch in flight.  A launch takes the next pair round
// robin (g_conv_sched_next, shared by every instance), so launches on concurrent streams use different pairs unless
// kSchedSlots launches apart.  Every pair is zero between launches: the last CTA of a launch to stop claiming resets it
// (conv3d_igemm_kernel).
constexpr int kSchedSlots = 1024;
__device__ unsigned int g_conv_sched[kSchedSlots][2];
static std::atomic<unsigned int> g_conv_sched_next{0};

// Shared-memory tiles of the TMA epilogue (see conv3d_igemm_kernel): residual prefetch ring and output staging buffers.
// The short reductions run 2 CTAs per SM and have room for one staging buffer and a residual ring of 2 (1 with split weights);
// the long reductions run 1 CTA per SM and double-buffer the staging.
__host__ __device__ constexpr int epi_res_slots(int min_blocks, bool tma_epi, bool ws) { return tma_epi && min_blocks > 1 ? (ws ? 1 : 2) : 0; }
__host__ __device__ constexpr int epi_out_slots(int min_blocks, bool tma_epi) { return tma_epi ? (min_blocks > 1 ? 1 : 2) : 0; }

struct TilePos { int l, tix, tiy, tiz, nb; };

__device__ __forceinline__ TilePos tile_pos(const ConvDev& P, int m_tile) {
    TilePos p;
    p.l = 0;
#pragma unroll
    for (int i = 1; i < NRPN_CONV_MAX_LEVELS; ++i) if (i < P.n_levels && m_tile >= P.lv[i].tile_begin) p.l = i;
    const ConvLevelDev& L = P.lv[p.l];
    int t = m_tile - L.tile_begin;
    p.tiz = t % L.tz; t /= L.tz;
    p.tiy = t % L.ty; t /= L.ty;
    p.tix = t % L.tx; p.nb = t / L.tx;
    return p;
}

// Output voxel of accumulator row `row` of a tile, and the residual row that is added to it (nullptr: none).
struct RowPos { bool valid; size_t vox; const __nv_bfloat16* rrow; };

__device__ __forceinline__ RowPos row_pos(const ConvLevelDev& L, const TilePos& p, int row) {
    RowPos r;
    const int lz = __ffs(L.bz) - 1, ly = __ffs(L.by) - 1;             // brick sides are powers of two (choose_brick)
    const int zi = row & (L.bz - 1), yi = (row >> lz) & (L.by - 1), xi = row >> (lz + ly);
    const int gx = p.tix * L.bx + xi, gy = p.tiy * L.by + yi, gz = p.tiz * L.bz + zi;
    r.valid = gx < L.xo && gy < L.yo && gz < L.zo;
    r.vox = (((size_t)p.nb * L.xo + gx) * L.yo + gy) * L.zo + gz;
    r.rrow = nullptr;
    if (L.res != nullptr && r.valid) {
        int rx = gx, ry = gy, rz = gz;
        if (L.xr != L.xo || L.yr != L.yo || L.zr != L.zo) {   // F.interpolate(mode='nearest', size=...)
            rx = min((int)floorf((float)gx * L.rsx), L.xr - 1);
            ry = min((int)floorf((float)gy * L.rsy), L.yr - 1);
            rz = min((int)floorf((float)gz * L.rsz), L.zr - 1);
        }
        r.rrow = L.res + ((((size_t)p.nb * L.xr + rx) * L.yr + ry) * L.zr + rz) * L.ldr;
    }
    return r;
}

__device__ __forceinline__ float activate(float v, int relu) {
    if (relu == 1) return fmaxf(v, 0.0f);
    if (relu == 2) return 0.5f * v * (1.0f + erff(v * 0.70710678118654752f));     // exact (erf) GELU: Swin MLP, feature_extractor.py:635
    return v;
}

// TMA_EPI (16-bit output): the consumers write the tile, 64 channels at a time, into a swizzled 128 x 64 staging buffer and
// one thread stores it with cp.async.bulk.tensor (hardware clips partial bricks and channels past Cout).
//   - short reductions (N = 64 tiles of the HBM-bound 1^3 layers, 2 CTAs / SM, Cout % 64 == 0): the producer warp also
//     prefetches the residual tile of a same-shape skip connection into shared memory (2-deep ring) with the operands, and
//     the epilogue never reads global memory from a register.  One staging buffer.
//   - long reductions (1 CTA / SM): any residual is read from global memory as in the register epilogue.  Two staging
//     buffers, so that the consumers fill one while the previous sub-tile's store reads the other: the tensor pipe idles
//     for the shared-memory writes only, not for scattered 4-byte global stores.
//
// WS (weight split, the <=1e-3 parity mode of the backbone): every weight is the sum of TWO 16-bit numbers, w = hi + lo with
// lo = round16(w - hi), packed as (taps, 2, CoutPad, Cin).  One TMA box {64, BLOCK_N, 2} brings both planes of a k-block; the
// consumers run the k-block's MMAs twice on the SAME activation tile (B = hi, then B = lo) into the same accumulator, so the
// weights enter the fp32 accumulation with ~22 significant bits and only the activations carry 16-bit rounding error.
template <int BLOCK_N, int STAGES, int MIN_BLOCKS, bool TMA_EPI = false, bool WS = false>
__global__ void __launch_bounds__(kConvThreads, MIN_BLOCKS) conv3d_igemm_kernel(const __grid_constant__ ConvMaps maps, const ConvDev P) {
    constexpr int kBPlane = BLOCK_N * kBlockK * 2;
    constexpr int kBBytes = kBPlane * (WS ? 2 : 1);
    constexpr int kStageBytes = kABytes + kBBytes;
    constexpr bool kResRing = TMA_EPI && MIN_BLOCKS > 1;                // the short reductions' residual prefetch
    constexpr int RES_SLOTS = epi_res_slots(MIN_BLOCKS, TMA_EPI, WS);
    constexpr int OUT_SLOTS = epi_out_slots(MIN_BLOCKS, TMA_EPI);
    constexpr int kEpiBytes = (RES_SLOTS + OUT_SLOTS) * kEpiTileBytes;  // residual ring + output staging

    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* smem_res = smem + STAGES * kStageBytes;                 // [RES_SLOTS][128 rows][128 B], 128B-swizzled
    uint8_t* smem_out = smem_res + RES_SLOTS * kEpiTileBytes;        // [OUT_SLOTS][128 rows][128 B], 128B-swizzled
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * kStageBytes + kEpiBytes);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + STAGES;
    uint64_t* rfull_bar = bars + 2 * STAGES;
    uint64_t* rempty_bar = bars + 2 * STAGES + 2;
    uint64_t* tfull_bar = bars + 2 * STAGES + 4;
    uint64_t* tempty_bar = tfull_bar + kTileRing;
    int* tile_ring = reinterpret_cast<int*>(tempty_bar + kTileRing);

    const int warp = threadIdx.x >> 5;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], 2); }   // one arrival per consumer warpgroup
        for (int a = 0; a < 2; ++a) { ptx::mbar_init(&rfull_bar[a], 1); ptx::mbar_init(&rempty_bar[a], 1); }
        for (int s = 0; s < kTileRing; ++s) { ptx::mbar_init(&tfull_bar[s], 1); ptx::mbar_init(&tempty_bar[s], kConsumerThreads); }
        ptx::fence_barrier_init();
        for (int l = 0; l < P.n_levels; ++l) ptx::prefetch_tmap(&maps.x[l]);
        if (TMA_EPI) for (int l = 0; l < P.n_levels; ++l) ptx::prefetch_tmap(&maps.y[l]);
        if (kResRing) for (int l = 0; l < P.n_levels; ++l) ptx::prefetch_tmap(&maps.r[l]);
        ptx::prefetch_tmap(&maps.w);
    }
    ptx::pdl_trigger();                 // the next layer may start its own prologue as our CTAs retire
    __syncthreads();
    ptx::pdl_wait();                    // everything above overlapped the previous layer's tail; its outputs are visible from here

    const int total_tiles = P.total_m_tiles * P.n_tiles_n;     // work items = output tiles
    const int kblocks = P.n_taps * P.kc_blocks;

    if (warp == kConsumerThreads / 32) {
        // ------------------------------------------------------------------ TMA producer (whole warp walks, one elected lane issues)
        const bool leader = ptx::elect_one();
        const int leader_lane = __ffs(__ballot_sync(0xffffffffu, leader)) - 1;
        unsigned int* sched = g_conv_sched[P.sched_slot];
        int stage = 0; uint32_t phase = 0;
        int rslot = 0; uint32_t rphase = 0;
        int tslot = 0; uint32_t tphase = 0;
        for (int tile = blockIdx.x;;) {
            // hand the tile to the consumers; total_tiles (past the last tile) ends their loop
            ptx::mbar_wait(&tempty_bar[tslot], tphase ^ 1u);
            if (leader) { tile_ring[tslot] = tile; ptx::mbar_arrive(&tfull_bar[tslot]); }
            __syncwarp();
            if (++tslot == kTileRing) { tslot = 0; tphase ^= 1u; }
            if (tile >= total_tiles) break;
            const int n_tile = tile % P.n_tiles_n, m_tile = tile / P.n_tiles_n;
            const TilePos tp = tile_pos(P, m_tile);
            const ConvLevelDev& L = P.lv[tp.l];
            const int x0 = tp.tix * L.bx, y0 = tp.tiy * L.by, z0 = tp.tiz * L.bz, n0 = n_tile * BLOCK_N;
            for (int kb = 0; kb < kblocks; ++kb) {
                const int tap = kb / P.kc_blocks, kc = kb - tap * P.kc_blocks;
                const int dx = P.tap[tap][0], dy = P.tap[tap][1], dz = P.tap[tap][2];
                ptx::mbar_wait(&empty_bar[stage], phase ^ 1u);
                if (leader) {
                    uint8_t* sa = smem + stage * kStageBytes;
                    uint8_t* sb = sa + kABytes;
                    ptx::mbar_expect_tx(&full_bar[stage], kStageBytes);
                    ptx::tma_load_5d(sa, &maps.x[tp.l], &full_bar[stage], kc * kBlockK, z0 + dz, y0 + dy, x0 + dx, tp.nb);
                    ptx::tma_load_3d(sb, &maps.w, &full_bar[stage], kc * kBlockK, n0, WS ? 2 * tap : tap);   // WS: box depth 2 = hi, lo
                }
                __syncwarp();
                if (++stage == STAGES) { stage = 0; phase ^= 1u; }
            }
            if (kResRing && L.res_tma) {                          // residual tile of this output tile, two tiles ahead of its use
                ptx::mbar_wait(&rempty_bar[rslot], rphase ^ 1u);
                if (leader) {
                    ptx::mbar_expect_tx(&rfull_bar[rslot], kEpiTileBytes);
                    ptx::tma_load_5d(smem_res + rslot * kEpiTileBytes, &maps.r[tp.l], &rfull_bar[rslot], n0, z0, y0, x0, tp.nb);
                }
                __syncwarp();
                if (++rslot == RES_SLOTS) { rslot = 0; rphase ^= 1u; }
            }
            // Claim the next tile once this one's loads are issued: a CTA that started late, or shares its SM with other
            // work, simply claims fewer tiles.  A launch with one tile per CTA claims nothing.
            int next = total_tiles;
            if (leader && (int)gridDim.x < total_tiles) next = (int)gridDim.x + (int)atomicAdd(&sched[0], 1u);
            tile = __shfl_sync(0xffffffffu, next, leader_lane);
        }
        // The claim that came back past the last tile was this CTA's last: once every CTA has made it, the last one to
        // count itself done zeroes the pair for the next launch that takes it.
        if (leader && (int)gridDim.x < total_tiles) {
            __threadfence();
            if (atomicAdd(&sched[1], 1u) == gridDim.x - 1) { atomicExch(&sched[0], 0u); atomicExch(&sched[1], 0u); }
        }
        return;
    }

    // ---------------------------------------------------------------------- consumers (warpgroups 0 and 1): MMA + epilogue
    const int t = threadIdx.x & 127, wg = threadIdx.x >> 7;
    int stage = 0; uint32_t phase = 0;
    int rslot = 0; uint32_t rphase = 0;
    int tslot = 0; uint32_t tphase = 0;
    uint32_t n_stores = 0;                                  // bulk stores issued so far: staging buffer n_stores % OUT_SLOTS is next
    float acc[BLOCK_N / 2];
    auto next_tile = [&]() {                                // the producer's next tile index (total_tiles: no more)
        ptx::mbar_wait(&tfull_bar[tslot], tphase);
        const int tile = tile_ring[tslot];
        ptx::mbar_arrive(&tempty_bar[tslot]);
        if (++tslot == kTileRing) { tslot = 0; tphase ^= 1u; }
        return tile;
    };
    for (int tile = next_tile(); tile < total_tiles; tile = next_tile()) {
        const int n_tile = tile % P.n_tiles_n, m_tile = tile / P.n_tiles_n;
        const TilePos tp = tile_pos(P, m_tile);
        const ConvLevelDev& L = P.lv[tp.l];
        const int n0 = n_tile * BLOCK_N;

        ptx::reg_fence(acc);
        int prev = 0;
        for (int kb = 0; kb < kblocks; ++kb) {
            ptx::mbar_wait(&full_bar[stage], phase);
            const uint32_t sa = ptx::smem_u32(smem + stage * kStageBytes);
            const uint64_t da = ptx::make_desc_sw128(sa + (uint32_t)(wg * (kABytes / 2)));      // this warpgroup's 64 rows
            const uint64_t db = ptx::make_desc_sw128(sa + kABytes);
            // one branch per k-block on the activation format, so that each path is an unbroken chain of MMAs
            auto issue = [&](auto f16) {
                ptx::wgmma_fence();
#pragma unroll
                for (int h = 0; h < (WS ? 2 : 1); ++h) {
#pragma unroll
                    for (int k = 0; k < kBlockK / kUmmaK; ++k)
                        // advance 16 elements (32 bytes) along K inside the 128-byte swizzle atom: +2 in the >>4 address field
                        ptx::Wgmma<BLOCK_N, decltype(f16)::value>::template ss<0, 0>(
                            acc, da + (uint64_t)(2 * k), db + (uint64_t)(h * (kBPlane >> 4) + 2 * k), (kb | k | h) ? 1u : 0u);
                }
                ptx::wgmma_commit();
            };
            if (P.fp16) issue(std::true_type{}); else issue(std::false_type{});
            ptx::wgmma_wait<1>();                            // the previous k-block's MMAs have retired: its stage is free
            if (kb > 0 && t == 0) ptx::mbar_arrive(&empty_bar[prev]);
            prev = stage;
            if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
        ptx::wgmma_wait<0>();
        ptx::reg_fence(acc);
        if (t == 0) ptx::mbar_arrive(&empty_bar[prev]);

        if constexpr (TMA_EPI) {
            // ---- shared-memory epilogue: output through swizzled 128 x 64 staging sub-tiles + TMA stores
            const bool res_smem = kResRing && L.res_tma != 0;      // residual from the TMA-fed ring, else from global memory
            if (res_smem) ptx::mbar_wait(&rfull_bar[rslot], rphase);
            const uint8_t* rsm = smem_res + rslot * kEpiTileBytes;
            const __nv_bfloat16* rrow[2] = {nullptr, nullptr};            // residual rows read from global memory
            if (!res_smem && L.res != nullptr) {
#pragma unroll
                for (int h = 0; h < 2; ++h) rrow[h] = row_pos(L, tp, wg * 64 + ptx::frag_row(t, h)).rrow;
            }
#pragma unroll
            for (int c = 0; c < BLOCK_N / 64; ++c) {
                const int c0 = n0 + 64 * c;
                if (c0 >= P.cout) continue;                       // the same for every thread: nothing of this sub-tile is stored
                uint8_t* so = smem_out + (OUT_SLOTS == 1 ? 0 : n_stores % OUT_SLOTS) * kEpiTileBytes;
                if (OUT_SLOTS == 1) {
                    // the staging tile is free once the previous tile's bulk store has finished READING it
                    if (threadIdx.x == 0) ptx::bulk_wait_read0();
                    ptx::named_barrier(1, kConsumerThreads);
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = wg * 64 + ptx::frag_row(t, h);
                    // 128B swizzle: 16-byte chunk j of the row lands at chunk j ^ (row & 7)
                    const uint32_t rbase = (uint32_t)(row * 128 + ((row & 7) << 4) + (ptx::frag_col(t, 0) & 7) * 2);
#pragma unroll
                    for (int j = 0; j < 8; ++j) {                 // 16-byte chunk j (8 channels) of the 128-byte row
                        const int ch = c0 + ptx::frag_col(t, j);
                        const uint32_t off = rbase ^ (uint32_t)(j << 4);
                        float v0 = 0.0f, v1 = 0.0f;
                        if (ch < P.cout) {                        // Cout % 8 == 0: the pair is wholly in or out
                            const float2 s = __ldg(reinterpret_cast<const float2*>(P.shift + ch));
                            v0 = acc[4 * (8 * c + j) + 2 * h] + s.x; v1 = acc[4 * (8 * c + j) + 2 * h + 1] + s.y;
                            if (res_smem || rrow[h] != nullptr) {
                                const uint32_t rv = res_smem ? *reinterpret_cast<const uint32_t*>(rsm + off)
                                                             : __ldg(reinterpret_cast<const unsigned int*>(rrow[h] + ch));
                                const float2 f = unpack_act2(rv, P.fp16);
                                v0 += f.x; v1 += f.y;
                            }
                        }
                        *reinterpret_cast<uint32_t*>(so + off) = pack_act2(activate(v0, P.relu), activate(v1, P.relu), P.fp16);
                    }
                }
                ptx::fence_proxy_async();                        // generic-proxy smem writes -> visible to the TMA engine
                // double buffering: once the previous store has read its buffer, the barrier below frees it for the next sub-tile
                if (OUT_SLOTS > 1 && threadIdx.x == 0) ptx::bulk_wait_read0();
                ptx::named_barrier(1, kConsumerThreads);
                if (threadIdx.x == 0) {
                    // the tile position is recomputed here rather than kept live through the epilogue (register pressure)
                    const TilePos q = tile_pos(P, tile / P.n_tiles_n);
                    const ConvLevelDev& Lq = P.lv[q.l];
                    ptx::tma_store_5d(&maps.y[q.l], so, c0, q.tiz * Lq.bz, q.tiy * Lq.by, q.tix * Lq.bx, q.nb);
                    ptx::bulk_commit();
                }
                ++n_stores;
            }
            if (res_smem) {
                if (threadIdx.x == 0) ptx::mbar_arrive(&rempty_bar[rslot]);   // every consumer has passed the last barrier
                if (++rslot == RES_SLOTS) { rslot = 0; rphase ^= 1u; }
            }
            continue;
        }
        // ---- register epilogue: each thread owns 2 channels of every 8-channel group in two rows of the tile
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const RowPos rp = row_pos(L, tp, wg * 64 + ptx::frag_row(t, h));
            if (!rp.valid) continue;
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j) {
                const int ch = n0 + ptx::frag_col(t, j);
                if (ch >= P.cout) continue;                  // Cout % 8 == 0: the pair is wholly in or out
                const float2 s = __ldg(reinterpret_cast<const float2*>(P.shift + ch));
                float v0 = acc[4 * j + 2 * h] + s.x, v1 = acc[4 * j + 2 * h + 1] + s.y;
                if (rp.rrow != nullptr) {
                    const float2 f = unpack_act2(__ldg(reinterpret_cast<const unsigned int*>(rp.rrow + ch)), P.fp16);
                    v0 += f.x; v1 += f.y;
                }
                v0 = activate(v0, P.relu); v1 = activate(v1, P.relu);
                if (P.out_fp32) *reinterpret_cast<float2*>(reinterpret_cast<float*>(L.y) + rp.vox * L.ldy + ch) = make_float2(v0, v1);
                else *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(L.y) + rp.vox * L.ldy + ch) = pack_act2(v0, v1, P.fp16);
            }
        }
    }
    if (TMA_EPI && threadIdx.x == 0) ptx::bulk_wait_all();          // the staging tile must outlive its last bulk store
}

// ------------------------------------------------------------------------------------------------ host
template <int BLOCK_N, int STAGES, int MIN_BLOCKS, bool TMA_EPI = false, bool WS = false>
static int launch_conv(const ConvMaps& maps, const ConvDev& P, cudaStream_t st) {
    constexpr int smem = STAGES * (kABytes + BLOCK_N * kBlockK * 2 * (WS ? 2 : 1)) +
                         (epi_res_slots(MIN_BLOCKS, TMA_EPI, WS) + epi_out_slots(MIN_BLOCKS, TMA_EPI)) * kEpiTileBytes + 1024 + 256;
    static_assert((smem + 1024) * MIN_BLOCKS <= 228 * 1024, "shared memory budget");
    static_assert((2 * STAGES + 4 + 2 * kTileRing) * 8 + kTileRing * 4 <= 256, "barriers and tile ring");
    static bool attr_set = false;
    if (!attr_set) {
        NRPN_CUDA_TRY(cudaFuncSetAttribute(conv3d_igemm_kernel<BLOCK_N, STAGES, MIN_BLOCKS, TMA_EPI, WS>,
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        attr_set = true;
    }
    ConvDev Q = P;
    Q.sched_slot = (int)(g_conv_sched_next.fetch_add(1u, std::memory_order_relaxed) % kSchedSlots);
    const int total_tiles = P.total_m_tiles * P.n_tiles_n;
    const int slots = num_sms() * MIN_BLOCKS;
    const int grid = total_tiles < slots ? total_tiles : slots;
    // No CTA owns a fixed tile set, so every launch may start its prologue on SMs that the previous layer's CTAs leave.
    NRPN_CUDA_TRY(launch_pdl(conv3d_igemm_kernel<BLOCK_N, STAGES, MIN_BLOCKS, TMA_EPI, WS>, dim3(grid), dim3(kConvThreads), smem, st, true, maps, Q));
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

// Every instance nrpn_conv3d_fprop launches, under the name nrpn_conv3d_variant reports for it.  Index:
// 8 wsplit + 2 (0 for a short reduction, else 1 + log2(BLOCK_N / 64)) + TMA epilogue.
struct ConvInstance { const char* name; int (*launch)(const ConvMaps&, const ConvDev&, cudaStream_t); };
static const ConvInstance kConvInstances[16] = {
    {"igemm<64,2,3>", launch_conv<64, 2, 3>},
    {"igemm<64,2,2,tma-epilogue>", launch_conv<64, 2, 2, true>},
    {"igemm<64,8,1>", launch_conv<64, 8, 1>},
    {"igemm<64,8,1,tma-epilogue>", launch_conv<64, 8, 1, true>},
    {"igemm<128,6,1>", launch_conv<128, 6, 1>},
    {"igemm<128,6,1,tma-epilogue>", launch_conv<128, 6, 1, true>},
    {"igemm<256,4,1>", launch_conv<256, 4, 1>},
    {"igemm<256,4,1,tma-epilogue>", launch_conv<256, 4, 1, true>},
    {"igemm<64,2,3,wsplit>", launch_conv<64, 2, 3, false, true>},
    {"igemm<64,2,2,tma-epilogue,wsplit>", launch_conv<64, 2, 2, true, true>},
    {"igemm<64,6,1,wsplit>", launch_conv<64, 6, 1, false, true>},
    {"igemm<64,6,1,tma-epilogue,wsplit>", launch_conv<64, 6, 1, true, true>},
    {"igemm<128,4,1,wsplit>", launch_conv<128, 4, 1, false, true>},
    {"igemm<128,4,1,tma-epilogue,wsplit>", launch_conv<128, 4, 1, true, true>},
    {"igemm<256,2,1,wsplit>", launch_conv<256, 2, 1, false, true>},
    {"igemm<256,2,1,tma-epilogue,wsplit>", launch_conv<256, 2, 1, true, true>},
};

static void choose_brick(int xo, int yo, int zo, int& bx, int& by, int& bz) {
    long best = -1;
    for (int ez = 0; ez <= 7; ++ez) for (int ey = 0; ey + ez <= 7; ++ey) {
        const int ex = 7 - ez - ey;
        const int cz = 1 << ez, cy = 1 << ey, cx = 1 << ex;
        if (cz > 256 || cy > 256 || cx > 256) continue;
        const long vol = (long)ceil_div(xo, cx) * cx * ceil_div(yo, cy) * cy * ceil_div(zo, cz) * cz;
        // prefer less padding, then compact bricks (smallest halo => best L2 reuse across the filter taps)
        const long score = vol * 4096 + (long)(cx + 2) * (cy + 2) * (cz + 2);
        if (best < 0 || score < best) { best = score; bx = cx; by = cy; bz = cz; }
    }
}

struct ConvPlan {
    const ConvInstance* inst;   // nullptr: the halo-slab kernel (conv3d_slab.cu)
    int block_n, cout_pad;      // N tile of the instance; Cout padded to nrpn_conv3d_block_n(cout)
    bool tma_epi;               // shared-memory (TMA-store) epilogue
    ConvDev P;
};

// Validates a descriptor and decides what nrpn_conv3d_fprop launches for it.  Host logic only: pointers are checked and
// compared, never dereferenced.  The A/B switches NRPN_CONV_NARROW, NRPN_CONV_TMA_EPI (and NRPN_CONV_SLAB) are read on every call.
static int conv_plan(const nrpn_conv_desc* d, ConvPlan& p) {
    if (!d || !d->w || !d->shift) return NRPN_ERR_INVALID;
    if (d->cin < 64 || d->cin % 64 != 0 || d->cout < 8 || d->cout % 8 != 0) return NRPN_ERR_UNSUPPORTED;
    if (d->n_taps < 1 || d->n_taps > NRPN_CONV_MAX_TAPS || d->n_levels < 1 || d->n_levels > NRPN_CONV_MAX_LEVELS)
        return NRPN_ERR_INVALID;
    if (d->stride != 1 && d->stride != 2) return NRPN_ERR_UNSUPPORTED;
    if (d->stride == 2) {       // strided access is expressed through a sub-sampled tensor map: taps must not move
        for (int t = 0; t < d->n_taps; ++t)
            if (d->tap_off[t][0] || d->tap_off[t][1] || d->tap_off[t][2]) return NRPN_ERR_UNSUPPORTED;
    }
    if (!conv_pairs_aligned(d)) return NRPN_ERR_INVALID;
    for (int l = 0; l < d->n_levels; ++l) {
        const nrpn_conv_level& S = d->level[l];
        if (!S.x || !S.y || S.n < 1 || S.xi < 1 || S.yi < 1 || S.zi < 1 || S.xo < 1 || S.yo < 1 || S.zo < 1) return NRPN_ERR_INVALID;
        if (S.ldy < d->cout || S.ldy % 8 != 0) return NRPN_ERR_INVALID;
        if (S.res && (S.ldr < d->cout || S.ldr % 8 != 0 || S.xr < 1 || S.yr < 1 || S.zr < 1)) return NRPN_ERR_INVALID;
        if (d->stride == 2 && (S.xo != (S.xi + 1) / 2 || S.yo != (S.yi + 1) / 2 || S.zo != (S.zi + 1) / 2)) return NRPN_ERR_INVALID;
    }
    p.inst = nullptr;
    if (!d->wsplit && conv3d_slab_eligible(d)) return NRPN_OK;

    ConvDev& P = p.P;
    memset(&P, 0, sizeof(P));
    P.n_levels = d->n_levels; P.n_taps = d->n_taps; P.kc_blocks = d->cin / kBlockK;
    P.cout = d->cout; P.relu = d->relu; P.out_fp32 = d->out_fp32; P.shift = d->shift; P.fp16 = d->act_fp16 ? 1 : 0;
    for (int t = 0; t < d->n_taps; ++t) { P.tap[t][0] = d->tap_off[t][0]; P.tap[t][1] = d->tap_off[t][1]; P.tap[t][2] = d->tap_off[t][2]; P.tap[t][3] = 0; }
    int tiles = 0;
    for (int l = 0; l < d->n_levels; ++l) {
        const nrpn_conv_level& S = d->level[l];
        ConvLevelDev& L = P.lv[l];
        L.n = S.n; L.xo = S.xo; L.yo = S.yo; L.zo = S.zo;
        choose_brick(S.xo, S.yo, S.zo, L.bx, L.by, L.bz);
        L.tx = ceil_div(S.xo, L.bx); L.ty = ceil_div(S.yo, L.by); L.tz = ceil_div(S.zo, L.bz);
        L.tile_begin = tiles;
        tiles += S.n * L.tx * L.ty * L.tz;
        L.xr = S.res ? S.xr : S.xo; L.yr = S.res ? S.yr : S.yo; L.zr = S.res ? S.zr : S.zo;
        L.rsx = (float)L.xr / (float)S.xo; L.rsy = (float)L.yr / (float)S.yo; L.rsz = (float)L.zr / (float)S.zo;
        L.ldy = S.ldy; L.ldr = S.ldr; L.y = S.y; L.res = reinterpret_cast<const __nv_bfloat16*>(S.res);
    }
    P.total_m_tiles = tiles;

    // Weights are padded to nrpn_conv3d_block_n(cout) (a multiple of 64). Long reductions (3^3 taps) use the widest N tile
    // that fits, one CTA per SM, deep smem ring: tensor-pipe bound.  Short reductions (1^3 convs: at most 8 k-blocks) are
    // HBM / epilogue-latency bound: they run N = 64 tiles with 3 CTAs per SM so that 3x more loads/stores are in flight.
    const int pad_n = nrpn_conv3d_block_n(d->cout);
    p.cout_pad = ceil_div(d->cout, pad_n) * pad_n;
    const bool short_k = d->n_taps * P.kc_blocks <= 8;
    p.block_n = short_k ? 64 : pad_n;
    // Late ResNet stages (5x8x8 .. 10x16x16 voxels, K up to 13 824): a handful of 128 x 256 tiles leaves most SMs idle while each
    // tile runs a long reduction.  When even 64-wide tiles fit in one wave, they are used instead: 4x the CTAs (same reduction
    // order per output element, bit-identical results).
    if (!short_k && p.block_n > 64 && tiles * (p.cout_pad / 64) <= num_sms()) {
        const char* e = getenv("NRPN_CONV_NARROW");
        if (!(e && e[0] == '0')) p.block_n = 64;
    }
    P.n_tiles_n = p.cout_pad / p.block_n;
    // shared-memory (TMA) epilogue: 16-bit output; the short reductions also need whole 64-channel output tiles
    { const char* e = getenv("NRPN_CONV_TMA_EPI"); p.tma_epi = !(e && e[0] == '0'); }       // A/B switch for tests and profiling
    p.tma_epi = p.tma_epi && !d->out_fp32 && (!short_k || d->cout % 64 == 0);
    for (int l = 0; l < d->n_levels; ++l) {
        const nrpn_conv_level& S = d->level[l];
        const ConvLevelDev& L = P.lv[l];
        if (reinterpret_cast<uintptr_t>(S.y) % 16 != 0 || (S.res && reinterpret_cast<uintptr_t>(S.res) % 16 != 0)) p.tma_epi = false;
        // a nearest-upsampled residual (FPN top-down) is gathered per row from registers: the pipelined register epilogue
        // with 3 CTAs per SM is faster for it (measured: lat3+up 0.207 ms vs 0.275 ms)
        if (L.xr != L.xo || L.yr != L.yo || L.zr != L.zo) p.tma_epi = false;
    }
    // once tma_epi holds, every residual has the output's extent: the short reductions prefetch it through maps.r
    for (int l = 0; l < d->n_levels; ++l) P.lv[l].res_tma = (p.tma_epi && short_k && d->level[l].res) ? 1 : 0;
    const int tile_kind = short_k ? 0 : (p.block_n == 64 ? 1 : (p.block_n == 128 ? 2 : 3));
    p.inst = &kConvInstances[8 * (d->wsplit ? 1 : 0) + 2 * tile_kind + (p.tma_epi ? 1 : 0)];
    return NRPN_OK;
}

}  // namespace nrpn

using namespace nrpn;

extern "C" {
#pragma GCC visibility push(default)

int nrpn_conv3d_block_n(int cout) { return cout <= 64 ? 64 : (cout <= 128 ? 128 : 256); }

const char* nrpn_conv3d_variant(const nrpn_conv_desc* d) {
    ConvPlan p;
    const int rc = conv_plan(d, p);
    if (rc == NRPN_ERR_UNSUPPORTED) return "unsupported";
    if (rc != NRPN_OK) return "invalid";
    return p.inst ? p.inst->name : "slab<4x16x8,N64>";
}

int nrpn_conv3d_fprop(const nrpn_conv_desc* d, nrpn_stream_t stream) {
    ConvPlan p;
    { const int rc = conv_plan(d, p); if (rc) return rc; }
    cudaStream_t st = (cudaStream_t)stream;
    if (!p.inst) return conv3d_slab_launch(d, st);

    ConvMaps maps;
    const int s = d->stride;
    for (int l = 0; l < d->n_levels; ++l) {
        const nrpn_conv_level& S = d->level[l];
        const ConvLevelDev& L = p.P.lv[l];
        if (p.tma_epi) {
            // output / residual tensors (C, Z, Y, X, N) with the row pitch ldy / ldr; one box = one 64-channel brick tile
            cuuint32_t ebox[5] = {64, (cuuint32_t)L.bz, (cuuint32_t)L.by, (cuuint32_t)L.bx, 1};
            cuuint64_t ydim[5] = {(cuuint64_t)d->cout, (cuuint64_t)S.zo, (cuuint64_t)S.yo, (cuuint64_t)S.xo, (cuuint64_t)S.n};
            cuuint64_t ystr[4] = {(cuuint64_t)S.ldy * 2, (cuuint64_t)S.zo * S.ldy * 2, (cuuint64_t)S.yo * S.zo * S.ldy * 2,
                                  (cuuint64_t)S.xo * S.yo * S.zo * S.ldy * 2};
            { const int rc = encode_tmap(&maps.y[l], S.y, ydim, ystr, ebox); if (rc) return rc; }
            if (L.res_tma) {
                cuuint64_t rstr[4] = {(cuuint64_t)S.ldr * 2, (cuuint64_t)S.zo * S.ldr * 2, (cuuint64_t)S.yo * S.zo * S.ldr * 2,
                                      (cuuint64_t)S.xo * S.yo * S.zo * S.ldr * 2};
                const int rc = encode_tmap(&maps.r[l], S.res, ydim, rstr, ebox);
                if (rc) return rc;
            } else maps.r[l] = maps.y[l];
        }

        // activation tensor map: (C, Z, Y, X, N), optionally sub-sampled by `stride` on the three spatial axes
        const cuuint64_t cin = (cuuint64_t)d->cin;
        cuuint64_t gdim[5] = {cin, (cuuint64_t)ceil_div(S.zi, s), (cuuint64_t)ceil_div(S.yi, s), (cuuint64_t)ceil_div(S.xi, s), (cuuint64_t)S.n};
        cuuint64_t gstr[4] = {cin * 2 * s, (cuuint64_t)S.zi * cin * 2 * s, (cuuint64_t)S.yi * S.zi * cin * 2 * s,
                              (cuuint64_t)S.xi * S.yi * S.zi * cin * 2};
        cuuint32_t box[5] = {(cuuint32_t)kBlockK, (cuuint32_t)L.bz, (cuuint32_t)L.by, (cuuint32_t)L.bx, 1};
        { const int rc = encode_tmap(&maps.x[l], S.x, gdim, gstr, box); if (rc) return rc; }
    }
    for (int l = d->n_levels; l < NRPN_CONV_MAX_LEVELS; ++l) { maps.x[l] = maps.x[0]; maps.y[l] = maps.y[0]; maps.r[l] = maps.r[0]; }
    if (!p.tma_epi) for (int l = 0; l < NRPN_CONV_MAX_LEVELS; ++l) { maps.y[l] = maps.x[0]; maps.r[l] = maps.x[0]; }
    {
        // wsplit: (taps, 2, CoutPad, cin) -- the hi and lo planes of a tap are consecutive slices, one box of depth 2 fetches both
        const int planes = d->wsplit ? 2 : 1;
        cuuint64_t gdim[3] = {(cuuint64_t)d->cin, (cuuint64_t)p.cout_pad, (cuuint64_t)d->n_taps * planes};
        cuuint64_t gstr[2] = {(cuuint64_t)d->cin * 2, (cuuint64_t)p.cout_pad * d->cin * 2};
        cuuint32_t box[3] = {(cuuint32_t)kBlockK, (cuuint32_t)p.block_n, (cuuint32_t)planes};
        const int rc = encode_tmap(&maps.w, d->w, gdim, gstr, box);
        if (rc) return rc;
    }
    return p.inst->launch(maps, p.P, st);
}

#pragma GCC visibility pop
}  // extern "C"
