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
//     so the producer streams the next tile's operands while the consumers run the epilogue.  Persistent CTAs walk a static
//     tile list that may span up to 4 pyramid levels sharing the same weights (the RPN head on P2..P5 is ONE launch per
//     layer).  Prologue (barriers, tensor-map prefetch) runs ahead of griddepcontrol.wait (programmatic dependent launch).
//   - epilogue (fused): + shift (bias / folded BN), + residual (same shape, or nearest-upsampled coarser level for the FPN
//     top-down path), ReLU / GELU, convert to bf16 / fp16 / fp32; or -- TMA_EPI variant of the 1^3 layers -- residual tiles
//     prefetched by TMA into shared memory and output tiles stored with cp.async.bulk.tensor.
//   - variants: <256,4,1> <128,6,1> <64,8,1> (long reductions; <64,8,1> also for layers with fewer tiles than SMs),
//     <64,2,3> / <64,2,2,TMA_EPI> (reductions of at most 8 k-blocks), optional split-K (NRPN_SPLITK=1, off by default).
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
    int splits, cout_pad;      // split-K: `splits` CTAs share one output tile and reduce through `ws`
    float* ws;                 // fp32 (tiles, splits, 128, BLOCK_N) partial tiles, rewritten by every launch
    unsigned* counters;        // one arrival counter per output tile, zero between launches
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
    const int zi = row % L.bz, yi = (row / L.bz) % L.by, xi = row / (L.bz * L.by);
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

// TMA_EPI (N = 64 tiles of the HBM-bound 1^3 layers, bf16 output, Cout % 64 == 0): the epilogue never touches global memory
// from a register.  The producer warp prefetches the residual tile of a same-shape skip connection into shared memory
// (2-deep ring) together with the operands; the consumers add it from shared memory, write the 16-bit tile into a
// swizzled staging buffer and one thread stores it with cp.async.bulk.tensor (hardware clips partial bricks).
//
// WS (weight split, the <=1e-3 parity mode of the backbone): every weight is the sum of TWO 16-bit numbers, w = hi + lo with
// lo = round16(w - hi), packed as (taps, 2, CoutPad, Cin).  One TMA box {64, BLOCK_N, 2} brings both planes of a k-block; the
// consumers run the k-block's MMAs twice on the SAME activation tile (B = hi, then B = lo) into the same accumulator, so the
// weights enter the fp32 accumulation with ~22 significant bits and only the activations carry 16-bit rounding error.
template <int BLOCK_N, int STAGES, int MIN_BLOCKS, bool TMA_EPI = false, bool WS = false>
__global__ void __launch_bounds__(kConvThreads, MIN_BLOCKS) conv3d_igemm_kernel(const __grid_constant__ ConvMaps maps, const ConvDev P) {
    static_assert(!TMA_EPI || BLOCK_N == 64, "the TMA epilogue stages 128 x 64 tiles");
    constexpr int kBPlane = BLOCK_N * kBlockK * 2;
    constexpr int kBBytes = kBPlane * (WS ? 2 : 1);
    constexpr int kStageBytes = kABytes + kBBytes;
    constexpr int RES_SLOTS = (TMA_EPI && WS) ? 1 : 2;              // residual prefetch depth (shared-memory budget of 2 CTAs / SM)
    constexpr int kEpiBytes = TMA_EPI ? (RES_SLOTS + 1) * kEpiTileBytes : 0;      // residual ring + output staging (1)

    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* smem_res = smem + STAGES * kStageBytes;                 // [2][128 rows][128 B], 128B-swizzled (TMA_EPI)
    uint8_t* smem_out = smem_res + RES_SLOTS * kEpiTileBytes;        // [128 rows][128 B], 128B-swizzled (TMA_EPI)
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * kStageBytes + kEpiBytes);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + STAGES;
    uint64_t* rfull_bar = bars + 2 * STAGES;
    uint64_t* rempty_bar = bars + 2 * STAGES + 2;
    uint32_t* ticket_slot = reinterpret_cast<uint32_t*>(bars + 2 * STAGES + 4);

    const int warp = threadIdx.x >> 5;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], 2); }   // one arrival per consumer warpgroup
        for (int a = 0; a < 2; ++a) { ptx::mbar_init(&rfull_bar[a], 1); ptx::mbar_init(&rempty_bar[a], 1); }
        ptx::fence_barrier_init();
        for (int l = 0; l < P.n_levels; ++l) ptx::prefetch_tmap(&maps.x[l]);
        if (TMA_EPI) for (int l = 0; l < P.n_levels; ++l) { ptx::prefetch_tmap(&maps.y[l]); ptx::prefetch_tmap(&maps.r[l]); }
        ptx::prefetch_tmap(&maps.w);
    }
    ptx::pdl_trigger();                 // the next layer may start its own prologue as our CTAs retire
    __syncthreads();
    ptx::pdl_wait();                    // everything above overlapped the previous layer's tail; its outputs are visible from here

    const int total_tiles = P.total_m_tiles * P.n_tiles_n * P.splits;     // work items = (output tile, k-split)
    const int kblocks = P.n_taps * P.kc_blocks;

    if (warp == kConsumerThreads / 32) {
        // ------------------------------------------------------------------ TMA producer (whole warp walks, one elected lane issues)
        const bool leader = ptx::elect_one();
        int stage = 0; uint32_t phase = 0;
        int rslot = 0; uint32_t rphase = 0;
        for (int item = blockIdx.x; item < total_tiles; item += gridDim.x) {
            const int split = item % P.splits, tile = item / P.splits;
            const int kb0 = (kblocks * split) / P.splits, kb1 = (kblocks * (split + 1)) / P.splits;
            const int n_tile = tile % P.n_tiles_n, m_tile = tile / P.n_tiles_n;
            const TilePos tp = tile_pos(P, m_tile);
            const ConvLevelDev& L = P.lv[tp.l];
            const int x0 = tp.tix * L.bx, y0 = tp.tiy * L.by, z0 = tp.tiz * L.bz, n0 = n_tile * BLOCK_N;
            for (int kb = kb0; kb < kb1; ++kb) {
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
            if (TMA_EPI && L.res_tma) {                          // residual tile of this output tile, two tiles ahead of its use
                ptx::mbar_wait(&rempty_bar[rslot], rphase ^ 1u);
                if (leader) {
                    ptx::mbar_expect_tx(&rfull_bar[rslot], kEpiTileBytes);
                    ptx::tma_load_5d(smem_res + rslot * kEpiTileBytes, &maps.r[tp.l], &rfull_bar[rslot], n0, z0, y0, x0, tp.nb);
                }
                __syncwarp();
                if (++rslot == RES_SLOTS) { rslot = 0; rphase ^= 1u; }
            }
        }
        return;
    }

    // ---------------------------------------------------------------------- consumers (warpgroups 0 and 1): MMA + epilogue
    const int t = threadIdx.x & 127, wg = threadIdx.x >> 7;
    int stage = 0; uint32_t phase = 0;
    int rslot = 0; uint32_t rphase = 0;
    float acc[BLOCK_N / 2];
    for (int item = blockIdx.x; item < total_tiles; item += gridDim.x) {
        const int split = item % P.splits, tile = item / P.splits;
        const int nkb = (kblocks * (split + 1)) / P.splits - (kblocks * split) / P.splits;
        const int n_tile = tile % P.n_tiles_n, m_tile = tile / P.n_tiles_n;
        const TilePos tp = tile_pos(P, m_tile);
        const ConvLevelDev& L = P.lv[tp.l];
        const int n0 = n_tile * BLOCK_N;

        ptx::reg_fence(acc);
        int prev = 0;
        for (int kb = 0; kb < nkb; ++kb) {
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
        if (nkb > 0 && t == 0) ptx::mbar_arrive(&empty_bar[prev]);

        if (P.splits > 1) {
            // ---- split-K (deterministic): every CTA stores its partial tile into its own fp32 slab of the workspace with
            // plain stores; the last CTA to arrive sums the slabs in split order and runs the normal epilogue.
            float* slab0 = P.ws + ((size_t)tile * P.splits) * (kBlockM * BLOCK_N);          // slabs of this output tile
            float* wslab = slab0 + (size_t)split * (kBlockM * BLOCK_N);
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    __stcg(reinterpret_cast<float2*>(wslab + (size_t)(wg * 64 + ptx::frag_row(t, h)) * BLOCK_N + ptx::frag_col(t, j)),
                           make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]));
            __threadfence();
            ptx::named_barrier(1, kConsumerThreads);
            if (threadIdx.x == 0) *ticket_slot = atomicAdd(P.counters + tile, 1u);
            ptx::named_barrier(1, kConsumerThreads);
            const bool last = (*ticket_slot == (uint32_t)(P.splits - 1));
            if (last && threadIdx.x < kBlockM) {
                __threadfence();
                const int row = threadIdx.x;                 // one accumulator row per thread
                const RowPos rp = row_pos(L, tp, row);
                if (rp.valid) {
                    const float* rrow0 = slab0 + (size_t)row * BLOCK_N;
                    for (int ch = n0; ch < n0 + BLOCK_N && ch < P.cout; ch += 8) {
                        float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0;
                        for (int sp = 0; sp < P.splits; ++sp) {                                  // fixed order => reproducible
                            const float* wp = rrow0 + (size_t)sp * (kBlockM * BLOCK_N) + (ch - n0);
                            const float4 b0 = __ldcg(reinterpret_cast<const float4*>(wp));
                            const float4 b1 = __ldcg(reinterpret_cast<const float4*>(wp + 4));
                            a0.x += b0.x; a0.y += b0.y; a0.z += b0.z; a0.w += b0.w;
                            a1.x += b1.x; a1.y += b1.y; a1.z += b1.z; a1.w += b1.w;
                        }
                        const float4 s0 = __ldg(reinterpret_cast<const float4*>(P.shift + ch));
                        const float4 s1 = __ldg(reinterpret_cast<const float4*>(P.shift + ch + 4));
                        float v[8] = {a0.x + s0.x, a0.y + s0.y, a0.z + s0.z, a0.w + s0.w, a1.x + s1.x, a1.y + s1.y, a1.z + s1.z, a1.w + s1.w};
                        if (rp.rrow != nullptr) {
                            const uint4 rv4 = __ldg(reinterpret_cast<const uint4*>(rp.rrow + ch));
                            const uint32_t* rb = reinterpret_cast<const uint32_t*>(&rv4);
#pragma unroll
                            for (int i = 0; i < 4; ++i) { const float2 f = unpack_act2(rb[i], P.fp16); v[2 * i] += f.x; v[2 * i + 1] += f.y; }
                        }
#pragma unroll
                        for (int i = 0; i < 8; ++i) v[i] = activate(v[i], P.relu);
                        if (P.out_fp32) {
                            float* o = reinterpret_cast<float*>(L.y) + rp.vox * L.ldy + ch;
                            *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
                            *reinterpret_cast<float4*>(o + 4) = make_float4(v[4], v[5], v[6], v[7]);
                        } else {
                            __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(L.y) + rp.vox * L.ldy + ch;
                            *reinterpret_cast<uint4*>(o) = make_uint4(pack_act2(v[0], v[1], P.fp16), pack_act2(v[2], v[3], P.fp16),
                                                                      pack_act2(v[4], v[5], P.fp16), pack_act2(v[6], v[7], P.fp16));
                        }
                    }
                }
                if (row == 0) P.counters[tile] = 0u;
            }
            ptx::named_barrier(1, kConsumerThreads);         // ticket_slot is reused by the next work item
            continue;
        }
        if constexpr (TMA_EPI) {
            // ---- shared-memory epilogue: residual from the TMA-fed ring, output through a swizzled staging tile + TMA store
            const bool res_smem = L.res_tma != 0;
            if (res_smem) ptx::mbar_wait(&rfull_bar[rslot], rphase);
            // the staging tile is free once the previous tile's bulk store has finished READING it
            if (threadIdx.x == 0) ptx::bulk_wait_read0();
            ptx::named_barrier(1, kConsumerThreads);
            const uint8_t* rsm = smem_res + rslot * kEpiTileBytes;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = wg * 64 + ptx::frag_row(t, h);
                const RowPos rp = res_smem ? RowPos{true, 0, nullptr} : row_pos(L, tp, row);
                const int sw = row & 7;
#pragma unroll
                for (int j = 0; j < 8; ++j) {                 // 16-byte chunk j (8 channels) of the 128-byte row
                    const int col = ptx::frag_col(t, j), ch = n0 + col;
                    const uint32_t off = (uint32_t)(row * 128 + ((j ^ sw) << 4) + (col & 7) * 2);
                    const float2 s = __ldg(reinterpret_cast<const float2*>(P.shift + ch));
                    float v0 = acc[4 * j + 2 * h] + s.x, v1 = acc[4 * j + 2 * h + 1] + s.y;
                    if (res_smem || rp.rrow != nullptr) {
                        const uint32_t rv = res_smem ? *reinterpret_cast<const uint32_t*>(rsm + off)
                                                     : __ldg(reinterpret_cast<const unsigned int*>(rp.rrow + ch));
                        const float2 f = unpack_act2(rv, P.fp16);
                        v0 += f.x; v1 += f.y;
                    }
                    *reinterpret_cast<uint32_t*>(smem_out + off) = pack_act2(activate(v0, P.relu), activate(v1, P.relu), P.fp16);
                }
            }
            ptx::fence_proxy_async();                            // generic-proxy smem writes -> visible to the TMA engine
            ptx::named_barrier(1, kConsumerThreads);
            if (threadIdx.x == 0) {
                if (res_smem) ptx::mbar_arrive(&rempty_bar[rslot]);
                ptx::tma_store_5d(&maps.y[tp.l], smem_out, n0, tp.tiz * L.bz, tp.tiy * L.by, tp.tix * L.bx, tp.nb);
                ptx::bulk_commit();
            }
            if (res_smem && ++rslot == RES_SLOTS) { rslot = 0; rphase ^= 1u; }
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
static int launch_conv(const ConvMaps& maps, const ConvDev& P, int total_tiles, cudaStream_t st) {
    constexpr int smem = STAGES * (kABytes + BLOCK_N * kBlockK * 2 * (WS ? 2 : 1)) + (TMA_EPI ? ((WS ? 1 : 2) + 1) * kEpiTileBytes : 0) + 1024 + 256;
    static_assert((smem + 1024) * MIN_BLOCKS <= 228 * 1024, "shared memory budget");
    static bool attr_set = false;
    if (!attr_set) {
        NRPN_CUDA_TRY(cudaFuncSetAttribute(conv3d_igemm_kernel<BLOCK_N, STAGES, MIN_BLOCKS, TMA_EPI, WS>,
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        attr_set = true;
    }
    const int slots = num_sms() * MIN_BLOCKS;
    const int grid = total_tiles < slots ? total_tiles : slots;
    NRPN_CUDA_TRY(launch_pdl(conv3d_igemm_kernel<BLOCK_N, STAGES, MIN_BLOCKS, TMA_EPI, WS>, dim3(grid), dim3(kConvThreads), smem, st, total_tiles <= 2 * slots, maps, P));
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

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

// Split-K: layers with far fewer output tiles than SMs and a long reduction (late ResNet stages: 5x8x8 .. 10x16x16 voxels,
// K up to 13 824) are latency bound on streaming their weights through a handful of CTAs. The kernel can spread the
// k-blocks of each tile over `splits` CTAs (per-split fp32 slabs, last CTA reduces in a fixed order: bit-reproducible).
// The single-CTA slab reduction is serial, so the split is OFF unless NRPN_SPLITK=1 is set; batching several scenes per
// launch (bench.py --scenes-per-step) is what feeds these layers instead.
static int choose_splits(int total_tiles, int kblocks, bool short_k) {
    static const bool enabled = [] { const char* e = getenv("NRPN_SPLITK"); return e && e[0] == '1'; }();
    if (!enabled) return 1;
    if (short_k || kblocks < 8 || total_tiles * 2 > num_sms()) return 1;
    int s = num_sms() / total_tiles;
    if (s > kblocks / 4) s = kblocks / 4;
    if (s > 32) s = 32;
    return s < 2 ? 1 : s;
}

struct ConvGeom { int pad_n, cout_pad, block_n, kblocks, m_tiles, n_tiles_n, splits; bool short_k, tma_epi; size_t ws_bytes, counter_bytes; };

static int conv_geometry(const nrpn_conv_desc* d, ConvGeom& g) {
    g.pad_n = nrpn_conv3d_block_n(d->cout);
    g.cout_pad = ceil_div(d->cout, g.pad_n) * g.pad_n;
    g.kblocks = d->n_taps * (d->cin / kBlockK);
    g.short_k = g.kblocks <= 8;
    g.block_n = g.short_k ? 64 : g.pad_n;
    g.n_tiles_n = g.cout_pad / g.block_n;
    int tiles = 0;
    for (int l = 0; l < d->n_levels; ++l) {
        const nrpn_conv_level& S = d->level[l];
        if (S.n < 1 || S.xo < 1 || S.yo < 1 || S.zo < 1) return NRPN_ERR_INVALID;
        int bx, by, bz;
        choose_brick(S.xo, S.yo, S.zo, bx, by, bz);
        tiles += S.n * ceil_div(S.xo, bx) * ceil_div(S.yo, by) * ceil_div(S.zo, bz);
    }
    g.m_tiles = tiles;
    // Late ResNet stages (5x8x8 .. 10x16x16 voxels, K up to 13 824): a handful of 128 x 256 tiles leaves most SMs idle while each
    // tile runs a long reduction.  Two remedies: split-K over the full-width tiles (opt-in, NRPN_SPLITK=1, decided first so that it
    // reaches the layers it is meant for), otherwise -- the default -- 64-wide tiles when even those fit in one wave: 4x the CTAs
    // (same reduction order per output element, bit-identical results).
    g.splits = d->wsplit ? 1 : choose_splits(tiles * g.n_tiles_n, g.kblocks, g.short_k);
    if (g.splits == 1 && !g.short_k && g.block_n > 64 && tiles * (g.cout_pad / 64) <= num_sms()) {
        const char* e = getenv("NRPN_CONV_NARROW");
        if (!(e && e[0] == '0')) { g.block_n = 64; g.n_tiles_n = g.cout_pad / 64; }
    }
    g.counter_bytes = align_up((size_t)tiles * g.n_tiles_n * 4, 256);
    g.ws_bytes = g.splits > 1 ? g.counter_bytes + (size_t)tiles * g.n_tiles_n * g.splits * kBlockM * g.block_n * 4 : 0;
    // shared-memory (TMA) epilogue: the HBM-bound short reductions with whole 64-channel bf16 output tiles
    { const char* e = getenv("NRPN_CONV_TMA_EPI"); g.tma_epi = !(e && e[0] == '0'); }       // A/B switch for tests and profiling
    g.tma_epi = g.tma_epi && g.short_k && g.splits == 1 && !d->out_fp32 && d->cout % 64 == 0;
    for (int l = 0; l < d->n_levels && g.tma_epi; ++l) {
        const nrpn_conv_level& S = d->level[l];
        if (reinterpret_cast<uintptr_t>(S.y) % 16 != 0 || (S.res && reinterpret_cast<uintptr_t>(S.res) % 16 != 0)) g.tma_epi = false;
        // a nearest-upsampled residual (FPN top-down) is gathered per row from registers: the pipelined register epilogue
        // with 3 CTAs per SM is faster for it (measured: lat3+up 0.207 ms vs 0.275 ms)
        if (S.res && (S.xr != S.xo || S.yr != S.yo || S.zr != S.zo)) g.tma_epi = false;
    }
    return NRPN_OK;
}

}  // namespace nrpn

using namespace nrpn;

extern "C" {
#pragma GCC visibility push(default)

size_t nrpn_conv3d_workspace_bytes(const nrpn_conv_desc* d) {
    if (!d || d->cin < 64 || d->cin % 64 != 0 || d->n_levels < 1 || d->n_levels > NRPN_CONV_MAX_LEVELS || d->n_taps < 1) return 0;
    ConvGeom g;
    if (conv_geometry(d, g) != NRPN_OK) return 0;
    return g.ws_bytes;
}

int nrpn_conv3d_block_n(int cout) { return cout <= 64 ? 64 : (cout <= 128 ? 128 : 256); }

const char* nrpn_conv3d_variant(const nrpn_conv_desc* d) {
    if (!d || d->n_taps < 1 || d->n_taps > NRPN_CONV_MAX_TAPS || d->n_levels < 1 || d->n_levels > NRPN_CONV_MAX_LEVELS) return "invalid";
    if (d->cin < 64 || d->cin % 64 != 0 || d->cout < 8 || d->cout % 8 != 0 || (d->stride != 1 && d->stride != 2)) return "unsupported";
    if (!d->wsplit && conv3d_slab_eligible(d)) return "slab<4x16x8,N64>";
    ConvGeom g;
    if (conv_geometry(d, g) != NRPN_OK) return "invalid";
    if (d->wsplit) {
        if (g.short_k) return g.tma_epi ? "igemm<64,2,2,tma-epilogue,wsplit>" : "igemm<64,2,3,wsplit>";
        return g.block_n == 64 ? "igemm<64,6,1,wsplit>" : (g.block_n == 128 ? "igemm<128,4,1,wsplit>" : "igemm<256,2,1,wsplit>");
    }
    if (g.short_k) return g.tma_epi ? "igemm<64,2,2,tma-epilogue>" : "igemm<64,2,3>";
    return g.block_n == 64 ? "igemm<64,8,1>" : (g.block_n == 128 ? "igemm<128,6,1>" : "igemm<256,4,1>");
}

int nrpn_conv3d_fprop(const nrpn_conv_desc* d, nrpn_stream_t stream) {
    if (!d || !d->w || !d->shift) return NRPN_ERR_INVALID;
    if (d->cin < 64 || d->cin % 64 != 0 || d->cout < 8 || d->cout % 8 != 0) return NRPN_ERR_UNSUPPORTED;
    if (d->n_taps < 1 || d->n_taps > NRPN_CONV_MAX_TAPS || d->n_levels < 1 || d->n_levels > NRPN_CONV_MAX_LEVELS)
        return NRPN_ERR_INVALID;
    if (d->stride != 1 && d->stride != 2) return NRPN_ERR_UNSUPPORTED;
    if (d->stride == 2) {       // strided access is expressed through a sub-sampled tensor map: taps must not move
        for (int t = 0; t < d->n_taps; ++t)
            if (d->tap_off[t][0] || d->tap_off[t][1] || d->tap_off[t][2]) return NRPN_ERR_UNSUPPORTED;
    }
    EncodeTiledFn encode = get_encode();
    if (!encode) return NRPN_ERR_NO_DEVICE;
    if (!d->wsplit && conv3d_slab_eligible(d)) return conv3d_slab_launch(d, (cudaStream_t)stream);

    // Weights are padded to nrpn_conv3d_block_n(cout) (a multiple of 64). Long reductions (3^3 taps) use the widest N tile
    // that fits, one CTA per SM, deep smem ring: tensor-pipe bound.  Short reductions (1^3 convs: at most 8 k-blocks) are
    // HBM / epilogue-latency bound: they run N = 64 tiles with 3 CTAs per SM so that 3x more loads/stores are in flight.
    ConvGeom geo;
    { const int rc = conv_geometry(d, geo); if (rc) return rc; }
    const int cout_pad = geo.cout_pad;
    const bool short_k = geo.short_k;
    const int block_n = geo.block_n;
    int splits = geo.splits;
    if (splits > 1 && (!d->workspace || d->workspace_bytes < geo.ws_bytes)) splits = 1;      // no (or too small a) workspace: run unsplit
    ConvMaps maps;
    ConvDev P;
    memset(&P, 0, sizeof(P));
    P.n_levels = d->n_levels; P.n_taps = d->n_taps; P.kc_blocks = d->cin / kBlockK; P.n_tiles_n = cout_pad / block_n;
    P.cout = d->cout; P.relu = d->relu; P.out_fp32 = d->out_fp32; P.shift = d->shift; P.fp16 = d->act_fp16 ? 1 : 0;
    for (int t = 0; t < d->n_taps; ++t) { P.tap[t][0] = d->tap_off[t][0]; P.tap[t][1] = d->tap_off[t][1]; P.tap[t][2] = d->tap_off[t][2]; P.tap[t][3] = 0; }

    int tiles = 0;
    const int s = d->stride;
    for (int l = 0; l < d->n_levels; ++l) {
        const nrpn_conv_level& S = d->level[l];
        ConvLevelDev& L = P.lv[l];
        if (!S.x || !S.y || S.n < 1 || S.xi < 1 || S.yi < 1 || S.zi < 1 || S.xo < 1 || S.yo < 1 || S.zo < 1) return NRPN_ERR_INVALID;
        if (S.ldy < d->cout || S.ldy % 8 != 0) return NRPN_ERR_INVALID;
        if (S.res && (S.ldr < d->cout || S.ldr % 8 != 0 || S.xr < 1 || S.yr < 1 || S.zr < 1)) return NRPN_ERR_INVALID;
        if (s == 2 && (S.xo != (S.xi + 1) / 2 || S.yo != (S.yi + 1) / 2 || S.zo != (S.zi + 1) / 2)) return NRPN_ERR_INVALID;
        L.n = S.n; L.xo = S.xo; L.yo = S.yo; L.zo = S.zo;
        choose_brick(S.xo, S.yo, S.zo, L.bx, L.by, L.bz);
        L.tx = ceil_div(S.xo, L.bx); L.ty = ceil_div(S.yo, L.by); L.tz = ceil_div(S.zo, L.bz);
        L.tile_begin = tiles;
        tiles += S.n * L.tx * L.ty * L.tz;
        L.xr = S.res ? S.xr : S.xo; L.yr = S.res ? S.yr : S.yo; L.zr = S.res ? S.zr : S.zo;
        L.rsx = (float)L.xr / (float)S.xo; L.rsy = (float)L.yr / (float)S.yo; L.rsz = (float)L.zr / (float)S.zo;
        L.ldy = S.ldy; L.ldr = S.ldr; L.y = S.y; L.res = reinterpret_cast<const __nv_bfloat16*>(S.res);
        L.res_tma = (geo.tma_epi && S.res && S.xr == S.xo && S.yr == S.yo && S.zr == S.zo) ? 1 : 0;
        if (geo.tma_epi) {
            // output / residual tensors (C, Z, Y, X, N) with the row pitch ldy / ldr; one box = one 64-channel brick tile
            cuuint32_t ebox[5] = {64, (cuuint32_t)L.bz, (cuuint32_t)L.by, (cuuint32_t)L.bx, 1};
            cuuint32_t eone[5] = {1, 1, 1, 1, 1};
            cuuint64_t ydim[5] = {(cuuint64_t)d->cout, (cuuint64_t)S.zo, (cuuint64_t)S.yo, (cuuint64_t)S.xo, (cuuint64_t)S.n};
            cuuint64_t ystr[4] = {(cuuint64_t)S.ldy * 2, (cuuint64_t)S.zo * S.ldy * 2, (cuuint64_t)S.yo * S.zo * S.ldy * 2,
                                  (cuuint64_t)S.xo * S.yo * S.zo * S.ldy * 2};
            CUresult ry = encode(&maps.y[l], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, S.y, ydim, ystr, ebox, eone, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                 CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (ry != CUDA_SUCCESS) { g_last_cuda_error = (int)ry; return NRPN_ERR_CUDA; }
            if (L.res_tma) {
                cuuint64_t rstr[4] = {(cuuint64_t)S.ldr * 2, (cuuint64_t)S.zo * S.ldr * 2, (cuuint64_t)S.yo * S.zo * S.ldr * 2,
                                      (cuuint64_t)S.xo * S.yo * S.zo * S.ldr * 2};
                CUresult rr = encode(&maps.r[l], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(S.res), ydim, rstr, ebox, eone,
                                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
                if (rr != CUDA_SUCCESS) { g_last_cuda_error = (int)rr; return NRPN_ERR_CUDA; }
            } else maps.r[l] = maps.y[l];
        }

        // activation tensor map: (C, Z, Y, X, N), optionally sub-sampled by `stride` on the three spatial axes
        const cuuint64_t cin = (cuuint64_t)d->cin;
        cuuint64_t gdim[5] = {cin, (cuuint64_t)ceil_div(S.zi, s), (cuuint64_t)ceil_div(S.yi, s), (cuuint64_t)ceil_div(S.xi, s), (cuuint64_t)S.n};
        cuuint64_t gstr[4] = {cin * 2 * s, (cuuint64_t)S.zi * cin * 2 * s, (cuuint64_t)S.yi * S.zi * cin * 2 * s,
                              (cuuint64_t)S.xi * S.yi * S.zi * cin * 2};
        cuuint32_t box[5] = {(cuuint32_t)kBlockK, (cuuint32_t)L.bz, (cuuint32_t)L.by, (cuuint32_t)L.bx, 1};
        cuuint32_t estr[5] = {1, 1, 1, 1, 1};
        CUresult r = encode(&maps.x[l], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(S.x), gdim, gstr, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { g_last_cuda_error = (int)r; return NRPN_ERR_CUDA; }
    }
    for (int l = d->n_levels; l < NRPN_CONV_MAX_LEVELS; ++l) { maps.x[l] = maps.x[0]; maps.y[l] = maps.y[0]; maps.r[l] = maps.r[0]; }
    if (!geo.tma_epi) for (int l = 0; l < NRPN_CONV_MAX_LEVELS; ++l) { maps.y[l] = maps.x[0]; maps.r[l] = maps.x[0]; }
    {
        // wsplit: (taps, 2, CoutPad, cin) -- the hi and lo planes of a tap are consecutive slices, one box of depth 2 fetches both
        const int planes = d->wsplit ? 2 : 1;
        cuuint64_t gdim[3] = {(cuuint64_t)d->cin, (cuuint64_t)cout_pad, (cuuint64_t)d->n_taps * planes};
        cuuint64_t gstr[2] = {(cuuint64_t)d->cin * 2, (cuuint64_t)cout_pad * d->cin * 2};
        cuuint32_t box[3] = {(cuuint32_t)kBlockK, (cuuint32_t)block_n, (cuuint32_t)planes};
        cuuint32_t estr[3] = {1, 1, 1};
        CUresult r = encode(&maps.w, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(d->w), gdim, gstr, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { g_last_cuda_error = (int)r; return NRPN_ERR_CUDA; }
    }
    P.total_m_tiles = tiles;
    P.splits = splits; P.cout_pad = cout_pad;
    P.counters = reinterpret_cast<unsigned*>(d->workspace);
    P.ws = splits > 1 ? reinterpret_cast<float*>(reinterpret_cast<char*>(d->workspace) + geo.counter_bytes) : nullptr;
    const int total_tiles = tiles * P.n_tiles_n * splits;
    cudaStream_t st = (cudaStream_t)stream;
    if (d->wsplit) {
        if (splits != 1) return NRPN_ERR_UNSUPPORTED;
        if (short_k && geo.tma_epi) return launch_conv<64, 2, 2, true, true>(maps, P, total_tiles, st);
        if (short_k) return launch_conv<64, 2, 3, false, true>(maps, P, total_tiles, st);
        if (block_n == 64) return launch_conv<64, 6, 1, false, true>(maps, P, total_tiles, st);
        if (block_n == 128) return launch_conv<128, 4, 1, false, true>(maps, P, total_tiles, st);
        return launch_conv<256, 2, 1, false, true>(maps, P, total_tiles, st);
    }
    if (short_k && geo.tma_epi && splits == 1) return launch_conv<64, 2, 2, true>(maps, P, total_tiles, st);
    if (short_k) return launch_conv<64, 2, 3>(maps, P, total_tiles, st);
    if (block_n == 64) return launch_conv<64, 8, 1>(maps, P, total_tiles, st);
    if (block_n == 128) return launch_conv<128, 6, 1>(maps, P, total_tiles, st);
    return launch_conv<256, 4, 1>(maps, P, total_tiles, st);
}

#pragma GCC visibility pop
}  // extern "C"
