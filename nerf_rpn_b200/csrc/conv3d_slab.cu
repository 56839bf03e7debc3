// Halo-slab implicit-GEMM convolution for the narrow (64-channel) stride-1 layers of the path: the 7^3 stride-2 stem on
// the packed space-to-depth input (feature_extractor.py:163, 4 x 4 x 2 taps of K = 64) and the 3^3 64->64 convolutions
// of ResNet layer1 (feature_extractor.py:31-68).
//
// Why a second kernel: with N = 64 output channels a tap-by-tap brick kernel (conv3d_igemm.cu) re-reads one 16 KB
// activation box AND one 8 KB weight block from L2 for every (tap, 128-voxel tile): 24 KB per 0.5 MFMA, so it is bound by
// L2 bandwidth well below the tensor-core rate.
// Here one CTA owns a tile of 4 x-planes x 16 (y) x 8 (z) = 512 output voxels, i.e. FOUR 128 x 64 accumulators:
//   - z is the fastest spatial axis, so 8 z-neighbours x 64 channels form exactly one 1024-byte SWIZZLE_128B atom.  For
//     each distinct z offset of the filter (a "phase") the halo slab {z0+dz .. +8, y0+dy_min .. y0+15+dy_max,
//     x0+dx_min .. x0+3+dx_max} is streamed x-plane by x-plane (one TMA box {64 ch, 8 z, Ys y} per plane, out-of-range
//     voxels zero-filled = the convolution padding) into a ring of shared-memory slots;
//   - the A operand of tap (dx, dy) for accumulator a is the 16 consecutive atoms starting at atom (dy - dy_min) of
//     plane (dx - dx_min + a): a plain SWIZZLE_128B K-major descriptor with a different start address -- shifts along
//     y and x are free, only shifts along z need their own copy of the slab;
//   - every 8 KB weight block is used by 16 MMAs (4 accumulators x K 64/16) instead of 4.
// L2 traffic per 128 output voxels drops from 768 KB to ~130 KB (stem).
// Roles: warps 0-7 = two consumer warpgroups (rows 0-63 / 64-127 of every accumulator: 4 x m64n64 wgmma accumulators in
// registers, then + shift, ReLU, 16-bit stores), warp 8 = slab (A) producer, warp 9 = weight (B) producer.
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include "common.cuh"
#include "wgmma.cuh"
#include "conv_internal.cuh"

namespace nrpn {

constexpr int kSlabAcc = 4;              // x-planes (accumulators) per tile
constexpr int kSlabTileY = 16;
constexpr int kSlabTileZ = 8;
constexpr int kSlabMaxSlots = 12;
constexpr int kSlabBStages = 4;
constexpr int kSlabBBytes = 64 * 64 * 2; // one tap of weights: 64 (Cout, padded) x 64 (Cin) bf16
constexpr int kSlabMaxAxis = 8;          // at most 8 distinct offsets per axis
constexpr int kSlabConsumers = 256;
constexpr int kSlabThreads = kSlabConsumers + 64;
constexpr int kSlabSmemLimit = 227 * 1024;

struct SlabDev {
    int n, xo, yo, zo;
    int tx, ty, tz, total_tiles;
    int n_phases, ndx, ndy;
    int dx0, dy0;
    int planes, slots, plane_bytes;
    int cout, relu, ldy, fp16;
    signed char dz[kSlabMaxAxis];
    unsigned char dyrel[kSlabMaxAxis];
    unsigned char widx[kSlabMaxAxis][kSlabMaxAxis][kSlabMaxAxis];     // [phase][dx index][dy index] -> tap index of the packed weights
    const float* shift;
    __nv_bfloat16* y;
};

struct SlabMaps { CUtensorMap x, w; };

__global__ void __launch_bounds__(kSlabThreads, 1) conv3d_slab_kernel(const __grid_constant__ SlabMaps maps, const SlabDev P) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + (size_t)P.slots * P.plane_bytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_b + kSlabBStages * kSlabBBytes);
    uint64_t* a_full = bars;
    uint64_t* a_empty = bars + kSlabMaxSlots;
    uint64_t* b_full = bars + 2 * kSlabMaxSlots;
    uint64_t* b_empty = b_full + kSlabBStages;

    const int warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) {
        for (int s = 0; s < P.slots; ++s) { ptx::mbar_init(&a_full[s], 1); ptx::mbar_init(&a_empty[s], 2); }      // one arrival per consumer warpgroup
        for (int s = 0; s < kSlabBStages; ++s) { ptx::mbar_init(&b_full[s], 1); ptx::mbar_init(&b_empty[s], 2); }
        ptx::fence_barrier_init();
        ptx::prefetch_tmap(&maps.x);
        ptx::prefetch_tmap(&maps.w);
    }
    ptx::pdl_trigger();
    __syncthreads();
    ptx::pdl_wait();                    // prologue overlapped the previous kernel's tail; its outputs are visible from here

    if (warp == kSlabConsumers / 32) {
        // ---------------------------------------------------------------- slab producer: one x-plane per TMA
        const bool leader = ptx::elect_one();
        int slot = 0; uint32_t par = 0;
        for (int tile = blockIdx.x; tile < P.total_tiles; tile += gridDim.x) {
            int t = tile;
            const int tiz = t % P.tz; t /= P.tz;
            const int tiy = t % P.ty; t /= P.ty;
            const int tix = t % P.tx; const int nb = t / P.tx;
            const int x0 = tix * kSlabAcc + P.dx0, y0 = tiy * kSlabTileY + P.dy0, z0 = tiz * kSlabTileZ;
            for (int ph = 0; ph < P.n_phases; ++ph) {
                const int z = z0 + P.dz[ph];
                for (int p = 0; p < P.planes; ++p) {
                    ptx::mbar_wait(&a_empty[slot], par ^ 1u);
                    if (leader) {
                        ptx::mbar_expect_tx(&a_full[slot], (uint32_t)P.plane_bytes);
                        ptx::tma_load_5d(smem_a + (size_t)slot * P.plane_bytes, &maps.x, &a_full[slot], 0, z, y0, x0 + p, nb);
                    }
                    __syncwarp();
                    if (++slot == P.slots) { slot = 0; par ^= 1u; }
                }
            }
        }
        return;
    }
    if (warp == kSlabConsumers / 32 + 1) {
        // ---------------------------------------------------------------- weight producer: one tap (8 KB) per TMA
        const bool leader = ptx::elect_one();
        int stage = 0; uint32_t par = 0;
        for (int tile = blockIdx.x; tile < P.total_tiles; tile += gridDim.x) {
            for (int ph = 0; ph < P.n_phases; ++ph)
                for (int dxi = 0; dxi < P.ndx; ++dxi)
                    for (int dyi = 0; dyi < P.ndy; ++dyi) {
                        ptx::mbar_wait(&b_empty[stage], par ^ 1u);
                        if (leader) {
                            ptx::mbar_expect_tx(&b_full[stage], kSlabBBytes);
                            ptx::tma_load_3d(smem_b + stage * kSlabBBytes, &maps.w, &b_full[stage], 0, 0, (int)P.widx[ph][dxi][dyi]);
                        }
                        __syncwarp();
                        if (++stage == kSlabBStages) { stage = 0; par ^= 1u; }
                    }
        }
        return;
    }

    // -------------------------------------------------------------------- consumers: MMA + epilogue
    const int t = threadIdx.x & 127, wg = threadIdx.x >> 7;
    const uint32_t sa0 = ptx::smem_u32(smem_a) + (uint32_t)(wg * 8192), sb0 = ptx::smem_u32(smem_b);     // rows 64 wg .. 64 wg + 63
    int a_slot = 0; uint32_t a_par = 0;          // ring position of plane 0 of the current phase
    int b_stage = 0; uint32_t b_par = 0;
    float acc[kSlabAcc][32];
    for (int tile = blockIdx.x; tile < P.total_tiles; tile += gridDim.x) {
        uint32_t accumulate = 0;
#pragma unroll
        for (int a = 0; a < kSlabAcc; ++a) ptx::reg_fence(acc[a]);
        for (int ph = 0; ph < P.n_phases; ++ph) {
            int waited = 0;
            for (int dxi = 0; dxi < P.ndx; ++dxi) {
                while (waited <= dxi + kSlabAcc - 1) {          // planes become visible in ring order
                    int s = a_slot + waited; uint32_t pr = a_par;
                    if (s >= P.slots) { s -= P.slots; pr ^= 1u; }
                    ptx::mbar_wait(&a_full[s], pr);
                    ++waited;
                }
                uint64_t plane_desc[kSlabAcc];
#pragma unroll
                for (int a = 0; a < kSlabAcc; ++a) {
                    int s = a_slot + dxi + a;
                    if (s >= P.slots) s -= P.slots;
                    plane_desc[a] = ptx::make_desc_sw128(sa0 + (uint32_t)(s * P.plane_bytes));
                }
                for (int dyi = 0; dyi < P.ndy; ++dyi) {
                    const uint64_t yoff = (uint64_t)P.dyrel[dyi] * 64u;          // dy atoms of 1024 B, in the >>4 address field
                    ptx::mbar_wait(&b_full[b_stage], b_par);
                    const uint64_t db = ptx::make_desc_sw128(sb0 + (uint32_t)(b_stage * kSlabBBytes));
                    auto issue = [&](auto f16) {
                        ptx::wgmma_fence();
#pragma unroll
                        for (int a = 0; a < kSlabAcc; ++a) {
                            const uint64_t da = plane_desc[a] + yoff;
#pragma unroll
                            for (int k = 0; k < 4; ++k)
                                ptx::Wgmma<64, decltype(f16)::value>::template ss<0, 0>(acc[a], da + (uint64_t)(2 * k), db + (uint64_t)(2 * k),
                                                                                         (accumulate | (uint32_t)k) ? 1u : 0u);
                        }
                        ptx::wgmma_commit();
                    };
                    if (P.fp16) issue(std::true_type{}); else issue(std::false_type{});
                    ptx::wgmma_wait<0>();
                    if (t == 0) ptx::mbar_arrive(&b_empty[b_stage]);
                    accumulate = 1u;
                    if (++b_stage == kSlabBStages) { b_stage = 0; b_par ^= 1u; }
                }
                // plane p is last read by (dx index min(p, ndx-1)): release what this dx index finished with
                const int p_lo = dxi, p_hi = (dxi == P.ndx - 1) ? P.planes - 1 : dxi;
                for (int p = p_lo; p <= p_hi; ++p) {
                    int s = a_slot + p;
                    if (s >= P.slots) s -= P.slots;
                    if (t == 0) ptx::mbar_arrive(&a_empty[s]);
                }
            }
            a_slot += P.planes;
            if (a_slot >= P.slots) { a_slot -= P.slots; a_par ^= 1u; }
        }
#pragma unroll
        for (int a = 0; a < kSlabAcc; ++a) ptx::reg_fence(acc[a]);

        // ---- epilogue: accumulator row = (y, z) inside the tile, z fastest
        int tt = tile;
        const int tiz = tt % P.tz; tt /= P.tz;
        const int tiy = tt % P.ty; tt /= P.ty;
        const int tix = tt % P.tx; const int nb = tt / P.tx;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = wg * 64 + ptx::frag_row(t, h);
            const int gy = tiy * kSlabTileY + (row >> 3), gz = tiz * kSlabTileZ + (row & 7);
            if (gy >= P.yo || gz >= P.zo) continue;
#pragma unroll
            for (int a = 0; a < kSlabAcc; ++a) {
                const int gx = tix * kSlabAcc + a;
                if (gx >= P.xo) continue;
                __nv_bfloat16* o = P.y + ((((size_t)nb * P.xo + gx) * P.yo + gy) * P.zo + gz) * P.ldy;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int ch = ptx::frag_col(t, j);
                    if (ch >= P.cout) continue;
                    const float2 s = __ldg(reinterpret_cast<const float2*>(P.shift + ch));
                    float v0 = acc[a][4 * j + 2 * h] + s.x, v1 = acc[a][4 * j + 2 * h + 1] + s.y;
                    if (P.relu == 1) { v0 = fmaxf(v0, 0.0f); v1 = fmaxf(v1, 0.0f); }
                    else if (P.relu == 2) { v0 = 0.5f * v0 * (1.0f + erff(v0 * 0.70710678118654752f)); v1 = 0.5f * v1 * (1.0f + erff(v1 * 0.70710678118654752f)); }
                    *reinterpret_cast<uint32_t*>(o + ch) = pack_act2(v0, v1, P.fp16);
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ host
// Decomposes the tap table into {z offsets} x {contiguous x offsets} x {y offsets}; false if it is not such a full box.
static bool slab_plan(const nrpn_conv_desc* d, SlabDev& P) {
    { const char* e = getenv("NRPN_CONV_SLAB"); if (e && e[0] == '0') return false; }   // A/B switch for tests and profiling
    if (d->cin != 64 || d->cout > 64 || d->cout % 8 != 0 || d->stride != 1 || d->n_levels != 1 || d->out_fp32) return false;
    if (d->n_taps < 8 || d->n_taps > NRPN_CONV_MAX_TAPS) return false;
    const nrpn_conv_level& S = d->level[0];
    if (S.res != nullptr) return false;
    if (S.xi < 1 || S.yi < 1 || S.zi < 1 || S.xo < 1 || S.yo < 1 || S.zo < 1) return false;   // input may be larger (packed stem: Z/2 + 1 rows)
    int vz[kSlabMaxAxis], vx[kSlabMaxAxis], vy[kSlabMaxAxis], nz = 0, nx = 0, ny = 0;
    auto insert = [](int* v, int& n, int val) -> bool {
        int i = 0;
        while (i < n && v[i] < val) ++i;
        if (i < n && v[i] == val) return true;
        if (n == kSlabMaxAxis) return false;
        for (int j = n; j > i; --j) v[j] = v[j - 1];
        v[i] = val; ++n;
        return true;
    };
    for (int t = 0; t < d->n_taps; ++t)
        if (!insert(vx, nx, d->tap_off[t][0]) || !insert(vy, ny, d->tap_off[t][1]) || !insert(vz, nz, d->tap_off[t][2])) return false;
    if (nx * ny * nz != d->n_taps) return false;
    if (vx[nx - 1] - vx[0] != nx - 1) return false;                     // slab planes are consecutive in x
    memset(P.widx, 0xFF, sizeof(P.widx));
    for (int t = 0; t < d->n_taps; ++t) {
        int iz = 0, ix = 0, iy = 0;
        while (vz[iz] != d->tap_off[t][2]) ++iz;
        while (vx[ix] != d->tap_off[t][0]) ++ix;
        while (vy[iy] != d->tap_off[t][1]) ++iy;
        if (P.widx[iz][ix][iy] != 0xFF) return false;                   // duplicate tap
        P.widx[iz][ix][iy] = (unsigned char)t;
    }
    const int ys = kSlabTileY + vy[ny - 1] - vy[0];
    if (ys > 256 || ys - kSlabTileY > 255) return false;
    P.n_phases = nz; P.ndx = nx; P.ndy = ny; P.dx0 = vx[0]; P.dy0 = vy[0];
    for (int i = 0; i < nz; ++i) P.dz[i] = (signed char)vz[i];
    for (int i = 0; i < ny; ++i) P.dyrel[i] = (unsigned char)(vy[i] - vy[0]);
    P.plane_bytes = ys * 1024;
    P.planes = kSlabAcc + nx - 1;
    const int avail = kSlabSmemLimit - 1024 - kSlabBStages * kSlabBBytes - 512;
    int slots = avail / P.plane_bytes;
    if (slots > kSlabMaxSlots) slots = kSlabMaxSlots;
    if (slots < P.planes + 1) return false;                            // the ring must hold a whole phase plus one plane in flight
    P.slots = slots;
    return true;
}

bool conv3d_slab_eligible(const nrpn_conv_desc* d) {
    SlabDev P;
    return slab_plan(d, P);
}

int conv3d_slab_launch(const nrpn_conv_desc* d, cudaStream_t st) {
    SlabDev P;
    memset(&P, 0, sizeof(P));
    if (!slab_plan(d, P)) return NRPN_ERR_UNSUPPORTED;
    const nrpn_conv_level& S = d->level[0];
    if (!S.x || !S.y || S.n < 1 || S.xo < 1 || S.yo < 1 || S.zo < 1) return NRPN_ERR_INVALID;
    if (S.ldy < d->cout || S.ldy % 8 != 0) return NRPN_ERR_INVALID;
    EncodeTiledFn encode = get_encode();
    if (!encode) return NRPN_ERR_NO_DEVICE;
    P.n = S.n; P.xo = S.xo; P.yo = S.yo; P.zo = S.zo;
    P.tx = ceil_div(S.xo, kSlabAcc); P.ty = ceil_div(S.yo, kSlabTileY); P.tz = ceil_div(S.zo, kSlabTileZ);
    P.total_tiles = S.n * P.tx * P.ty * P.tz;
    P.fp16 = d->act_fp16 ? 1 : 0;
    P.cout = d->cout; P.relu = d->relu; P.ldy = S.ldy; P.shift = d->shift; P.y = reinterpret_cast<__nv_bfloat16*>(S.y);

    SlabMaps maps;
    {   // activations (C, Z, Y, X, N): one box = one x-plane of the slab, {64 ch, 8 z, Ys y}
        cuuint64_t gdim[5] = {64, (cuuint64_t)S.zi, (cuuint64_t)S.yi, (cuuint64_t)S.xi, (cuuint64_t)S.n};
        cuuint64_t gstr[4] = {128, (cuuint64_t)S.zi * 128, (cuuint64_t)S.yi * S.zi * 128, (cuuint64_t)S.xi * S.yi * S.zi * 128};
        cuuint32_t box[5] = {64, (cuuint32_t)kSlabTileZ, (cuuint32_t)(P.plane_bytes / 1024), 1, 1};
        cuuint32_t estr[5] = {1, 1, 1, 1, 1};
        CUresult r = encode(&maps.x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(S.x), gdim, gstr, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { g_last_cuda_error = (int)r; return NRPN_ERR_CUDA; }
    }
    {   // weights (Cin, CoutPad = 64, taps)
        cuuint64_t gdim[3] = {64, 64, (cuuint64_t)d->n_taps};
        cuuint64_t gstr[2] = {128, 64 * 128};
        cuuint32_t box[3] = {64, 64, 1};
        cuuint32_t estr[3] = {1, 1, 1};
        CUresult r = encode(&maps.w, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(d->w), gdim, gstr, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { g_last_cuda_error = (int)r; return NRPN_ERR_CUDA; }
    }
    const int smem = 1024 + P.slots * P.plane_bytes + kSlabBStages * kSlabBBytes + 512;
    static int smem_set = 0;
    if (smem > smem_set) {
        NRPN_CUDA_TRY(cudaFuncSetAttribute(conv3d_slab_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        smem_set = smem;
    }
    const int grid = P.total_tiles < num_sms() ? P.total_tiles : num_sms();
    NRPN_CUDA_TRY(launch_pdl(conv3d_slab_kernel, dim3(grid), dim3(kSlabThreads), smem, st, P.total_tiles <= 2 * num_sms(), maps, P));
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

}  // namespace nrpn
