// GroupNorm(32, 256) + ReLU on channels-last 16-bit (bf16 or fp16, selected by act_fp16) activations, in place (FCOS towers,
// Conv3d -> GroupNorm -> ReLU, fcos/fcos.py:43-69).  Statistics are per (sample, pyramid level, group) over 8 channels x all voxels.
// Two kernels per call, HBM bound: (1) per-CTA partial sums (fp32 per thread, fp64 across threads) written to a scratch
// array, (2) every CTA first reduces the partials of its (sample, level) in a FIXED order (bit-reproducible), then applies
// y = relu((x - mean) * rstd * gamma + beta).  One thread owns one 16-byte chunk = the 8 channels of one group of one
// voxel, so a warp reads 512 contiguous bytes.  Up to 4 pyramid levels per launch.
#include "common.cuh"

namespace nrpn {

constexpr int kGnMaxBlocks = 512;    // CTAs per (level, sample): ceil(voxels / 64), at most this many
constexpr int kGnGroups = 32;

struct GnDev {
    int n_levels, n, relu, fp16;
    float eps;
    __nv_bfloat16* x[NRPN_CONV_MAX_LEVELS];
    int voxels[NRPN_CONV_MAX_LEVELS];
    int blocks[NRPN_CONV_MAX_LEVELS];      // CTAs per sample for this level
    int block_begin[NRPN_CONV_MAX_LEVELS]; // first CTA index of the level (levels are laid out back to back, samples inside)
    const float* gamma; const float* beta;
    double* partial;                 // [global CTA][group][2]
};

__device__ __forceinline__ void gn_locate(const GnDev& P, int cta, int& l, int& smp, int& blk) {
    l = 0;
#pragma unroll
    for (int i = 1; i < NRPN_CONV_MAX_LEVELS; ++i) if (i < P.n_levels && cta >= P.block_begin[i]) l = i;
    const int r = cta - P.block_begin[l];
    smp = r / P.blocks[l]; blk = r - smp * P.blocks[l];
}

__global__ void __launch_bounds__(256) gn_stats_kernel(GnDev P) {
    int l, smp, blk;
    gn_locate(P, blockIdx.x, l, smp, blk);
    const int V = P.voxels[l], nb = P.blocks[l];
    const __nv_bfloat16* x = P.x[l] + (size_t)smp * V * 256;
    const int g = threadIdx.x & 31, r = threadIdx.x >> 5;       // 32 groups x 8 rows per CTA step
    float s = 0.f, q = 0.f;
    const int step = nb * 8;
    int v = blk * 8 + r;
    for (; v + 3 * step < V; v += 4 * step) {                  // four independent 16-byte loads in flight per thread
        uint4 raw[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) raw[u] = __ldg(reinterpret_cast<const uint4*>(x + (size_t)(v + u * step) * 256 + g * 8));
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const uint32_t* h = reinterpret_cast<const uint32_t*>(&raw[u]);
#pragma unroll
            for (int i = 0; i < 4; ++i) { const float2 f = unpack_act2(h[i], P.fp16); s += f.x + f.y; q += f.x * f.x + f.y * f.y; }
        }
    }
    for (; v < V; v += step) {
        const uint4 raw = __ldg(reinterpret_cast<const uint4*>(x + (size_t)v * 256 + g * 8));
        const uint32_t* h = reinterpret_cast<const uint32_t*>(&raw);
#pragma unroll
        for (int i = 0; i < 4; ++i) { const float2 f = unpack_act2(h[i], P.fp16); s += f.x + f.y; q += f.x * f.x + f.y * f.y; }
    }
    __shared__ double ss[8][32], sq[8][32];
    ss[r][g] = (double)s; sq[r][g] = (double)q;
    __syncthreads();
    if (r == 0) {
        double a = 0.0, b = 0.0;
#pragma unroll
        for (int i = 0; i < 8; ++i) { a += ss[i][g]; b += sq[i][g]; }
        double* o = P.partial + ((size_t)blockIdx.x * kGnGroups + g) * 2;
        o[0] = a; o[1] = b;
    }
}

__global__ void __launch_bounds__(256) gn_apply_kernel(GnDev P) {
    int l, smp, blk;
    gn_locate(P, blockIdx.x, l, smp, blk);
    const int V = P.voxels[l], nb = P.blocks[l];
    __nv_bfloat16* x = P.x[l] + (size_t)smp * V * 256;
    const int g = threadIdx.x & 31, r = threadIdx.x >> 5;
    __shared__ double red[8][32][2];
    __shared__ float mean_s[32], rstd_s[32];
    {   // every CTA reduces the partial sums of its (level, sample) in the same fixed order: bit-reproducible
        const double* p = P.partial + ((size_t)(P.block_begin[l] + smp * nb) * kGnGroups) * 2;
        double a = 0.0, b = 0.0;
        for (int i = r; i < nb; i += 8) { a += p[((size_t)i * kGnGroups + g) * 2]; b += p[((size_t)i * kGnGroups + g) * 2 + 1]; }
        red[r][g][0] = a; red[r][g][1] = b;
    }
    __syncthreads();
    if (r == 0) {
        double a = 0.0, b = 0.0;
#pragma unroll
        for (int i = 0; i < 8; ++i) { a += red[i][g][0]; b += red[i][g][1]; }
        const double cnt = (double)V * 8.0;
        const double m = a / cnt;
        double var = b / cnt - m * m;                      // biased variance, as torch.nn.GroupNorm
        if (var < 0.0) var = 0.0;
        mean_s[g] = (float)m;
        rstd_s[g] = (float)(1.0 / sqrt(var + (double)P.eps));
    }
    __syncthreads();
    const float mean = mean_s[g], rstd = rstd_s[g];
    float ga[8], be[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { ga[i] = __ldg(P.gamma + g * 8 + i) * rstd; be[i] = __ldg(P.beta + g * 8 + i) - mean * ga[i]; }
    const int step = nb * 8;
    auto apply = [&](uint4 raw) {
        uint32_t* h = reinterpret_cast<uint32_t*>(&raw);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float2 f = unpack_act2(h[i], P.fp16);
            f.x = f.x * ga[2 * i] + be[2 * i]; f.y = f.y * ga[2 * i + 1] + be[2 * i + 1];
            if (P.relu) { f.x = fmaxf(f.x, 0.f); f.y = fmaxf(f.y, 0.f); }
            h[i] = pack_act2(f.x, f.y, P.fp16);
        }
        return raw;
    };
    int v = blk * 8 + r;
    for (; v + 3 * step < V; v += 4 * step) {
        uint4 raw[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) raw[u] = *reinterpret_cast<const uint4*>(x + (size_t)(v + u * step) * 256 + g * 8);
#pragma unroll
        for (int u = 0; u < 4; ++u) *reinterpret_cast<uint4*>(x + (size_t)(v + u * step) * 256 + g * 8) = apply(raw[u]);
    }
    for (; v < V; v += step) {
        uint4* ptr = reinterpret_cast<uint4*>(x + (size_t)v * 256 + g * 8);
        *ptr = apply(*ptr);
    }
}

}  // namespace nrpn

using namespace nrpn;

extern "C" {
#pragma GCC visibility push(default)

size_t nrpn_groupnorm_workspace_bytes(int n_levels, int n) {
    if (n_levels < 1 || n_levels > NRPN_CONV_MAX_LEVELS || n < 1) return 0;
    return (size_t)n_levels * n * kGnMaxBlocks * kGnGroups * 2 * sizeof(double);
}

int nrpn_groupnorm_relu(const nrpn_gn_level* levels, int n_levels, int n, int c, int groups, const float* gamma,
                        const float* beta, float eps, int relu, int act_fp16, void* workspace, size_t workspace_bytes, nrpn_stream_t stream) {
    if (!levels || !gamma || !beta || !workspace || n_levels < 1 || n_levels > NRPN_CONV_MAX_LEVELS || n < 1) return NRPN_ERR_INVALID;
    if (c != 256 || groups != 32) return NRPN_ERR_UNSUPPORTED;       // 8 channels per group = one 16-byte chunk per thread
    if (workspace_bytes < nrpn_groupnorm_workspace_bytes(n_levels, n)) return NRPN_ERR_WORKSPACE;
    GnDev P;
    P.n_levels = n_levels; P.n = n; P.relu = relu; P.fp16 = act_fp16 ? 1 : 0; P.eps = eps; P.gamma = gamma; P.beta = beta;
    P.partial = reinterpret_cast<double*>(workspace);
    int grid = 0;
    for (int l = 0; l < n_levels; ++l) {
        if (!levels[l].x || levels[l].voxels < 1) return NRPN_ERR_INVALID;
        P.x[l] = reinterpret_cast<__nv_bfloat16*>(levels[l].x); P.voxels[l] = levels[l].voxels;
        int nb = ceil_div(levels[l].voxels, 64);
        if (nb > kGnMaxBlocks) nb = kGnMaxBlocks;
        P.blocks[l] = nb; P.block_begin[l] = grid;
        grid += nb * n;
    }
    gn_stats_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(P);
    NRPN_LAUNCH_CHECK();
    gn_apply_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(P);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

#pragma GCC visibility pop
}  // extern "C"
