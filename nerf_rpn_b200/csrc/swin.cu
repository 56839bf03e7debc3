// Swin-3D support kernels (SwinTransformer_FPN, nerf_rpn/model/feature_extractor.py:382-789). The GEMMs of the transformer
// (qkv, proj, MLP, patch merging, patch embedding) run on the wgmma implicit-GEMM kernel as 1x1x1 convolutions over
// channels-last token grids; this file holds what is left around them:
//   patch_embed_pack      fp32 NCDHW grid -> (X/4, Y/4, Z/4, 256) 16-bit patch rows  (Conv3d k4 s4 as a GEMM, :731-733)
//   layernorm             per-token LayerNorm over C channels                        (:621,634,736)
//   patch_merge_ln        2x2x2 gather (zero pad on odd extents) + LayerNorm(8C)     (:661-685)
//   window_attention      4^3 shifted-window multi-head attention, head_dim 32        (:382-497)
// Activations are (N, H, W, D, ld) 16-bit -- bf16 or fp16, selected by act_fp16 -- with C real channels and ld >= C.
#include "common.cuh"
#include "wgmma.cuh"

namespace nrpn {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ---------------------------------------------------------------------------------------------- patch embedding
// row (i,j,k) channel ((c*4+px)*4+py)*4+pz = grid[c][4i+px][4j+py][4k+pz]; one thread per 16-byte chunk (8 channels =
// fixed c,px,py half of pz... 8 consecutive channels = pz 0..3 for py and py+1).
__global__ void patch_embed_pack_kernel(const float* __restrict__ grid, int n, int X, int Y, int Z, int H, int W, int D,
                                        __nv_bfloat16* __restrict__ out, int fp16) {
    const size_t total = (size_t)n * H * W * D * 32;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
        const int s = (int)(t & 31);
        size_t v = t >> 5;
        const int k = (int)(v % D); v /= D;
        const int j = (int)(v % W); v /= W;
        const int i = (int)(v % H); const int b = (int)(v / H);
        // chunk s covers channels 8s..8s+7: c = s/8, px = (s/2)%4, py = (s%2)*2 + {0,1}, pz = 0..3
        const int c = s >> 3, px = (s >> 1) & 3, py0 = (s & 1) * 2;
        float val[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int py = py0 + (e >> 2), pz = e & 3;
            val[e] = grid[((((size_t)b * 4 + c) * X + 4 * i + px) * Y + 4 * j + py) * Z + 4 * k + pz];
        }
        uint32_t h[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) h[q] = pack_act2(val[2 * q], val[2 * q + 1], fp16);
        *reinterpret_cast<uint4*>(out + (t << 3)) = make_uint4(h[0], h[1], h[2], h[3]);
    }
}

// ---------------------------------------------------------------------------------------------- LayerNorm
// one warp per token; two passes over the row held in registers (C <= 3072 -> <= 96 values per lane)
__global__ void __launch_bounds__(256) layernorm_kernel(const __nv_bfloat16* __restrict__ in, int ld_in, __nv_bfloat16* __restrict__ out,
                                                        int ld_out, long tokens, int C, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, float eps, int fp16) {
    const long tok = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (tok >= tokens) return;
    const __nv_bfloat16* x = in + tok * ld_in;
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s += load_act(x + c, fp16);
    const float mean = warp_sum(s) / (float)C;
    float q = 0.f;
    for (int c = lane; c < C; c += 32) { const float d = load_act(x + c, fp16) - mean; q += d * d; }
    const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
    __nv_bfloat16* y = out + tok * ld_out;
    for (int c = lane; c < C; c += 32) store_act(y + c, (load_act(x + c, fp16) - mean) * rstd * gamma[c] + beta[c], fp16);
}

// ---------------------------------------------------------------------------------------------- patch merging
// output token (i,j,k) of the (ceil(H/2), ceil(W/2), ceil(D/2)) grid = LN(concat of the 8 input tokens (2i+a, 2j+b, 2k+c)),
// parity order 000,100,010,110,001,101,011,111 over (H,W,D), zero for positions past an odd extent.
__global__ void __launch_bounds__(256) patch_merge_ln_kernel(const __nv_bfloat16* __restrict__ in, int ld_in, int n, int H, int W, int D, int C,
                                                             __nv_bfloat16* __restrict__ out, const float* __restrict__ gamma,
                                                             const float* __restrict__ beta, float eps, int fp16) {
    const int Ho = (H + 1) / 2, Wo = (W + 1) / 2, Do = (D + 1) / 2;
    const long tokens = (long)n * Ho * Wo * Do;
    const long tok = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (tok >= tokens) return;
    long v = tok;
    const int k = (int)(v % Do); v /= Do;
    const int j = (int)(v % Wo); v /= Wo;
    const int i = (int)(v % Ho); const int b = (int)(v / Ho);
    const int C8 = 8 * C;
    auto src = [&](int c8) -> float {
        const int part = c8 / C, c = c8 - part * C;
        const int a = part & 1, bb = (part >> 1) & 1, cc = (part >> 2) & 1;
        const int h = 2 * i + a, w = 2 * j + bb, d = 2 * k + cc;
        if (h >= H || w >= W || d >= D) return 0.f;
        return load_act(in + ((((size_t)b * H + h) * W + w) * D + d) * ld_in + c, fp16);
    };
    float s = 0.f;
    for (int c = lane; c < C8; c += 32) s += src(c);
    const float mean = warp_sum(s) / (float)C8;
    float q = 0.f;
    for (int c = lane; c < C8; c += 32) { const float d = src(c) - mean; q += d * d; }
    const float rstd = rsqrtf(warp_sum(q) / (float)C8 + eps);
    __nv_bfloat16* y = out + tok * C8;
    for (int c = lane; c < C8; c += 32) store_act(y + c, (src(c) - mean) * rstd * gamma[c] + beta[c], fp16);
}

// ---------------------------------------------------------------------------------------------- window attention on wgmma
// Window w of the zero-padded, cyclically shifted grid: padded coordinate p -> source coordinate (p + shift) mod P; sources past
// the real extent are padding tokens whose q/k/v equal the qkv bias (the reference pads AFTER norm1, so padded tokens enter the
// Linear as zeros).
struct AttnDev {
    const __nv_bfloat16* qkv; int ld_qkv;      // (N,H,W,D, 3C): [q | k | v], each head-major (head*32 + d)
    __nv_bfloat16* out; int ld_out;            // (N,H,W,D, ld): heads concatenated
    const float* qkv_bias;                     // (3C)
    const float* table;                        // (343, heads) relative position bias table
    int n, H, W, D, C, heads;
    int PH, PW, PD, sh, sw, sd;                // padded extents, effective shifts
    int nwh, nww, nwd;
    int fp16;                                  // 16-bit format of qkv / out: 0 bf16, 1 fp16
};

// One warpgroup per (64-token window, head): S = Q K^T is an m64n64k32 wgmma into registers; softmax runs on the accumulator
// fragments (a row's 64 scores are spread over the 4 threads of a quad: scale, relative-position bias, -100 region mask, exp,
// max and sum through quad shuffles); the un-normalised probabilities go to shared memory as 16-bit values and O = P V is a
// second wgmma (M 64, N 32, K 64) against V^T.  The 1/sum normalisation is applied to the fp32 accumulator.  Operands are
// written to shared memory by the threads themselves (a token's q/k/v are 64 contiguous bytes each) in the 128B-swizzled
// K-major layout; V is transposed on the way.  Two warpgroups per CTA work on two windows of the same head independently.
constexpr int kAttnThreads = 256;
constexpr int kAttnWgBytes = 8192 /*Q*/ + 8192 /*K*/ + 4096 /*V^T*/ + 8192 /*P*/;
constexpr int kAttnSmem = 2 * kAttnWgBytes + 1024 /*align*/ + 1408 /*table*/ + 512 /*regions*/;

__device__ __forceinline__ uint32_t attn_sw(int row, int chunk) { return (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4)); }

struct AttnTok { bool real; size_t tok; int ph, pw, pd; };

__device__ __forceinline__ AttnTok attn_tok(const AttnDev& P, int w, int tw) {
    AttnTok a;
    const int wd = w % P.nwd; w /= P.nwd;
    const int ww = w % P.nww; w /= P.nww;
    const int wh = w % P.nwh; const int b = w / P.nwh;
    a.ph = wh * 4 + (tw >> 4); a.pw = ww * 4 + ((tw >> 2) & 3); a.pd = wd * 4 + (tw & 3);   // position in the padded, shifted grid
    const int sh_ = (a.ph + P.sh) % P.PH, sw_ = (a.pw + P.sw) % P.PW, sd_ = (a.pd + P.sd) % P.PD;
    a.real = sh_ < P.H && sw_ < P.W && sd_ < P.D;
    a.tok = (((size_t)b * P.H + sh_) * P.W + sw_) * P.D + sd_;
    return a;
}

template <bool F16>
__device__ __forceinline__ void attn_mma_s(float (&s)[32], uint64_t dq, uint64_t dk) {
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < 2; ++k)                                   // head_dim 32 = two K-steps of 16
        ptx::Wgmma<64, F16>::template ss<0, 0>(s, dq + (uint64_t)(2 * k), dk + (uint64_t)(2 * k), k ? 1u : 0u);
    ptx::wgmma_commit();
}
template <bool F16>
__device__ __forceinline__ void attn_mma_o(float (&o)[16], uint64_t dp, uint64_t dv) {
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)                                   // 64 keys = four K-steps of 16
        ptx::Wgmma<32, F16>::template ss<0, 0>(o, dp + (uint64_t)(2 * k), dv + (uint64_t)(2 * k), k ? 1u : 0u);
    ptx::wgmma_commit();
}

__global__ void __launch_bounds__(kAttnThreads, 2) window_attention_tc_kernel(AttnDev P, int n_windows) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int t = threadIdx.x & 127, wg = threadIdx.x >> 7;
    uint8_t* Qs = smem + wg * kAttnWgBytes;
    uint8_t* Ks = Qs + 8192;
    uint8_t* Vt = Qs + 16384;                   // [32 rows (d)][64 tokens]
    uint8_t* Ps = Qs + 20480;                   // [64 rows (queries)][64 keys]
    float* tbl = reinterpret_cast<float*>(smem + 2 * kAttnWgBytes);          // 343 relative-position biases of this head
    int* region = reinterpret_cast<int*>(smem + 2 * kAttnWgBytes + 1408) + wg * 64;
    const int head = blockIdx.y;
    const int hc = head * 32;
    for (int i = threadIdx.x; i < 343; i += kAttnThreads) tbl[i] = P.table[i * P.heads + head];
    __syncthreads();
    const bool shifted = (P.sh + P.sw + P.sd) > 0;
    const uint64_t dq = ptx::make_desc_sw128(ptx::smem_u32(Qs)), dk = ptx::make_desc_sw128(ptx::smem_u32(Ks));
    const uint64_t dv = ptx::make_desc_sw128(ptx::smem_u32(Vt)), dp = ptx::make_desc_sw128(ptx::smem_u32(Ps));
    for (int pair = blockIdx.x; pair * 2 < n_windows; pair += gridDim.x) {
        const int w = pair * 2 + wg;
        if (w >= n_windows) break;
        {   // ---- stage: threads 0-63 write q and k of token t (rows of the K-major tiles), threads 64-127 v (column of V^T)
            const int tw = t & 63;
            const AttnTok a = attn_tok(P, w, tw);
            const __nv_bfloat16* row = P.qkv + a.tok * P.ld_qkv;
            auto load = [&](int off, int i) -> uint4 {           // 8 channels of q / k / v; padding tokens carry the qkv bias
                if (a.real) return __ldg(reinterpret_cast<const uint4*>(row + off + hc) + i);
                uint32_t u[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) u[k] = pack_act2(P.qkv_bias[off + hc + i * 8 + 2 * k], P.qkv_bias[off + hc + i * 8 + 2 * k + 1], P.fp16);
                return make_uint4(u[0], u[1], u[2], u[3]);
            };
            if (t < 64) {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    *reinterpret_cast<uint4*>(Qs + attn_sw(tw, i)) = load(0, i);
                    *reinterpret_cast<uint4*>(Ks + attn_sw(tw, i)) = load(P.C, i);
                }
            } else {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const uint4 vv = load(2 * P.C, i);
                    const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(&vv);
#pragma unroll
                    for (int u = 0; u < 8; ++u) *reinterpret_cast<__nv_bfloat16*>(Vt + attn_sw(i * 8 + u, tw >> 3) + (tw & 7) * 2) = e[u];
                }
                auto reg1 = [](int p, int Pext, int s) { return s == 0 ? 2 : (p < Pext - 4 ? 0 : (p < Pext - s ? 1 : 2)); };
                region[tw] = shifted ? (reg1(a.ph, P.PH, P.sh) * 9 + reg1(a.pw, P.PW, P.sw) * 3 + reg1(a.pd, P.PD, P.sd)) : 0;
            }
        }
        ptx::fence_proxy_async();
        ptx::named_barrier(1 + wg, 128);
        float s[32];
        ptx::reg_fence(s);
        if (P.fp16) attn_mma_s<true>(s, dq, dk); else attn_mma_s<false>(s, dq, dk);
        ptx::wgmma_wait<0>();
        ptx::reg_fence(s);
        // ---- softmax of rows q0 = frag_row(t, 0) and q0 + 8 over the window's 64 keys (this thread: 16 keys of each)
        float sum[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int q = ptx::frag_row(t, h);
            const int ti = q >> 4, tj = (q >> 2) & 3, tk = q & 3;
            const int myreg = region[q];
            float mx = -INFINITY;
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int c = ptx::frag_col(t, j) + e;
                    const int ji = c >> 4, jj = (c >> 2) & 3, jk = c & 3;
                    float a = s[4 * j + 2 * h + e] * 0.17677669529663687f + tbl[(ti - ji + 3) * 49 + (tj - jj + 3) * 7 + (tk - jk + 3)];
                    if (shifted && region[c] != myreg) a += -100.0f;
                    s[4 * j + 2 * h + e] = a; mx = fmaxf(mx, a);
                }
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            float sm = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float e0 = __expf(s[4 * j + 2 * h] - mx), e1 = __expf(s[4 * j + 2 * h + 1] - mx);
                sm += e0; sm += e1;
                *reinterpret_cast<uint32_t*>(Ps + attn_sw(q, j) + (t & 3) * 4) = pack_act2(e0, e1, P.fp16);
            }
            sm += __shfl_xor_sync(0xffffffffu, sm, 1);
            sm += __shfl_xor_sync(0xffffffffu, sm, 2);
            sum[h] = sm;
        }
        ptx::fence_proxy_async();
        ptx::named_barrier(1 + wg, 128);
        float o[16];
        ptx::reg_fence(o);
        if (P.fp16) attn_mma_o<true>(o, dp, dv); else attn_mma_o<false>(o, dp, dv);
        ptx::wgmma_wait<0>();
        ptx::reg_fence(o);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int q = ptx::frag_row(t, h);
            const AttnTok a = attn_tok(P, w, q);
            if (!a.real) continue;
            const float inv = 1.0f / sum[h];
            __nv_bfloat16* orow = P.out + a.tok * P.ld_out + hc;
#pragma unroll
            for (int j = 0; j < 4; ++j)
                *reinterpret_cast<uint32_t*>(orow + ptx::frag_col(t, j)) = pack_act2(o[4 * j + 2 * h] * inv, o[4 * j + 2 * h + 1] * inv, P.fp16);
        }
        ptx::named_barrier(1 + wg, 128);                   // the operand tiles and regions may be rewritten
    }
}

static inline unsigned grid_for(size_t total, int block) {
    size_t g = (total + block - 1) / block;
    const size_t cap = (size_t)num_sms() * 16;
    return (unsigned)(g < cap ? (g ? g : 1) : cap);
}

}  // namespace nrpn

using namespace nrpn;

extern "C" {
#pragma GCC visibility push(default)

int nrpn_patch_embed_pack(const float* grid, int n, int x, int y, int z, void* out, int act_fp16, nrpn_stream_t stream) {
    if (!grid || !out || n < 1 || x < 4 || y < 4 || z < 4) return NRPN_ERR_INVALID;
    const int H = x / 4, W = y / 4, D = z / 4;
    const size_t total = (size_t)n * H * W * D * 32;
    patch_embed_pack_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(grid, n, x, y, z, H, W, D, reinterpret_cast<__nv_bfloat16*>(out), act_fp16 ? 1 : 0);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

int nrpn_layernorm(const void* in, int ld_in, void* out, int ld_out, long tokens, int c, const float* gamma, const float* beta,
                   float eps, int act_fp16, nrpn_stream_t stream) {
    if (!in || !out || !gamma || !beta || tokens < 1 || c < 1 || ld_in < c || ld_out < c) return NRPN_ERR_INVALID;
    layernorm_kernel<<<(unsigned)ceil_div(tokens, 8L), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(in), ld_in, reinterpret_cast<__nv_bfloat16*>(out), ld_out, tokens, c, gamma, beta, eps, act_fp16 ? 1 : 0);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

int nrpn_patch_merge_ln(const void* in, int ld_in, int n, int h, int w, int d, int c, void* out, const float* gamma, const float* beta,
                        float eps, int act_fp16, nrpn_stream_t stream) {
    if (!in || !out || !gamma || !beta || n < 1 || h < 1 || w < 1 || d < 1 || c < 1 || ld_in < c) return NRPN_ERR_INVALID;
    const long tokens = (long)n * ((h + 1) / 2) * ((w + 1) / 2) * ((d + 1) / 2);
    patch_merge_ln_kernel<<<(unsigned)ceil_div(tokens, 8L), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(in), ld_in, n, h, w, d, c, reinterpret_cast<__nv_bfloat16*>(out), gamma, beta, eps, act_fp16 ? 1 : 0);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

int nrpn_window_attention(const void* qkv, int ld_qkv, void* out, int ld_out, const float* qkv_bias, const float* table, int n, int h,
                          int w, int d, int c, int heads, int shift, int act_fp16, nrpn_stream_t stream) {
    if (!qkv || !out || !qkv_bias || !table || n < 1 || h < 1 || w < 1 || d < 1 || heads < 1 || c != heads * 32) return NRPN_ERR_INVALID;
    if (ld_qkv < 3 * c || ld_out < c || (shift != 0 && shift != 2)) return NRPN_ERR_INVALID;
    // q / k / v segments and output rows are read and written in 16-byte chunks
    if (ld_qkv % 8 != 0 || ld_out % 8 != 0 || reinterpret_cast<uintptr_t>(qkv) % 16 != 0 || reinterpret_cast<uintptr_t>(out) % 16 != 0)
        return NRPN_ERR_INVALID;
    AttnDev P;
    P.qkv = reinterpret_cast<const __nv_bfloat16*>(qkv); P.ld_qkv = ld_qkv; P.out = reinterpret_cast<__nv_bfloat16*>(out); P.ld_out = ld_out;
    P.fp16 = act_fp16 ? 1 : 0;
    P.qkv_bias = qkv_bias; P.table = table; P.n = n; P.H = h; P.W = w; P.D = d; P.C = c; P.heads = heads;
    P.PH = (h + 3) / 4 * 4; P.PW = (w + 3) / 4 * 4; P.PD = (d + 3) / 4 * 4;
    P.sh = (4 >= P.PH) ? 0 : shift; P.sw = (4 >= P.PW) ? 0 : shift; P.sd = (4 >= P.PD) ? 0 : shift;   // no shift along an axis one window wide
    P.nwh = P.PH / 4; P.nww = P.PW / 4; P.nwd = P.PD / 4;
    const long windows = (long)n * P.nwh * P.nww * P.nwd;
    if (windows > 0x7fffffffL || heads > 65535) return NRPN_ERR_UNSUPPORTED;
    static bool attr_set = false;
    if (!attr_set) {
        NRPN_CUDA_TRY(cudaFuncSetAttribute(window_attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnSmem));
        attr_set = true;
    }
    const long pairs = (windows + 1) / 2;
    long gx = (long)num_sms() * 2 / heads;              // 2 resident CTAs per SM in total, each looping over window pairs
    if (gx < 1) gx = 1;
    if (gx > pairs) gx = pairs;
    window_attention_tc_kernel<<<dim3((unsigned)gx, heads), kAttnThreads, kAttnSmem, (cudaStream_t)stream>>>(P, (int)windows);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

#pragma GCC visibility pop
}  // extern "C"
