// Bandwidth-bound helpers around the convolutions (HBM roofline kernels; 16-byte coalesced accesses).
#include "common.cuh"

namespace nrpn {

// fp32 NCDHW grid (N,4,X,Y,Z) -> bf16 (N, X2, Y2, Z2+1, 64), X2 = ceil(X/2) etc.
// Row (i,j,k) holds two 2x2x2 space-to-depth blocks: channels [0,32) = block (i,j,k-1), [32,64) = block (i,j,k);
// inside a block channel = ((rx*2+ry)*2+rz)*4 + c for input voxel (2i+rx, 2j+ry, 2k'+rz), zero outside the grid.
// With this layout the reference's stem Conv3d(4,64,k=7,s=2,p=3) (feature_extractor.py:163) is a stride-1
// implicit GEMM with 4x4x2 taps of K = 64 (see nerf_rpn_b200/engine.py: pack_stem_weight).
// One thread writes one 16-byte chunk (8 channels); 8 consecutive lanes cover one 128-byte row.
// density_to_alpha (datasets.py:165-167, applied by the reference's dataset on the host when --normalize_density is set):
// alpha = clip(1 - exp(-exp(sigma) / 100), 0, 1) on the last channel, fp32 like numpy computes it on a float32 array.
__device__ __forceinline__ float density_to_alpha(float sigma) {
    const float a = 1.0f - expf(-__fdiv_rn(expf(sigma), 100.0f));
    return fminf(fmaxf(a, 0.0f), 1.0f);
}

// Per-chunk pieces of the stem packing.
// stem_chunk: coordinates of 16-byte chunk t of one scene's packed (X2, Y2, Z2+1, 64) rows -- first voxel (x, y, z) of the chunk's
// z pair, and its space-to-depth block index kk along z (-1 / Z2 for the zero rows at either end).
struct StemChunk { int x, y, z, kk; };
__device__ __forceinline__ StemChunk stem_chunk(size_t t, int Y2, int Z2) {
    StemChunk q;
    const int s = (int)(t & 7);
    size_t v = t >> 3;
    const int k = (int)(v % (Z2 + 1)); v /= (Z2 + 1);
    const int j = (int)(v % Y2);
    const int i = (int)(v / Y2);
    const int half = s >> 2, rx = (s >> 1) & 1, ry = s & 1;
    q.kk = k - 1 + half;                            // s2d block index along z
    q.x = 2 * i + rx; q.y = 2 * j + ry; q.z = 2 * q.kk;
    return q;
}

// The voxel pair (x,y,z), (x,y,z+1) of one NCDHW scene: p points at channel 0 of voxel (x,y,z), channel planes `plane` floats apart;
// val = {4 channels of z, 4 channels of z+1} (rz major, c minor); `second`: z+1 lies inside the scene (else those stay 0).
__device__ __forceinline__ void stem_load_ncdhw(const float* __restrict__ p, size_t plane, bool second, int alpha, float (&val)[8]) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        val[c] = p[c * plane];
        if (second) val[4 + c] = p[c * plane + 1];
    }
    if (alpha) { val[3] = density_to_alpha(val[3]); if (second) val[7] = density_to_alpha(val[7]); }
}

// Same pair from a channels-last scene: one 128-bit load per voxel.
__device__ __forceinline__ void stem_load_cl(const float4* __restrict__ p, bool second, int alpha, float4& a, float4& c) {
    a = __ldg(p);
    if (second) c = __ldg(p + 1);
    if (alpha) { a.w = density_to_alpha(a.w); if (second) c.w = density_to_alpha(c.w); }
}

// Same pair from a raw uint8 scene in its on-disk (X,Y,Z,4) order: one 32-bit load per voxel, each byte normalised with the
// correctly rounded fp32 x / 255 that datasets.py:59-61 performs on the host (.float() / 255.0).  No density_to_alpha: uint8 grids
// hold alphas already.
__device__ __forceinline__ void stem_load_u8(const uint32_t* __restrict__ p, bool second, float4& a, float4& c) {
    auto f = [](uint32_t w, int byte) { return __fdiv_rn((float)((w >> (8 * byte)) & 0xFFu), 255.0f); };
    const uint32_t w0 = __ldg(p), w1 = second ? __ldg(p + 1) : 0u;
    a = make_float4(f(w0, 0), f(w0, 1), f(w0, 2), f(w0, 3));
    c = make_float4(f(w1, 0), f(w1, 1), f(w1, 2), f(w1, 3));
}

__device__ __forceinline__ void stem_store(__nv_bfloat16* __restrict__ out, size_t t, float4 a, float4 c, int fp16) {
    const uint32_t h0 = pack_act2(a.x, a.y, fp16), h1 = pack_act2(a.z, a.w, fp16);
    const uint32_t h2 = pack_act2(c.x, c.y, fp16), h3 = pack_act2(c.z, c.w, fp16);
    *reinterpret_cast<uint4*>(out + (t << 3)) = make_uint4(h0, h1, h2, h3);
}

// The stem input of gridDim.y scenes padded to the element-wise maximum extent (X2, Y2, Z2 of that maximum): block row b packs
// scene b through its own pointer, extent and layout; a voxel outside the scene is the reference's zero padding
// (nerf_rpn.py:140-146) in all four channels -- density_to_alpha is applied to real voxels only.  A stacked batch is the case
// where every extent is the same.
struct StemBatch { nrpn_stem_src src[NRPN_STEM_MAX_SCENES]; };

__global__ void pack_stem_kernel(const __grid_constant__ StemBatch B, int X2, int Y2, int Z2, __nv_bfloat16* __restrict__ out, int fp16,
                                 int alpha) {
    const nrpn_stem_src S = B.src[blockIdx.y];         // a copy: the scene's fields sit in uniform registers, read once per block
    const size_t chunks = (size_t)X2 * Y2 * (Z2 + 1) * 8;
    out += blockIdx.y * chunks * 8;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < chunks; t += (size_t)gridDim.x * blockDim.x) {
        const StemChunk q = stem_chunk(t, Y2, Z2);
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f), c = a;
        if (q.kk >= 0 && q.z < S.z && q.x < S.x && q.y < S.y) {
            const size_t vox = ((size_t)q.x * S.y + q.y) * S.z + q.z;
            const bool second = q.z + 1 < S.z;
            if (S.layout == NRPN_STEM_F32_XYZC) {
                stem_load_cl(static_cast<const float4*>(S.grid) + vox, second, alpha, a, c);
            } else if (S.layout == NRPN_STEM_U8_XYZC) {
                stem_load_u8(static_cast<const uint32_t*>(S.grid) + vox, second, a, c);
            } else {
                float val[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) val[e] = 0.f;
                stem_load_ncdhw(static_cast<const float*>(S.grid) + vox, (size_t)S.x * S.y * S.z, second, alpha, val);
                a = make_float4(val[0], val[1], val[2], val[3]); c = make_float4(val[4], val[5], val[6], val[7]);
            }
        }
        stem_store(out, t, a, c, fp16);
    }
}

// F.max_pool3d(k=3, s=2, p=1) on channels-last bf16; one thread per (output voxel, 8 channels).
__global__ void maxpool_k3s2_kernel(const __nv_bfloat16* __restrict__ in, int n, int X, int Y, int Z, int C, int Xo, int Yo,
                                    int Zo, __nv_bfloat16* __restrict__ out, int fp16) {
    const int cg = C >> 3;
    const size_t total = (size_t)n * Xo * Yo * Zo * cg;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
        const int g = (int)(t % cg); size_t v = t / cg;
        const int k = (int)(v % Zo); v /= Zo;
        const int j = (int)(v % Yo); v /= Yo;
        const int i = (int)(v % Xo); const int b = (int)(v / Xo);
        float m[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) m[q] = -INFINITY;
        // out-of-range taps are clamped onto the border voxel instead of skipped: a maximum ignores duplicates, and the 27
        // loads become branch-free and independent (all in flight at once)
        const __nv_bfloat16* base = in + (size_t)b * X * Y * Z * C + g * 8;
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) {
            const int x = min(max(2 * i + dx, 0), X - 1);
#pragma unroll
            for (int dy = -1; dy <= 1; ++dy) {
                const int y = min(max(2 * j + dy, 0), Y - 1);
                uint4 raw[3];
#pragma unroll
                for (int dz = -1; dz <= 1; ++dz) {
                    const int z = min(max(2 * k + dz, 0), Z - 1);
                    raw[dz + 1] = __ldg(reinterpret_cast<const uint4*>(base + (((size_t)x * Y + y) * Z + z) * C));
                }
#pragma unroll
                for (int dz = 0; dz < 3; ++dz) {
                    const uint32_t* h = reinterpret_cast<const uint32_t*>(&raw[dz]);
#pragma unroll
                    for (int q = 0; q < 4; ++q) { const float2 f = unpack_act2(h[q], fp16); m[2 * q] = fmaxf(m[2 * q], f.x); m[2 * q + 1] = fmaxf(m[2 * q + 1], f.y); }
                }
            }
        }
        uint32_t o[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) o[q] = pack_act2(m[2 * q], m[2 * q + 1], fp16);
        *reinterpret_cast<uint4*>(out + ((((size_t)b * Xo + i) * Yo + j) * Zo + k) * C + g * 8) = make_uint4(o[0], o[1], o[2], o[3]);
    }
}

// nn.MaxPool3d(kernel 2, stride 2, ceil_mode=True) on channels-last bf16 (VGG stages, feature_extractor.py:347):
// output extent ceil(in/2); the last window is clipped at the border (maxpool_k2s2_window, common.cuh).
__global__ void maxpool_k2s2_ceil_kernel(const __nv_bfloat16* __restrict__ in, int n, int X, int Y, int Z, int C, int Xo, int Yo,
                                         int Zo, __nv_bfloat16* __restrict__ out, int fp16) {
    const int cg = C >> 3;
    const size_t total = (size_t)n * Xo * Yo * Zo * cg;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
        const int g = (int)(t % cg); size_t v = t / cg;
        const int k = (int)(v % Zo); v /= Zo;
        const int j = (int)(v % Yo); v /= Yo;
        const int i = (int)(v % Xo); const int b = (int)(v / Xo);
        float m[8]; int pos[8];
        maxpool_k2s2_window(in, X, Y, Z, C, b, i, j, k, g, fp16, m, pos);
        uint32_t o[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) o[q] = pack_act2(m[2 * q], m[2 * q + 1], fp16);
        *reinterpret_cast<uint4*>(out + ((((size_t)b * Xo + i) * Yo + j) * Zo + k) * C + g * 8) = make_uint4(o[0], o[1], o[2], o[3]);
    }
}

// Stride-1 stem packing (VGG_FPN for grids < 160: Conv3d(4,64,k=7,s=1,p=3), feature_extractor.py:341):
// fp32 NCDHW (N,4,X,Y,Z) -> bf16 (N, X, Y+1, Z, 64).  Row (x, yp, z) holds, for the two input rows y = yp-1 and yp, the seven
// z-neighbours z-3..z+3 of all 4 channels: channel = ((yy*7 + zz)*4 + c), 56 used + 8 zero.  The 7^3 conv becomes a
// 7 (dx) x 4 (y pairs) tap implicit GEMM with K = 64 per tap (packing.pack_stem_s1_weight).
__global__ void pack_stem_s1_kernel(const float* __restrict__ grid, int n, int X, int Y, int Z, __nv_bfloat16* __restrict__ out, int fp16) {
    const size_t total = (size_t)n * X * (Y + 1) * Z * 8;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
        const int s = (int)(t & 7);
        size_t v = t >> 3;
        const int z = (int)(v % Z); v /= Z;
        const int yp = (int)(v % (Y + 1)); v /= (Y + 1);
        const int x = (int)(v % X); const int b = (int)(v / X);
        float val[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int ch = s * 8 + e;
            float f = 0.f;
            if (ch < 56) {
                const int c = ch & 3, zz = (ch >> 2) % 7, yy = (ch >> 2) / 7;
                const int y = yp - 1 + yy, zi = z + zz - 3;
                if (y >= 0 && y < Y && zi >= 0 && zi < Z) f = grid[((((size_t)b * 4 + c) * X + x) * Y + y) * Z + zi];
            }
            val[e] = f;
        }
        uint32_t h[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) h[q] = pack_act2(val[2 * q], val[2 * q + 1], fp16);
        *reinterpret_cast<uint4*>(out + (t << 3)) = make_uint4(h[0], h[1], h[2], h[3]);
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

int nrpn_pack_stem_input(const nrpn_stem_src* src, int n, void* packed, int act_fp16, int density_to_alpha, nrpn_stream_t stream) {
    if (!src || !packed || n < 1) return NRPN_ERR_INVALID;
    int x = 0, y = 0, z = 0;
    for (int i = 0; i < n; ++i) {
        const nrpn_stem_src& S = src[i];
        if (!S.grid || S.x < 1 || S.y < 1 || S.z < 1) return NRPN_ERR_INVALID;
        const uintptr_t addr = reinterpret_cast<uintptr_t>(S.grid);
        switch (S.layout) {
            case NRPN_STEM_F32_NCDHW: break;
            case NRPN_STEM_F32_XYZC: if (addr % 16 != 0) return NRPN_ERR_INVALID; break;
            case NRPN_STEM_U8_XYZC: if (addr % 4 != 0 || density_to_alpha) return NRPN_ERR_INVALID; break;
            default: return NRPN_ERR_INVALID;
        }
        x = S.x > x ? S.x : x; y = S.y > y ? S.y : y; z = S.z > z ? S.z : z;
    }
    const int X2 = (x + 1) / 2, Y2 = (y + 1) / 2, Z2 = (z + 1) / 2;
    const size_t chunks_per_scene = (size_t)X2 * Y2 * (Z2 + 1) * 8;
    // one launch per NRPN_STEM_MAX_SCENES scenes (the size of the kernel's parameter table), each writing its slice of the padded batch
    for (int i0 = 0; i0 < n; i0 += NRPN_STEM_MAX_SCENES) {
        const int m = n - i0 < NRPN_STEM_MAX_SCENES ? n - i0 : NRPN_STEM_MAX_SCENES;
        StemBatch B;
        for (int i = 0; i < m; ++i) B.src[i] = src[i0 + i];
        const dim3 grid((grid_for(m * chunks_per_scene, 256) + m - 1) / m, m);
        pack_stem_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(B, X2, Y2, Z2, reinterpret_cast<__nv_bfloat16*>(packed) + i0 * chunks_per_scene * 8,
                                                                 act_fp16 ? 1 : 0, density_to_alpha ? 1 : 0);
        NRPN_LAUNCH_CHECK();
    }
    return NRPN_OK;
}

int nrpn_maxpool3d_k3s2(const void* in, int n, int x, int y, int z, int c, void* out, int act_fp16, nrpn_stream_t stream) {
    if (!in || !out || n < 1 || x < 1 || y < 1 || z < 1 || c < 8 || c % 8 != 0) return NRPN_ERR_INVALID;
    const int Xo = (x - 1) / 2 + 1, Yo = (y - 1) / 2 + 1, Zo = (z - 1) / 2 + 1;
    const size_t total = (size_t)n * Xo * Yo * Zo * (c / 8);
    maxpool_k3s2_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(in), n, x, y, z, c, Xo, Yo, Zo, reinterpret_cast<__nv_bfloat16*>(out), act_fp16 ? 1 : 0);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

int nrpn_maxpool3d_k2s2_ceil(const void* in, int n, int x, int y, int z, int c, void* out, int act_fp16, nrpn_stream_t stream) {
    if (!in || !out || n < 1 || x < 1 || y < 1 || z < 1 || c < 8 || c % 8 != 0) return NRPN_ERR_INVALID;
    const int Xo = (x + 1) / 2, Yo = (y + 1) / 2, Zo = (z + 1) / 2;
    const size_t total = (size_t)n * Xo * Yo * Zo * (c / 8);
    maxpool_k2s2_ceil_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(in), n, x, y, z, c, Xo, Yo, Zo, reinterpret_cast<__nv_bfloat16*>(out), act_fp16 ? 1 : 0);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

int nrpn_pack_stem_input_s1(const float* grid, int n, int x, int y, int z, void* packed, int act_fp16, nrpn_stream_t stream) {
    if (!grid || !packed || n < 1 || x < 1 || y < 1 || z < 1) return NRPN_ERR_INVALID;
    const size_t total = (size_t)n * x * (y + 1) * z * 8;
    pack_stem_s1_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(grid, n, x, y, z, reinterpret_cast<__nv_bfloat16*>(packed), act_fp16 ? 1 : 0);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

int nrpn_version(void) { return 105; }

const char* nrpn_status_string(int status) {
    switch (status) {
        case NRPN_OK: return "ok";
        case NRPN_ERR_INVALID: return "invalid argument";
        case NRPN_ERR_UNSUPPORTED: return "unsupported shape";
        case NRPN_ERR_WORKSPACE: return "workspace too small";
        case NRPN_ERR_CUDA: return "CUDA error";
        case NRPN_ERR_NO_DEVICE: return "no sm_90 device / driver entry point";
        default: return "unknown status";
    }
}

int nrpn_last_cuda_error(void) { return g_last_cuda_error; }

unsigned long long nrpn_launch_count(void) { return g_launch_count.load(); }

#pragma GCC visibility pop
}  // extern "C"
