// Box-overlap entry points and device-resident greedy NMS.
//   replaces: utils.py:215-265 (nms / batched_nms: Python while-loop, one host sync + ~40 ATen kernels +
//             the native vertex sort per kept box), utils.py:387-415 (box_iou_3d), cuda_op/sort_vert_kernel.cu.
// Design: sort once by (group, score desc, index) with an in-kernel bitonic network, build the 64-bit
// suppression bit-matrix only for same-group upper-triangle tiles (one thread per row, 64 columns per word,
// exact-zero culling by bounding circle / z range), resolve each group with one CTA that walks the matrix
// 64 rows at a time (warp-shuffle resolve of the diagonal word, coalesced OR of the kept rows), then sort
// the survivors by score.  No host round trips; everything is stream-ordered.  Beyond a scene's proposals: chunked kept-list scan (groups above
// 3 072 boxes) and, from 12 288 boxes, the cell-list path of nms_cells.cuh (levels: cross / adjacency / dependency rounds; reads a counter back per
// batch of rounds, so it is skipped under stream capture).  Every path decides a pair with the exact IoU of the sequential loop; what may skip the
// polygon clip is controlled by nrpn_set_nms_cull_mode (default: exact-zero tests only -> the keep set is provably the reference's).
namespace nrpn { static __device__ int g_iou_mode = 3; }      // see box_iou.cuh: which build of the reference chain is reproduced
namespace nrpn { static __device__ int g_lens_cull = 0; }     // footprint-lens cull, bit 1 of the NMS cull mode
#define NRPN_IOU_MODE (::nrpn::g_iou_mode)
#define NRPN_LENS_CULL (::nrpn::g_lens_cull)
#include "box_iou.cuh"
#include "nms_internal.cuh"

namespace nrpn {

thread_local int g_last_cuda_error = 0;
static std::atomic<int> g_nms_cull_mode{[] { const char* e = getenv("NRPN_NMS_CULL_MODE"); return e ? atoi(e) & 3 : 0; }()};
std::atomic<unsigned long long> g_launch_count{0};

// ---------------------------------------------------------------------------------------------- IoU
__global__ void iou_pairs_kernel(const float* __restrict__ a, const float* __restrict__ b, int n, int box_dim,
                                 float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (box_dim == 7) {
        ObbPrep pa, pb;
        obb_prepare(a + (size_t)i * 7, pa);
        obb_prepare(b + (size_t)i * 7, pb);
        out[i] = iou3d_obb(pa, pb, true);
    } else {
        out[i] = iou3d_aabb(a + (size_t)i * 6, b + (size_t)i * 6);
    }
}

// cal_iou_3d(verbose=True) (oriented_iou_loss.py:82-107): IoU, both corner sets, z_range and the 3-D union of every pair
__global__ void iou_pairs_verbose_kernel(const float* __restrict__ a, const float* __restrict__ b, int n, float* __restrict__ iou,
                                         float* __restrict__ corners1, float* __restrict__ corners2, float* __restrict__ z_range,
                                         float* __restrict__ u3d) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ObbPrep pa, pb;
    obb_prepare(a + (size_t)i * 7, pa);
    obb_prepare(b + (size_t)i * 7, pb);
    float zo = __fsub_rn(fminf(pa.zmax, pb.zmax), fmaxf(pa.zmin, pb.zmin));
    if (!(zo >= 0.0f)) zo = (zo != zo) ? zo : 0.0f;
    const float inter = rect_inter_area(pa.c, pb.c);
    const float u = __fsub_rn(__fadd_rn(pa.area, pb.area), inter);
    const float i3 = __fmul_rn(__fmul_rn(__fdiv_rn(inter, u), u), zo);
    const float u3 = __fsub_rn(__fadd_rn(pa.vol, pb.vol), i3);
    iou[i] = __fdiv_rn(i3, u3);
    u3d[i] = u3;
    float zr = __fsub_rn(fmaxf(pa.zmax, pb.zmax), fminf(pa.zmin, pb.zmin));
    if (!(zr >= 0.0f)) zr = (zr != zr) ? zr : 0.0f;
    z_range[i] = zr;
#pragma unroll
    for (int k = 0; k < 8; ++k) { corners1[(size_t)i * 8 + k] = pa.c[k]; corners2[(size_t)i * 8 + k] = pb.c[k]; }
}

// Intersection volume of two yaw-rotated boxes in fp64 (Sutherland-Hodgman clip of A's footprint by B's four half-planes x z overlap):
// the smooth function whose derivative the backward pass needs.
__device__ double inter_volume_d(const double* A, const double* B) {
    double px[12], py[12], qx[12], qy[12];
    int np = 4;
    const double sx[4] = {0.5, -0.5, -0.5, 0.5}, sy[4] = {0.5, 0.5, -0.5, -0.5};
    const double ca = cos(A[6]), sa = sin(A[6]), cb = cos(B[6]), sb = sin(B[6]);
    double bx[4], by[4];
    for (int k = 0; k < 4; ++k) {
        px[k] = A[0] + sx[k] * A[3] * ca - sy[k] * A[4] * sa; py[k] = A[1] + sx[k] * A[3] * sa + sy[k] * A[4] * ca;
        bx[k] = B[0] + sx[k] * B[3] * cb - sy[k] * B[4] * sb; by[k] = B[1] + sx[k] * B[3] * sb + sy[k] * B[4] * cb;
    }
    for (int e = 0; e < 4 && np > 0; ++e) {                     // clip against edge e of B (counter-clockwise: inside = left)
        const double ex = bx[(e + 1) & 3] - bx[e], ey = by[(e + 1) & 3] - by[e];
        int nq = 0;
        for (int k = 0; k < np; ++k) {
            const int k2 = k + 1 == np ? 0 : k + 1;
            const double d1 = ex * (py[k] - by[e]) - ey * (px[k] - bx[e]);
            const double d2 = ex * (py[k2] - by[e]) - ey * (px[k2] - bx[e]);
            if (d1 >= 0.0) { qx[nq] = px[k]; qy[nq] = py[k]; ++nq; }
            if ((d1 >= 0.0) != (d2 >= 0.0)) {
                const double t = d1 / (d1 - d2);
                qx[nq] = px[k] + t * (px[k2] - px[k]); qy[nq] = py[k] + t * (py[k2] - py[k]); ++nq;
            }
        }
        np = nq;
        for (int k = 0; k < np; ++k) { px[k] = qx[k]; py[k] = qy[k]; }
    }
    double area = 0.0;
    for (int k = 0; k < np; ++k) { const int k2 = k + 1 == np ? 0 : k + 1; area += px[k] * py[k2] - py[k] * px[k2]; }
    area = 0.5 * fabs(area);
    double zo = fmin(A[2] + 0.5 * A[5], B[2] + 0.5 * B[5]) - fmax(A[2] - 0.5 * A[5], B[2] - 0.5 * B[5]);
    if (!(zo > 0.0)) zo = 0.0;
    return area * zo;
}

// Backward of (iou, u3d) = cal_iou_3d(a, b, verbose) w.r.t. both boxes: with I the intersection volume, U = V1 + V2 - I, iou = I / U:
//   dL = [g_iou (U + I) / U^2 - g_u] dI + [g_u - g_iou I / U^2] d(V1 + V2);   dI by central differences of inter_volume_d in fp64
// (I is piecewise smooth in the 14 parameters; step 1e-5 of the pair's scale: truncation ~1e-10, round-off ~1e-11 relative).
// One thread per (pair, parameter).
__global__ void iou_pairs_grad_kernel(const float* __restrict__ a, const float* __restrict__ b, int n, const float* __restrict__ g_iou,
                                      const float* __restrict__ g_u, float* __restrict__ ga, float* __restrict__ gb) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * 14) return;
    const int i = t / 14, k = t % 14;
    double A[7], B[7];
    for (int j = 0; j < 7; ++j) { A[j] = (double)a[(size_t)i * 7 + j]; B[j] = (double)b[(size_t)i * 7 + j]; }
    const double I = inter_volume_d(A, B);
    const double V1 = A[3] * A[4] * A[5], V2 = B[3] * B[4] * B[5], U = V1 + V2 - I;
    const double gi = g_iou ? (double)g_iou[i] : 0.0, gu = g_u ? (double)g_u[i] : 0.0;
    const double cI = gi * (U + I) / (U * U) - gu, cV = gu - gi * I / (U * U);
    double scale = fmax(fmax(fabs(A[3]), fabs(A[4])), fmax(fabs(B[3]), fabs(B[4])));
    scale = fmax(scale, fmax(fabs(A[5]), fabs(B[5])));
    const double h = 1e-5 * (scale > 0.0 ? scale : 1.0);
    double* P = k < 7 ? A : B;
    const int j = k < 7 ? k : k - 7;
    const double keep = P[j];
    const double hh = j == 6 ? 1e-6 : h;
    P[j] = keep + hh; const double Ip = inter_volume_d(A, B);
    P[j] = keep - hh; const double Im = inter_volume_d(A, B);
    P[j] = keep;
    double dV = 0.0;
    if (j == 3) dV = P[4] * P[5]; else if (j == 4) dV = P[3] * P[5]; else if (j == 5) dV = P[3] * P[4];
    const double gval = cI * (Ip - Im) / (2.0 * hh) + cV * dV;
    (k < 7 ? ga : gb)[(size_t)i * 7 + j] = (float)gval;
}

// tile: 8 rows (a) x 32 cols (b) per 256-thread CTA; box preparation (fp64 sin/cos) once per box per tile.
__global__ void iou_matrix_kernel(const float* __restrict__ a, int n, const float* __restrict__ b, int m, int box_dim,
                                  float* __restrict__ out) {
    __shared__ ObbPrep sa[8];
    __shared__ ObbPrep sb[32];
    __shared__ float ra[8][6];
    __shared__ float rb[32][6];
    const int r0 = blockIdx.y * 8, c0 = blockIdx.x * 32;
    const int t = threadIdx.x;
    if (box_dim == 7) {
        if (t < 8 && r0 + t < n) obb_prepare(a + (size_t)(r0 + t) * 7, sa[t]);
        if (t >= 32 && t < 64 && c0 + (t - 32) < m) obb_prepare(b + (size_t)(c0 + t - 32) * 7, sb[t - 32]);
    } else {
        if (t < 48) { const int r = t / 6, k = t % 6; if (r0 + r < n) ra[r][k] = a[(size_t)(r0 + r) * 6 + k]; }
        if (t >= 64 && t < 64 + 192) { const int c = (t - 64) / 6, k = (t - 64) % 6; if (c0 + c < m) rb[c][k] = b[(size_t)(c0 + c) * 6 + k]; }
    }
    __syncthreads();
    const int r = t / 32, c = t % 32;
    if (r0 + r >= n || c0 + c >= m) return;
    float v;
    if (box_dim == 7) v = iou3d_obb(sa[r], sb[c], true);
    else v = iou3d_aabb(ra[r], rb[c]);
    out[(size_t)(r0 + r) * m + c0 + c] = v;
}

// ------------------------------------------------------------------------------- sort_vertices (K1)
// One thread per polygon, same contract as sort_vertices_forward (sort_vert.cpp:6-34); restates the
// selection sort of sort_vert_kernel.cu:42-134 with the polygon held in registers/local memory.
__global__ void sort_vertices_kernel(const float* __restrict__ vertices, const uint8_t* __restrict__ mask,
                                     const int32_t* __restrict__ num_valid, long total, int m, int32_t* __restrict__ idx) {
    const long p = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= total) return;
    float x[32], y[32], q[32];
    uint32_t mk = 0;
    for (int k = 0; k < m; ++k) {
        x[k] = vertices[(p * m + k) * 2];
        y[k] = vertices[(p * m + k) * 2 + 1];
        q[k] = pseudo_angle(x[k], y[k]);
        if (mask[p * m + k]) mk |= 1u << k;
    }
    const int nv = num_valid[p];
    int pad = 0;
    for (int j = 8; j < m; ++j) if (!((mk >> j) & 1u)) { pad = j; break; }
    int32_t* o = idx + p * 9;
    if (nv < 3) { for (int j = 0; j < 9; ++j) o[j] = pad; return; }
    int tk[9];
    int first = 0, prev = 0;
    for (int j = 0; j < nv; ++j) {
        float bx = 1.0f, by = -eps_f(), bq = 1.0f;
        int take = 0;
        for (int k = 0; k < m; ++k) {
            if (!((mk >> k) & 1u)) continue;
            bool ok = vert_less(x[k], y[k], q[k], bx, by, bq);
            if (ok && j > 0) ok = vert_less(x[prev], y[prev], q[prev], x[k], y[k], q[k]);
            if (ok) { bx = x[k]; by = y[k]; bq = q[k]; take = k; }
        }
        if (j == 0) first = take;
        if (j < 9) tk[j] = take;
        prev = take;
    }
    for (int j = 0; j < 9; ++j) o[j] = pad;
    for (int j = 0; j < nv && j < 9; ++j) o[j] = tk[j];
    if (nv < 9) o[nv] = first;
    if (nv == 8) {
        int counter = 0;
        for (int j = 0; j < 4; ++j) for (int k = 4; k < 8; ++k) counter += (tk[k] == tk[j]) ? 1 : 0;
        if (counter == 4) { o[4] = tk[0]; for (int j = 5; j < 9; ++j) o[j] = pad; }
    }
}

// ------------------------------------------------------------------------------------ bitonic sort
constexpr int kSortTile = 8192;       // elements sorted inside one CTA's shared memory (64 KB)
constexpr int kSortThreads = 1024;

__device__ __forceinline__ void cmp_swap(unsigned long long& a, unsigned long long& b, bool asc) {
    if ((a > b) == asc) { const unsigned long long t = a; a = b; b = t; }
}

// All stages with partner distance < tile, for merge sizes k in [k_lo, k_hi].
__global__ void __launch_bounds__(kSortThreads) bitonic_local_kernel(unsigned long long* __restrict__ keys, int n_pad,
                                                                    int tile, int k_lo, int k_hi) {
    extern __shared__ unsigned long long sk[];
    const int base = blockIdx.x * tile;
    for (int i = threadIdx.x; i < tile; i += blockDim.x) sk[i] = keys[base + i];
    __syncthreads();
    for (int k = k_lo; k <= k_hi; k <<= 1) {
        int j0 = k >> 1; if (j0 >= tile) j0 = tile >> 1;
        for (int j = j0; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < (tile >> 1); t += blockDim.x) {
                const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));   // index with bit j cleared
                const bool asc = (((base + i) & k) == 0);
                cmp_swap(sk[i], sk[i | j], asc);
            }
            __syncthreads();
        }
    }
    for (int i = threadIdx.x; i < tile; i += blockDim.x) keys[base + i] = sk[i];
}

__global__ void bitonic_global_kernel(unsigned long long* __restrict__ keys, int n_pad, int k, int j) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (n_pad >> 1)) return;
    const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
    const bool asc = ((i & k) == 0);
    unsigned long long a = keys[i], b = keys[i | j];
    if ((a > b) == asc) { keys[i] = b; keys[i | j] = a; }
}

int bitonic_sort_u64(unsigned long long* keys, int n_pad, cudaStream_t st) {
    static bool attr_set = false;
    if (!attr_set) {
        NRPN_CUDA_TRY(cudaFuncSetAttribute(bitonic_local_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSortTile * 8));
        attr_set = true;
    }
    const int tile = n_pad < kSortTile ? n_pad : kSortTile;
    const int blocks = n_pad / tile;
    bitonic_local_kernel<<<blocks, kSortThreads, tile * 8, st>>>(keys, n_pad, tile, 2, tile);
    NRPN_LAUNCH_CHECK();
    for (int k = tile << 1; k <= n_pad; k <<= 1) {
        for (int j = k >> 1; j >= tile; j >>= 1) {
            bitonic_global_kernel<<<ceil_div(n_pad >> 1, 256), 256, 0, st>>>(keys, n_pad, k, j);
            NRPN_LAUNCH_CHECK();
        }
        bitonic_local_kernel<<<blocks, kSortThreads, tile * 8, st>>>(keys, n_pad, tile, k, k);
        NRPN_LAUNCH_CHECK();
    }
    return NRPN_OK;
}

// ---------------------------------------------------------------------------------------------- NMS
static inline int next_pow2(int v) { int p = 1; while (p < v) p <<= 1; return p; }

constexpr int kNmsMatrixMax = 32768;     // capacity of the full bit-matrix path (n x n/64 words); see nms_use_matrix()
constexpr int kNmsMaxBoxes = 1 << 21;       // chunked path beyond (index field of the sort key is 24 bits)
constexpr int kChunk = 4096;                // largest chunk of the chunked path (64 words)
constexpr int kNmsDirectMax = 3072;         // the full matrix (all same-group pairs) is only built up to here

// Greedy NMS needs IoU(i, j) only for KEPT i; the full matrix evaluates every same-group pair.  Beyond a few thousand
// boxes the chunked path (test each chunk against the kept list, then resolve the chunk's own small matrix) does far
// fewer polygon clips whenever suppression is heavy (FCOS: ~10 000 candidates in one group, a few hundred survivors).
// `max_group` = the caller's upper bound on the size of one group (n when unknown): the matrix only evaluates same-group tiles.
static inline bool nms_use_matrix(int n, int max_group) { return n <= kNmsMatrixMax && max_group <= kNmsDirectMax; }
static inline int nms_chunk_size(int n) { return n <= 65536 ? 1024 : kChunk; }
constexpr int kPrepFloats = 16;

// ---- binned chunked path ------------------------------------------------------------------------------------------------------
// With n in the hundreds of thousands the chunk-against-kept-list scan is O(n * kept): 1 M boxes spent 3.7 s in it.  Whether box j
// can be suppressed by kept box k is decided by two necessary conditions that can be INDEXED: (a) their volumes are within a factor
// 1 / thr_m of each other (IoU <= min V / max V), (b) their bounding circles and z ranges intersect.  Kept boxes are therefore filed in
// a uniform grid per volume class -- class width log2(1 / thr_m), so partners sit in the same or an adjacent class; cell size >= the
// class's largest diameter / depth -- and a box only visits the cells its circle and z range can reach in its three classes.
// Every candidate still goes through the same cull + exact polygon clip: the keep set is the sequential greedy loop's, bit for bit.
constexpr int kBinMinBoxes = 65536;
constexpr int kCellMinBoxes = 12288;     // cell-list path (nms_cells.cuh) from here (above the 4 x 2 500 boxes of a scene's proposals, whose NMS runs
                                         // inside the captured launch sequence); it shares the grid / box_cell buffers below
constexpr int kRatioCullMinBoxes = 16384; // opt-in geometric culls (nrpn_set_nms_cull_mode) never apply below this
static int cell_min_boxes() {            // NRPN_NMS_CELLS_MIN: where the cell-list path takes over (tuning runs); the ratio culls keep their 16 384 floor
    static const int v = [] { const char* e = getenv("NRPN_NMS_CELLS_MIN"); const int k = e ? atoi(e) : kCellMinBoxes; return k < 1024 ? 1024 : k; }();
    return v;
}
constexpr int kBinClasses = 16;
constexpr int kBinMaxXY = 32, kBinMaxZ = 16;
constexpr int kBinCellsPerClass = kBinMaxXY * kBinMaxXY * kBinMaxZ;
constexpr int kBinCells = kBinClasses * kBinCellsPerClass + 1;      // + one cell for boxes the culls cannot reason about (visited by everyone)
constexpr int kBinStatWords = 8 + 2 * kBinClasses;

struct BinGrid {
    float x0, y0, z0, lv0, inv_lw;       // origin of the box centres, log2-volume origin, 1 / class width
    int n_cls;
    float S[kBinClasses], Sz[kBinClasses], rmax[kBinClasses], dmax[kBinClasses];
    int nx[kBinClasses], ny[kBinClasses], nz[kBinClasses];
};

struct NmsWs {
    unsigned long long* keys;     // n_pad
    unsigned long long* keys2;    // n_pad
    float* prep;                  // n * 16
    int* sgroup;                  // n
    int* seg;                     // 512 (start[256], end[256])
    unsigned long long* keepbits; // W
    unsigned long long* mask;     // n * W (matrix path) or kChunk * 64 (chunked path)
    unsigned long long* removed0; // 64 words: suppression by earlier chunks (chunked path)
    int* kept_pos;                // n (chunked path)
    int* state;                   // [0] kept count, [1..256] first kept index per group
    // binned chunked path (n >= kBinMinBoxes): kept boxes filed by (volume class, x, y, z) cell
    struct BinGrid* grid;         // grid parameters (device)
    unsigned* bstats;             // reduction scratch of the grid (ordered-uint min / max)
    int* box_cell;                // n: cell of every box
    int* cell_start;              // kBinCells + 1: exclusive scan of the per-cell box counts (capacity of the cell's segment)
    int* cell_fill;               // kBinCells: kept boxes filed so far
    float4* cell_recs;            // n x 3 float4: per kept box {cull record (8 floats), position, group, -, -}, cell by cell
    size_t total;
};

static NmsWs nms_layout(void* base, int n) {
    NmsWs w;
    const int n_pad = next_pow2(n < 2 ? 2 : n);
    const int W = ceil_div(n, 64);
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
    char* b = (char*)base;
    w.keys = (unsigned long long*)(b + take((size_t)n_pad * 8));
    w.keys2 = (unsigned long long*)(b + take((size_t)n_pad * 8));
    w.prep = (float*)(b + take((size_t)n * kPrepFloats * 4));
    w.sgroup = (int*)(b + take((size_t)n * 4));
    w.seg = (int*)(b + take(512 * 4));
    w.keepbits = (unsigned long long*)(b + take((size_t)W * 8));
    const bool chunked = n > kNmsMatrixMax;                 // below that either path may be chosen at run time
    w.mask = (unsigned long long*)(b + take(chunked ? (size_t)kChunk * 64 * 8 : (size_t)n * W * 8));
    w.removed0 = (unsigned long long*)(b + take(64 * 8));
    w.kept_pos = (int*)(b + take((size_t)n * 4));
    w.state = (int*)(b + take(258 * 4));          // [0] kept count, [1..256] per-group starts, [257] kept boxes already filed in the grid
    const bool binned = n >= (cell_min_boxes() < kBinMinBoxes ? cell_min_boxes() : kBinMinBoxes);
    w.grid = (BinGrid*)(b + take(sizeof(BinGrid)));
    w.bstats = (unsigned*)(b + take(kBinStatWords * 4));
    w.box_cell = (int*)(b + take(binned ? (size_t)n * 4 : 4));
    w.cell_start = (int*)(b + take(binned ? (size_t)(kBinCells + 1) * 4 : 4));
    w.cell_fill = (int*)(b + take(binned ? (size_t)kBinCells * 4 : 4));
    w.cell_recs = (float4*)(b + take(binned ? (size_t)n * 48 : 16));
    w.total = off;
    return w;
}

__global__ void nms_keys_kernel(const float* __restrict__ scores, const int32_t* __restrict__ group, int n, int n_pad,
                                unsigned long long* __restrict__ keys) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_pad) return;
    unsigned long long k = ~0ull;
    if (i < n) {
        const unsigned long long g = group ? (unsigned long long)(group[i] & 0xFF) : 0ull;
        const unsigned long long s = (unsigned long long)(~float_to_ordered(scores[i]));
        k = (g << 56) | (s << 24) | (unsigned long long)i;
    }
    keys[i] = k;
}

__global__ void nms_prep_kernel(const unsigned long long* __restrict__ keys, const float* __restrict__ boxes, int box_dim,
                                int n, float* __restrict__ prep, int* __restrict__ sgroup, int* __restrict__ seg,
                                const int32_t* __restrict__ group_src = nullptr) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const unsigned long long k = keys[p];
    const int idx = (int)(k & 0xFFFFFFull);
    const int g = group_src ? (int)(group_src[idx] & 0xFF) : (int)(k >> 56);     // keys sorted by score alone carry no group byte
    sgroup[p] = g;
    if (p == 0 || (int)(keys[p - 1] >> 56) != g) seg[g] = p;
    if (p == n - 1 || (int)(keys[p + 1] >> 56) != g) seg[256 + g] = p + 1;
    float* o = prep + (size_t)p * kPrepFloats;
    if (box_dim == 7) {
        ObbPrep pp;
        obb_prepare(boxes + (size_t)idx * 7, pp);
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = pp.c[i];
        o[8] = pp.area; o[9] = pp.vol; o[10] = pp.zmin; o[11] = pp.zmax; o[12] = pp.cx; o[13] = pp.cy; o[14] = pp.rad;
        o[15] = __int_as_float(pp.cullable);
    } else {
        float b[6];
#pragma unroll
        for (int i = 0; i < 6; ++i) { b[i] = boxes[(size_t)idx * 6 + i]; o[i] = b[i]; }
        // cull record of an axis-aligned box (binned path only): volume, z range, bounding circle of the footprint
        const float w = b[3] - b[0], h = b[4] - b[1], d = b[5] - b[2];
        bool fin = true;
#pragma unroll
        for (int i = 0; i < 6; ++i) fin = fin && isfinite(b[i]);
        o[6] = 0.f; o[7] = 0.f;
        o[8] = w * h; o[9] = w * h * d; o[10] = b[2]; o[11] = b[5]; o[12] = 0.5f * (b[0] + b[3]); o[13] = 0.5f * (b[1] + b[4]);
        o[14] = 0.5f * sqrtf(w * w + h * h) * 1.001f + 1e-3f;
        o[15] = __int_as_float((fin && w > 0.f && h > 0.f && d > 0.f) ? 1 : 0);
    }
}

__device__ __forceinline__ void load_prep(const float* __restrict__ s, ObbPrep& p) {
#pragma unroll
    for (int i = 0; i < 8; ++i) p.c[i] = s[i];
    p.area = s[8]; p.vol = s[9]; p.zmin = s[10]; p.zmax = s[11]; p.cx = s[12]; p.cy = s[13]; p.rad = s[14];
    p.cullable = __float_as_int(s[15]);
}

// grid (W, W); CTA (cb, rb) with cb >= rb fills mask[rows of chunk rb][word cb]: a 64 x 64 tile of pairs, 256 threads
// (64-thread CTAs left the 136-tile matrices of the chunked path with 2 warps per SM: 0.8 ms per 1024-box chunk under ncu).
// Oriented boxes take two phases so that the expensive polygon clip never runs on a half-empty warp:
//   1. thread <-> row: the cheap tests (column right of the row, same group, not provably zero) give a 64-bit candidate
//      word per row; the candidates of the whole tile are compacted into a list in shared memory;
//   2. thread <-> list entry: full IoU of (row, column) with both records read from shared memory; hits are OR-ed into
//      the row's word with a shared-memory atomic.
// (One row per thread with the test inline ran the full clip whenever ANY of the 32 rows of a warp needed it:
//  measured 0.4 ns per pair regardless of how many pairs overlapped.)
constexpr int kMaskThreads = 256;

__global__ void __launch_bounds__(kMaskThreads) nms_mask_kernel(const float* __restrict__ prep, const int* __restrict__ sgroup, int n,
                                                                int W, int box_dim, float thr, float thr_m, int ignore_group,
                                                                unsigned long long* __restrict__ mask) {
    const int cb = blockIdx.x, rb = blockIdx.y;
    if (cb < rb) return;
    __shared__ __align__(16) float sp[64][kPrepFloats];      // columns
    __shared__ __align__(16) float sr[64][kPrepFloats];      // rows
    __shared__ int sg[64], sgr[64];
    __shared__ unsigned long long sbits[64];
    __shared__ unsigned short list[4096], list2[4096];
    __shared__ int warp_total[kMaskThreads / 32];
    __shared__ int s_total2;
    const int t = threadIdx.x;
    const int col0 = cb * 64, row0 = rb * 64;
    const int row_last = min(row0 + 63, n - 1);
    // groups ascend along the sorted order: no common group -> all-zero word
    const bool tile_live = sgroup[row_last] >= sgroup[col0];
    if (!tile_live) { if (t < 64 && row0 + t < n) mask[(size_t)(row0 + t) * W + cb] = 0ull; return; }
    {   // 64 column records + 64 row records, one float4 per thread (4 float4 per record)
        const int rec = t >> 2, part = t & 3;
        const int c = col0 + rec, r = row0 + rec;
        if (c < n) *reinterpret_cast<float4*>(&sp[rec][part * 4]) = *reinterpret_cast<const float4*>(prep + (size_t)c * kPrepFloats + part * 4);
        if (r < n) *reinterpret_cast<float4*>(&sr[rec][part * 4]) = *reinterpret_cast<const float4*>(prep + (size_t)r * kPrepFloats + part * 4);
        if (t < 64) { sg[t] = (col0 + t < n) ? sgroup[col0 + t] : -1; sgr[t] = (row0 + t < n) ? sgroup[row0 + t] : -2; sbits[t] = 0ull; }
        if (t == 0) s_total2 = 0;
    }
    __syncthreads();
    // thread <-> (row, 16-column quarter)
    const int rl = t & 63, quarter = t >> 6;
    const int row = row0 + rl;
    const int g = sgr[rl];
    const bool row_live = row < n && g != ignore_group;
    if (box_dim != 7) {
        unsigned long long bits = 0ull;
        if (row_live) {
            for (int c = quarter * 16; c < quarter * 16 + 16; ++c) {
                const int col = col0 + c;
                if (col <= row || sg[c] != g) continue;
                const float iou = iou3d_aabb(sr[rl], sp[c]);
                if (!(iou <= thr)) bits |= 1ull << c;
            }
        }
        if (bits) atomicOr(&sbits[rl], bits);
        __syncthreads();
        if (t < 64 && row0 + t < n) mask[(size_t)(row0 + t) * W + cb] = sbits[t];
        return;
    }
    // ---- phase 1: candidate bits of this thread's 16 columns
    const bool cull_ok = (0.0f <= thr);
    unsigned cand = 0u;
    if (row_live) {
        for (int k = 0; k < 16; ++k) {
            const int c = quarter * 16 + k, col = col0 + c;
            if (col <= row || sg[c] != g) continue;
            if (cull_ok && obb_surely_not_above(&sr[rl][8], &sp[c][8], thr_m)) continue;
            cand |= 1u << k;
        }
    }
    // exclusive prefix sum of the candidate counts over the CTA
    const int cnt = __popc(cand);
    const int lane = t & 31, wid = t >> 5;
    int incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
    if (lane == 31) warp_total[wid] = incl;
    __syncthreads();
    int base = incl - cnt, total = 0;
#pragma unroll
    for (int w = 0; w < kMaskThreads / 32; ++w) { if (w < wid) base += warp_total[w]; total += warp_total[w]; }
    while (cand) {
        const int k = __ffs((int)cand) - 1;
        cand &= cand - 1u;
        list[base++] = (unsigned short)((rl << 6) | (quarter * 16 + k));
    }
    __syncthreads();
    // ---- phase 1.5: separating-axis test (exact-zero cull, box_iou.cuh) on the compacted pairs, survivors compacted again -- the test is ~200
    // instructions against ~7 000 for the clip, and a warp only skips the clip when ALL of its 32 pairs are separable, so it has to run first
    const unsigned short* todo = list;
    int total2 = total;
    if (cull_ok) {
        for (int i0 = 0; i0 < total; i0 += kMaskThreads) {
            const int i = i0 + t;
            bool keep = false;
            int e = 0;
            if (i < total) {
                e = list[i];
                ObbPrep a, b;
                load_prep(sr[e >> 6], a);
                load_prep(sp[e & 63], b);
                keep = !obb_footprints_surely_disjoint(a, b);
            }
            const unsigned m = __ballot_sync(0xffffffffu, keep);
            int wbase = 0;
            if (lane == 0 && m) wbase = atomicAdd(&s_total2, __popc(m));
            wbase = __shfl_sync(0xffffffffu, wbase, 0);
            if (keep) list2[wbase + __popc(m & ((1u << lane) - 1u))] = (unsigned short)e;
        }
        __syncthreads();
        todo = list2; total2 = s_total2;
    }
    // ---- phase 2: one candidate pair per thread
    for (int i = t; i < total2; i += kMaskThreads) {
        const int e = todo[i], r = e >> 6, c = e & 63;
        ObbPrep a, b;
        load_prep(sr[r], a);
        load_prep(sp[c], b);
        if (!(iou3d_obb_full(a, b) <= thr)) atomicOr(&sbits[r], 1ull << c);
    }
    __syncthreads();
    if (t < 64 && row0 + t < n) mask[(size_t)(row0 + t) * W + cb] = sbits[t];
}

__device__ __forceinline__ unsigned long long shfl64(unsigned long long v, int src) {
    const unsigned lo = __shfl_sync(0xffffffffu, (unsigned)(v & 0xffffffffull), src);
    const unsigned hi = __shfl_sync(0xffffffffu, (unsigned)(v >> 32), src);
    return ((unsigned long long)hi << 32) | lo;
}

// one CTA per group id
__global__ void __launch_bounds__(256) nms_resolve_kernel(const unsigned long long* __restrict__ mask, int W, int n,
                                                          const int* __restrict__ seg, int ignore_group,
                                                          unsigned long long* __restrict__ keepbits) {
    const int g = blockIdx.x;
    if (g == ignore_group) return;
    const int s = seg[g], e = seg[256 + g];
    if (e <= s) return;
    __shared__ unsigned long long removed[kNmsMatrixMax / 64];
    __shared__ unsigned long long kept_sh;
    const int c0 = s >> 6, c1 = (e - 1) >> 6;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int w = c0 + tid; w <= c1; w += blockDim.x) removed[w] = 0ull;
    __syncthreads();
    for (int c = c0; c <= c1; ++c) {
        if (warp == 0) {
            const int r_lo = c * 64 + lane, r_hi = r_lo + 32;
            const bool v_lo = r_lo >= s && r_lo < e, v_hi = r_hi >= s && r_hi < e;
            const unsigned long long d_lo = v_lo ? mask[(size_t)r_lo * W + c] : 0ull;
            const unsigned long long d_hi = v_hi ? mask[(size_t)r_hi * W + c] : 0ull;
            const unsigned b_lo = __ballot_sync(0xffffffffu, v_lo), b_hi = __ballot_sync(0xffffffffu, v_hi);
            const unsigned long long valid = ((unsigned long long)b_hi << 32) | b_lo;
            unsigned long long rem = removed[c] | ~valid;
            unsigned long long kept = 0ull;
#pragma unroll 8
            for (int i = 0; i < 64; ++i) {
                const unsigned long long rowbits = shfl64(i < 32 ? d_lo : d_hi, i & 31);
                if (!((rem >> i) & 1ull)) { kept |= 1ull << i; rem |= rowbits; }
            }
            if (lane == 0) { kept_sh = kept; if (kept) atomicOr(&keepbits[c], kept); }
        }
        __syncthreads();
        // OR the kept rows into the removed words right of the diagonal: lane <-> word (coalesced), warp <-> 8 of the 64
        // rows, so up to 8 independent loads per thread are in flight (this loop used to be one thread per word walking
        // the kept rows serially: 64 dependent L2 round trips per chunk)
        const unsigned long long kept = kept_sh;
        const unsigned long long mine = (kept >> (warp * 8)) & 0xFFull;
        if (mine) {
            for (int w = c + 1 + lane; w <= c1; w += 32) {
                unsigned long long acc = 0ull;
#pragma unroll
                for (int i = 0; i < 8; ++i)
                    if ((mine >> i) & 1ull) acc |= mask[(size_t)(c * 64 + warp * 8 + i) * W + w];
                if (acc) atomicOr(&removed[w], acc);
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------ chunked path (n > 32 768)
// Sorted boxes are processed in chunks of 4096: (a) every box of the chunk is tested against the boxes KEPT so far
// (one warp per box, lanes stride over the kept list of its group, exact-zero culling first), (b) the 4096 x 4096 bit
// matrix of the chunk is built with the same tile kernel as the matrix path, (c) one CTA resolves the chunk and appends
// the survivors to the kept list. Greedy semantics are unchanged: a box is suppressed iff a higher-scored KEPT box of
// its group overlaps it by more than the threshold.
constexpr int kCrossTile = 256;      // kept records staged per step (one per thread)

// One warp per box of the chunk, 8 boxes per CTA.  The kept list is streamed through shared memory in tiles of 256 cull
// records (floats 8..15 of the prepared record); every lane runs the exact-zero test on one kept box, survivors are pushed
// into a per-warp queue and the full polygon clip only runs on full batches of 32 queued candidates (then once on the
// remainder).  "Suppressed by any kept box of my group" does not depend on the order of the tests, so the result is the
// one of the sequential greedy loop.
__global__ void __launch_bounds__(256) nms_cross_kernel(const float* __restrict__ prep, const int* __restrict__ sgroup, int box_dim,
                                                        float thr, float thr_m, int ignore_group, int chunk_begin, int chunk_n,
                                                        const int* __restrict__ kept_pos, const int* __restrict__ state,
                                                        unsigned long long* __restrict__ removed0) {
    __shared__ __align__(16) float tile[kCrossTile][8];
    __shared__ int tile_pos[kCrossTile];
    __shared__ int queue[8][64], queue2[8][64];
    __shared__ int min_start;
    const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31;
    const int w = blockIdx.x * 8 + wid;
    const bool valid = w < chunk_n;
    const int p = chunk_begin + (valid ? w : 0);
    const int g = valid ? sgroup[p] : -1;
    bool sup = false, done = !valid;
    if (valid && g == ignore_group) { sup = true; done = true; }
    const int kc = state[0];
    const int start = done ? 0x7fffffff : state[1 + g];
    if (tid == 0) min_start = 0x7fffffff;
    __syncthreads();
    if (lane == 0 && !done) atomicMin(&min_start, start);
    __syncthreads();
    const bool cull_ok = (0.0f <= thr);
    const float* bp = prep + (size_t)p * kPrepFloats;
    if (box_dim != 7) {
        // axis-aligned boxes: the IoU itself is a dozen instructions, no staging needed
        if (!done) {
            float b[6];
#pragma unroll
            for (int i = 0; i < 6; ++i) b[i] = bp[i];
            for (int k0 = start; k0 < kc; k0 += 32) {
                const int k = k0 + lane;
                bool hit = false;
                if (k < kc) {
                    const float* a = prep + (size_t)kept_pos[k] * kPrepFloats;
                    float aa[6];
#pragma unroll
                    for (int i = 0; i < 6; ++i) aa[i] = a[i];
                    hit = !(iou3d_aabb(aa, b) <= thr);
                }
                if (__any_sync(0xffffffffu, hit)) { sup = true; break; }
            }
        }
        if (sup && lane == 0) atomicOr(&removed0[w >> 6], 1ull << (w & 63));
        return;
    }
    ObbPrep b;
    load_prep(bp, b);
    float btail[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) btail[i] = bp[8 + i];
    int qn = 0, qn2 = 0;
    for (int k0 = min_start; k0 < kc; k0 += kCrossTile) {
        {
            const int k = k0 + tid;
            if (k < kc) {
                const int pos = kept_pos[k];
                tile_pos[tid] = pos;
                const float4* src = reinterpret_cast<const float4*>(prep + (size_t)pos * kPrepFloats + 8);
                *reinterpret_cast<float4*>(&tile[tid][0]) = src[0];
                *reinterpret_cast<float4*>(&tile[tid][4]) = src[1];
            }
        }
        __syncthreads();
        if (!done) {
            for (int s0 = 0; s0 < kCrossTile; s0 += 32) {
                const int kk = k0 + s0 + lane;
                if (k0 + s0 >= kc) break;
                const bool c = kk < kc && kk >= start && !(cull_ok && obb_surely_not_above(tile[s0 + lane], btail, thr_m));
                const unsigned m = __ballot_sync(0xffffffffu, c);
                if (m) {
                    if (c) queue[wid][qn + __popc(m & ((1u << lane) - 1u))] = tile_pos[s0 + lane];
                    qn += __popc(m);
                    __syncwarp();
                    if (qn >= 32) {
                        // stage 2: separating-axis test on a full warp of queued kept boxes; its survivors wait for a full warp of exact clips
                        const int pos_a = queue[wid][lane];
                        ObbPrep a;
                        load_prep(prep + (size_t)pos_a * kPrepFloats, a);
                        const bool keep = !(cull_ok && obb_footprints_surely_disjoint(a, b));
                        const unsigned m2 = __ballot_sync(0xffffffffu, keep);
                        if (keep) queue2[wid][qn2 + __popc(m2 & ((1u << lane) - 1u))] = pos_a;
                        qn2 += __popc(m2);
                        const int rest = qn - 32;
                        const int moved = lane < rest ? queue[wid][32 + lane] : 0;
                        __syncwarp();
                        if (lane < rest) queue[wid][lane] = moved;
                        qn = rest;
                        __syncwarp();
                        if (qn2 >= 32) {
                            load_prep(prep + (size_t)queue2[wid][lane] * kPrepFloats, a);
                            const bool hit = !(iou3d_obb_full(a, b) <= thr);
                            if (__any_sync(0xffffffffu, hit)) { sup = true; done = true; break; }
                            const int rest2 = qn2 - 32;
                            const int moved2 = lane < rest2 ? queue2[wid][32 + lane] : 0;
                            __syncwarp();
                            if (lane < rest2) queue2[wid][lane] = moved2;
                            qn2 = rest2;
                            __syncwarp();
                        }
                    }
                }
            }
        }
        if (__syncthreads_and(done ? 1 : 0)) break;          // also fences the tile before it is overwritten
    }
    if (!done) {                                                  // remainders of both stages (each fewer than 32 entries)
        bool hit = false;
        if (lane < qn) {
            ObbPrep a;
            load_prep(prep + (size_t)queue[wid][lane] * kPrepFloats, a);
            hit = obb_suppresses(a, b, thr);
        }
        if (lane < qn2) {
            ObbPrep a;
            load_prep(prep + (size_t)queue2[wid][lane] * kPrepFloats, a);
            hit = hit || !(iou3d_obb_full(a, b) <= thr);
        }
        if (__any_sync(0xffffffffu, hit)) sup = true;
    }
    if (sup && lane == 0) atomicOr(&removed0[w >> 6], 1ull << (w & 63));
}

// one CTA: resolve the chunk (all groups at once: mask bits only ever connect boxes of the same group), append survivors
__global__ void __launch_bounds__(256) nms_chunk_resolve_kernel(const unsigned long long* __restrict__ cmask, int Wc, int chunk_begin,
                                                                int chunk_n, const int* __restrict__ sgroup,
                                                                unsigned long long* __restrict__ removed0, int* __restrict__ kept_pos,
                                                                int* __restrict__ state, unsigned long long* __restrict__ keepbits) {
    __shared__ unsigned long long removed[64];
    __shared__ unsigned long long kept_sh;
    __shared__ int kept_base;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 64) { removed[tid] = removed0[tid]; removed0[tid] = 0ull; }       // leave the scratch zeroed for the next chunk
    if (tid == 0) kept_base = state[0];
    __syncthreads();
    for (int c = 0; c < Wc; ++c) {
        if (warp == 0) {
            const int r_lo = c * 64 + lane, r_hi = r_lo + 32;
            const bool v_lo = r_lo < chunk_n, v_hi = r_hi < chunk_n;
            const unsigned long long d_lo = v_lo ? cmask[(size_t)r_lo * Wc + c] : 0ull;
            const unsigned long long d_hi = v_hi ? cmask[(size_t)r_hi * Wc + c] : 0ull;
            const unsigned b_lo = __ballot_sync(0xffffffffu, v_lo), b_hi = __ballot_sync(0xffffffffu, v_hi);
            const unsigned long long valid = ((unsigned long long)b_hi << 32) | b_lo;
            unsigned long long rem = removed[c] | ~valid;
            unsigned long long kept = 0ull;
#pragma unroll 8
            for (int i = 0; i < 64; ++i) {
                const unsigned long long rowbits = shfl64(i < 32 ? d_lo : d_hi, i & 31);
                if (!((rem >> i) & 1ull)) { kept |= 1ull << i; rem |= rowbits; }
            }
            // append survivors in order; remember where each group's kept boxes start
            const int base = kept_base;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int i = lane + 32 * h;
                if ((kept >> i) & 1ull) {
                    const int pos = chunk_begin + c * 64 + i;
                    const int ki = base + __popcll(kept & ((1ull << i) - 1ull));
                    kept_pos[ki] = pos;
                    atomicMin(&state[1 + sgroup[pos]], ki);
                }
            }
            if (lane == 0) { kept_sh = kept; kept_base = base + __popcll(kept); keepbits[(chunk_begin >> 6) + c] = kept; }
        }
        __syncthreads();
        const unsigned long long kept = kept_sh;
        const unsigned long long mine = (kept >> (warp * 8)) & 0xFFull;
        if (mine) {
            for (int w = c + 1 + lane; w < Wc; w += 32) {
                unsigned long long acc = 0ull;
#pragma unroll
                for (int i = 0; i < 8; ++i)
                    if ((mine >> i) & 1ull) acc |= cmask[(size_t)(c * 64 + warp * 8 + i) * Wc + w];
                if (acc) atomicOr(&removed[w], acc);
            }
        }
        __syncthreads();
    }
    if (tid == 0) state[0] = kept_base;
}


// ------------------------------------------------------------------------------ binned chunked path (n >= kBinMinBoxes)
__device__ __forceinline__ float ordered_to_float(unsigned u) { return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u); }

// pass 0 (pass == 0): min / max of centre x, y, z and of log2(volume) over the cullable boxes.  pass 1: per-class max radius / depth.
__global__ void nms_bin_stats_kernel(const float* __restrict__ prep, int n, int pass, const BinGrid* __restrict__ grid, unsigned* __restrict__ st) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const float* t = prep + (size_t)p * kPrepFloats + 8;
    if (!__float_as_int(t[7])) return;
    const float zc = 0.5f * (t[2] + t[3]), lv = log2f(t[1]);
    if (pass == 0) {
        atomicMin(&st[0], float_to_ordered(t[4])); atomicMax(&st[1], float_to_ordered(t[4]));
        atomicMin(&st[2], float_to_ordered(t[5])); atomicMax(&st[3], float_to_ordered(t[5]));
        atomicMin(&st[4], float_to_ordered(zc)); atomicMax(&st[5], float_to_ordered(zc));
        atomicMin(&st[6], float_to_ordered(lv)); atomicMax(&st[7], float_to_ordered(lv));
    } else {
        int c = (int)floorf((lv - grid->lv0) * grid->inv_lw);
        c = c < 0 ? 0 : (c >= grid->n_cls ? grid->n_cls - 1 : c);
        atomicMax(&st[8 + c], float_to_ordered(t[6]));
        atomicMax(&st[8 + kBinClasses + c], float_to_ordered(t[3] - t[2]));
    }
}

__global__ void nms_bin_stats_init_kernel(unsigned* __restrict__ st) {
    const int t = threadIdx.x;
    if (t < kBinStatWords) st[t] = (t < 8 && !(t & 1)) ? 0xFFFFFFFFu : 0u;          // mins start at +max, maxes at the lowest key
}

// stage 0: class mapping from the global extents; stage 1: per-class cell sizes / counts from the per-class maxima
__global__ void nms_bin_grid_kernel(const unsigned* __restrict__ st, float thr_m, int stage, BinGrid* __restrict__ g) {
    if (threadIdx.x != 0) return;
    if (stage == 0) {
        const bool any = st[0] != 0xFFFFFFFFu;
        g->x0 = any ? ordered_to_float(st[0]) : 0.f; g->y0 = any ? ordered_to_float(st[2]) : 0.f; g->z0 = any ? ordered_to_float(st[4]) : 0.f;
        g->lv0 = any ? ordered_to_float(st[6]) : 0.f;
        const float span = any ? ordered_to_float(st[7]) - g->lv0 : 0.f;
        float width = (thr_m > 0.f && thr_m < 1.f) ? log2f(1.0f / thr_m) : 1e30f;        // no ratio cull: a single class
        if (span / width > (float)(kBinClasses - 1)) width = span / (float)(kBinClasses - 1) * 1.0001f;   // wider classes stay conservative
        g->inv_lw = 1.0f / width;
        int nc = (int)floorf(span * g->inv_lw) + 1;
        g->n_cls = nc < 1 ? 1 : (nc > kBinClasses ? kBinClasses : nc);
        return;
    }
    const float ex = ordered_to_float(st[1]) - g->x0, ey = ordered_to_float(st[3]) - g->y0, ez = ordered_to_float(st[5]) - g->z0;
    for (int c = 0; c < kBinClasses; ++c) {
        const float r = st[8 + c] ? ordered_to_float(st[8 + c]) : 0.f, d = st[8 + kBinClasses + c] ? ordered_to_float(st[8 + kBinClasses + c]) : 0.f;
        g->rmax[c] = r; g->dmax[c] = d;
        // cells half of the class's largest diameter / depth wide: a query window of +-(r_j + r_c) / S cells then hugs the volume that can
        // hold a partner (3 x 3 cells of size 2 r_c would cover 3x that area) while a box still visits only ~100 cells per class
        float S = fmaxf(r, fmaxf(ex, ey) / (float)kBinMaxXY * 1.0001f);
        float Sz = fmaxf(0.5f * d, ez / (float)kBinMaxZ * 1.0001f);
        if (!(S > 0.f)) S = 1.0f;
        if (!(Sz > 0.f)) Sz = 1.0f;
        g->S[c] = S; g->Sz[c] = Sz;
        int nx = (int)floorf(ex / S) + 1, ny = (int)floorf(ey / S) + 1, nz = (int)floorf(ez / Sz) + 1;
        g->nx[c] = nx < 1 ? 1 : (nx > kBinMaxXY ? kBinMaxXY : nx);
        g->ny[c] = ny < 1 ? 1 : (ny > kBinMaxXY ? kBinMaxXY : ny);
        g->nz[c] = nz < 1 ? 1 : (nz > kBinMaxZ ? kBinMaxZ : nz);
    }
}

__device__ __forceinline__ int bin_clampi(int v, int n) { return v < 0 ? 0 : (v >= n ? n - 1 : v); }

// cell of every box (kBinCells - 1 = the "everywhere" cell of boxes without a usable cull record) + per-cell counts
__global__ void nms_bin_assign_kernel(const float* __restrict__ prep, int n, const BinGrid* __restrict__ g, int* __restrict__ box_cell,
                                      int* __restrict__ cell_count) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const float* t = prep + (size_t)p * kPrepFloats + 8;
    int cell = kBinCells - 1;
    if (__float_as_int(t[7])) {
        int c = (int)floorf((log2f(t[1]) - g->lv0) * g->inv_lw);
        c = bin_clampi(c, g->n_cls);
        const int ix = bin_clampi((int)floorf((t[4] - g->x0) / g->S[c]), g->nx[c]);
        const int iy = bin_clampi((int)floorf((t[5] - g->y0) / g->S[c]), g->ny[c]);
        const int iz = bin_clampi((int)floorf((0.5f * (t[2] + t[3]) - g->z0) / g->Sz[c]), g->nz[c]);
        cell = c * kBinCellsPerClass + (iz * kBinMaxXY + iy) * kBinMaxXY + ix;
    }
    box_cell[p] = cell;
    atomicAdd(&cell_count[cell], 1);
}

// exclusive scan of cell_count (kBinCells entries) into cell_start (kBinCells + 1), one CTA
__global__ void __launch_bounds__(1024) nms_bin_scan_kernel(const int* __restrict__ cell_count, int* __restrict__ cell_start) {
    __shared__ int part[1024];
    const int t = threadIdx.x;
    const int per = (kBinCells + 1023) / 1024;
    const int b = t * per, e = b + per < kBinCells ? b + per : kBinCells;
    int s = 0;
    for (int i = b; i < e; ++i) s += cell_count[i];
    part[t] = s;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) { const int v = t >= o ? part[t - o] : 0; __syncthreads(); part[t] += v; __syncthreads(); }
    int run = part[t] - s;
    for (int i = b; i < e; ++i) { cell_start[i] = run; run += cell_count[i]; }
    if (t == 1023) cell_start[kBinCells] = part[1023];
}

// One warp per box of the chunk.  Lanes take the cells of the box's 3-D window in the current volume class (32 cells per batch), each lane walks
// its own cell's kept records -- 48-byte records {cull record, position, group} stored cell by cell, so the walk is one sequential stream per
// lane with no dependent look-ups; entries that survive the group / cull tests are queued and the exact IoU runs on full batches of 32
// (cf. nms_cross_kernel).
__global__ void __launch_bounds__(256, 2) nms_cross_binned_kernel(const float* __restrict__ prep, const int* __restrict__ sgroup, int box_dim,
                                                                  float thr, float thr_m, int ignore_group, int chunk_begin, int chunk_n,
                                                                  const BinGrid* __restrict__ grid, const int* __restrict__ cell_start,
                                                                  const int* __restrict__ cell_fill, const float4* __restrict__ cell_recs,
                                                                  unsigned long long* __restrict__ removed0) {
    __shared__ int queue[8][64];
    const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31;
    const int w = blockIdx.x * 8 + wid;
    if (w >= chunk_n) return;
    const int p = chunk_begin + w;
    const int g = sgroup[p];
    if (g == ignore_group) { if (lane == 0) atomicOr(&removed0[w >> 6], 1ull << (w & 63)); return; }
    const float* bp = prep + (size_t)p * kPrepFloats;
    float btail[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) btail[i] = bp[8 + i];
    const bool cull_ok = (0.0f <= thr);
    const BinGrid& G = *grid;
    const bool j_cull = __float_as_int(btail[7]) != 0 && cull_ok;
    int cj = 0;
    if (j_cull) cj = bin_clampi((int)floorf((log2f(btail[1]) - G.lv0) * G.inv_lw), G.n_cls);
    const float zc = 0.5f * (btail[2] + btail[3]), dj = btail[3] - btail[2];
    int qn = 0;
    bool sup = false;

    auto exact = [&](int pos) -> bool {                 // the decision of the sequential loop for one kept box
        const float* ap = prep + (size_t)pos * kPrepFloats;
        if (box_dim == 7) { ObbPrep a, b; load_prep(ap, a); load_prep(bp, b); return obb_suppresses(a, b, thr); }
        float aa[6], bb[6];
#pragma unroll
        for (int i = 0; i < 6; ++i) { aa[i] = ap[i]; bb[i] = bp[i]; }
        return !(iou3d_aabb(aa, bb) <= thr);
    };
    auto visit = [&](int beg, int end) {                // every lane walks its own record range; reports through `sup`
        int e = beg;
        while (true) {
            const bool have = e < end;
            if (!__any_sync(0xffffffffu, have)) break;
            bool c = false;
            int pos = 0;
            if (have) {
                const float4* r = cell_recs + (size_t)e * 3;
                const float4 r0 = __ldg(r), r1 = __ldg(r + 1), r2 = __ldg(r + 2);
                pos = __float_as_int(r2.x);
                if (__float_as_int(r2.y) == g) {
                    const float at[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
                    c = !(cull_ok && obb_surely_not_above(at, btail, thr_m));
                }
                ++e;
            }
            const unsigned m = __ballot_sync(0xffffffffu, c);
            if (m) {
                if (c) queue[wid][qn + __popc(m & ((1u << lane) - 1u))] = pos;
                qn += __popc(m);
                __syncwarp();
                if (qn >= 32) {
                    const bool hit = exact(queue[wid][lane]);
                    if (__any_sync(0xffffffffu, hit)) { sup = true; return; }
                    const int rest = qn - 32;
                    const int moved = lane < rest ? queue[wid][32 + lane] : 0;
                    __syncwarp();
                    if (lane < rest) queue[wid][lane] = moved;
                    qn = rest;
                    __syncwarp();
                }
            }
        }
    };

    {   // boxes without a cull record sit in the last cell: everyone visits it, the lanes share its records in contiguous pieces
        const int cs = cell_start[kBinCells - 1], cf = cell_fill[kBinCells - 1];
        const int per = (cf + 31) / 32;
        const int b0 = cs + lane * per, b1 = min(cs + cf, b0 + per);
        visit(b0, b1 > b0 ? b1 : b0);
    }
    if (!sup) {
        const int c_lo = j_cull ? max(cj - 1, 0) : 0, c_hi = j_cull ? min(cj + 1, G.n_cls - 1) : G.n_cls - 1;
        for (int c = c_lo; c <= c_hi && !sup; ++c) {
            int ix0 = 0, ix1 = G.nx[c] - 1, iy0 = 0, iy1 = G.ny[c] - 1, iz0 = 0, iz1 = G.nz[c] - 1;
            if (j_cull) {
                const float R = btail[6] + G.rmax[c], Rz = 0.5f * (dj + G.dmax[c]);
                ix0 = bin_clampi((int)floorf((btail[4] - R - G.x0) / G.S[c]), G.nx[c]); ix1 = bin_clampi((int)floorf((btail[4] + R - G.x0) / G.S[c]), G.nx[c]);
                iy0 = bin_clampi((int)floorf((btail[5] - R - G.y0) / G.S[c]), G.ny[c]); iy1 = bin_clampi((int)floorf((btail[5] + R - G.y0) / G.S[c]), G.ny[c]);
                iz0 = bin_clampi((int)floorf((zc - Rz - G.z0) / G.Sz[c]), G.nz[c]); iz1 = bin_clampi((int)floorf((zc + Rz - G.z0) / G.Sz[c]), G.nz[c]);
            }
            const int wx = ix1 - ix0 + 1, wy = iy1 - iy0 + 1, wxy = wx * wy, n_cells = wxy * (iz1 - iz0 + 1);
            for (int k0 = 0; k0 < n_cells && !sup; k0 += 32) {
                const int k = k0 + lane;
                int beg = 0, end = 0;
                if (k < n_cells) {
                    const int kz = k / wxy, kr = k - kz * wxy;
                    const int cell = c * kBinCellsPerClass + ((iz0 + kz) * kBinMaxXY + (iy0 + kr / wx)) * kBinMaxXY + ix0 + kr % wx;
                    beg = cell_start[cell]; end = beg + cell_fill[cell];
                }
                visit(beg, end);
            }
        }
    }
    if (!sup && qn > 0) {
        bool hit = false;
        if (lane < qn) hit = exact(queue[wid][lane]);
        if (__any_sync(0xffffffffu, hit)) sup = true;
    }
    if (sup && lane == 0) atomicOr(&removed0[w >> 6], 1ull << (w & 63));
}

// files the survivors of a resolved chunk (kept_pos[k0 .. k1)) in their cells
__global__ void nms_bin_file_kernel(const int* __restrict__ kept_pos, const int* __restrict__ state, int* __restrict__ filed, const int* __restrict__ box_cell,
                                    const float* __restrict__ prep, const int* __restrict__ sgroup, const int* __restrict__ cell_start,
                                    int* __restrict__ cell_fill, float4* __restrict__ cell_recs) {
    const int k0 = filed[0], k1 = state[0];
    for (int k = k0 + blockIdx.x * blockDim.x + threadIdx.x; k < k1; k += gridDim.x * blockDim.x) {
        const int pos = kept_pos[k], cell = box_cell[pos];
        const float4* t = reinterpret_cast<const float4*>(prep + (size_t)pos * kPrepFloats + 8);
        float4* r = cell_recs + (size_t)(cell_start[cell] + atomicAdd(&cell_fill[cell], 1)) * 3;
        r[0] = t[0]; r[1] = t[1];
        r[2] = make_float4(__int_as_float(pos), __int_as_float(sgroup[pos]), 0.f, 0.f);
    }
}
__global__ void nms_bin_filed_kernel(const int* __restrict__ state, int* __restrict__ filed) { filed[0] = state[0]; }

__global__ void nms_state_init_kernel(int* __restrict__ state) {
    const int t = threadIdx.x;
    if (t == 0) state[0] = 0;
    if (t < 256) state[1 + t] = 0x7fffffff;
}

__global__ void nms_keys2_kernel(const unsigned long long* __restrict__ keys, const unsigned long long* __restrict__ keepbits,
                                 int n, int n_pad, unsigned long long* __restrict__ keys2) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_pad) return;
    unsigned long long k = ~0ull;
    if (p < n && ((keepbits[p >> 6] >> (p & 63)) & 1ull)) k = keys[p] & 0x00FFFFFFFFFFFFFFull;   // drop the group byte
    keys2[p] = k;
}

__global__ void nms_emit_kernel(const unsigned long long* __restrict__ keys2, int n, int64_t* __restrict__ keep,
                                int32_t* __restrict__ n_keep) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const bool v = keys2[p] != ~0ull;
    if (v) keep[p] = (int64_t)(keys2[p] & 0xFFFFFFull);
    const bool vn = (p + 1 < n) ? (keys2[p + 1] != ~0ull) : false;
    if (v && !vn) *n_keep = p + 1;
    if (p == 0 && !v) *n_keep = 0;
}


#include "nms_cells.cuh"

static int level_growth_pct() {          // level e -> e * pct / 100 (NRPN_NMS_LEVEL_GROWTH_PCT, tuning runs; >= 110)
    static const int v = [] { const char* e = getenv("NRPN_NMS_LEVEL_GROWTH_PCT"); const int k = e ? atoi(e) : kLevelGrowth * 100; return k < 110 ? 110 : k; }();
    return v;
}

static size_t cl_layout(void* base, int n, CellWs* out) {
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
    char* b = (char*)base;
    CellWs c;
    c.state = (signed char*)(b + take((size_t)n));
    c.adj_cnt = (int*)(b + take((size_t)n * 4));
    c.adj = (int*)(b + take((size_t)n * kAdjSlots * 4));
    for (CellIndex* X : {&c.A, &c.B}) {
        X->start = (int*)(b + take((size_t)(kBinCells + 1) * 4));
        X->cursor = (int*)(b + take((size_t)kBinCells * 4));
        X->recs = (float4*)(b + take((size_t)n * 48));
        X->item_start = (int*)(b + take((size_t)(kBinCells + 1) * 4));
        X->items = (int2*)(b + take(((size_t)n / kQB + kBinCells + 2) * 8));
    }
    c.totals = (unsigned long long*)(b + take((size_t)kScanBlocks * 8));
    c.meta = (int*)(b + take(64));
    c.und = (int*)(b + take(kRoundBatch * 4));
    c.fail = (int*)(b + take(64));
    c.blk = (int*)(b + take(((size_t)n / 1024 + 2) * 4));
    if (out) *out = c;
    return off;
}

// returns NRPN_OK with *declined = true when the input needs the chunked path (nothing has been written to keep / n_keep then)
static int nms_run_cells(const float* boxes, int box_dim, const float* scores, const int32_t* group, int n, float thr, int ignore_group,
                         int64_t* keep, int32_t* n_keep, const NmsWs& w, const CellWs& c, cudaStream_t st, bool* declined, float thr_m) {
    *declined = false;
    const int n_pad = next_pow2(n);
    nms_keys_kernel<<<ceil_div(n_pad, 256), 256, 0, st>>>(scores, nullptr, n, n_pad, w.keys);
    NRPN_LAUNCH_CHECK();
    int rc = bitonic_sort_u64(w.keys, n_pad, st);
    if (rc) return rc;
    nms_prep_kernel<<<ceil_div(n, 128), 128, 0, st>>>(w.keys, boxes, box_dim, n, w.prep, w.sgroup, w.seg, group);
    NRPN_LAUNCH_CHECK();
    // grid of the cell lists (shared with the chunked path's index: extents -> volume classes -> per-class cell sizes -> cell of every box)
    nms_bin_stats_init_kernel<<<1, 64, 0, st>>>(w.bstats);
    nms_bin_stats_kernel<<<ceil_div(n, 256), 256, 0, st>>>(w.prep, n, 0, w.grid, w.bstats);
    nms_bin_grid_kernel<<<1, 32, 0, st>>>(w.bstats, thr_m, 0, w.grid);
    nms_bin_stats_kernel<<<ceil_div(n, 256), 256, 0, st>>>(w.prep, n, 1, w.grid, w.bstats);
    nms_bin_grid_kernel<<<1, 32, 0, st>>>(w.bstats, thr_m, 1, w.grid);
    NRPN_LAUNCH_CHECK();
    NRPN_CUDA_TRY(cudaMemsetAsync(w.cell_fill, 0, (size_t)kBinCells * 4, st));
    nms_bin_assign_kernel<<<ceil_div(n, 256), 256, 0, st>>>(w.prep, n, w.grid, w.box_cell, w.cell_fill);
    NRPN_LAUNCH_CHECK();
    NRPN_CUDA_TRY(cudaMemsetAsync(c.A.cursor, 0, (size_t)kBinCells * 4, st));
    NRPN_CUDA_TRY(cudaMemsetAsync(c.B.cursor, 0, (size_t)kBinCells * 4, st));
    NRPN_CUDA_TRY(cudaMemsetAsync(c.fail, 0, 4, st));
    cl_state_init_kernel<<<ceil_div(n, 256), 256, 0, st>>>(w.sgroup, n, ignore_group, c.state, c.adj_cnt);
    NRPN_LAUNCH_CHECK();

    static const int pair_grid = [] { int dev = 0, sms = 132; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); return 2 * sms; }();
    PairArgs pa;
    pa.prep = w.prep; pa.box_dim = box_dim; pa.thr = thr; pa.thr_m = thr_m; pa.grid = w.grid;
    pa.qstart = c.B.start; pa.qrecs = c.B.recs; pa.item_start = c.B.item_start; pa.items = c.B.items; pa.work = c.meta;
    pa.state = c.state; pa.adj_cnt = c.adj_cnt; pa.adj = c.adj; pa.fail = c.fail;
    int b = 0;
    for (int e = n < kLevel0 ? n : kLevel0; b < n; ) {
        const int m = e - b;
        if (b > 0) {
            cl_build_index(c.A, c, w, 0, b, ST_KEPT, false, st);             // kept boxes of the earlier levels
            cl_build_index(c.B, c, w, b, e, ST_UNDECIDED, true, st);         // this level's boxes as queries
            NRPN_LAUNCH_CHECK();
            NRPN_CUDA_TRY(cudaMemsetAsync(c.meta, 0, 4, st));
            pa.rstart = c.A.start; pa.rrecs = c.A.recs;
            cl_pairs_kernel<0><<<pair_grid, kPairThreads, 0, st>>>(pa);
            NRPN_LAUNCH_CHECK();
        }
        cl_build_index(c.B, c, w, b, e, ST_UNDECIDED, true, st);             // the survivors, against each other
        NRPN_LAUNCH_CHECK();
        NRPN_CUDA_TRY(cudaMemsetAsync(c.meta, 0, 4, st));
        pa.rstart = c.B.start; pa.rrecs = c.B.recs;
        cl_pairs_kernel<1><<<pair_grid, kPairThreads, 0, st>>>(pa);
        NRPN_LAUNCH_CHECK();
        const int rgrid = ceil_div(m, 256) < 1184 ? ceil_div(m, 256) : 1184;
        for (int rounds = 0;; rounds += kRoundBatch) {
            NRPN_CUDA_TRY(cudaMemsetAsync(c.und, 0, kRoundBatch * 4, st));
            for (int r = 0; r < kRoundBatch; ++r) cl_round_kernel<<<rgrid, 256, 0, st>>>(c.B.recs, c.B.start, c.adj_cnt, c.adj, c.state, c.und, r);
            NRPN_LAUNCH_CHECK();
            int h[2] = {0, 0};
            NRPN_CUDA_TRY(cudaMemcpyAsync(&h[0], c.und + kRoundBatch - 1, 4, cudaMemcpyDeviceToHost, st));
            NRPN_CUDA_TRY(cudaMemcpyAsync(&h[1], c.fail, 4, cudaMemcpyDeviceToHost, st));
            NRPN_CUDA_TRY(cudaStreamSynchronize(st));
            if (h[1] || rounds > kRoundCap) { *declined = true; return NRPN_OK; }
            if (h[0] == 0) break;
        }
        b = e;
        { const long long nx = (long long)e * level_growth_pct() / 100; e = nx > (long long)n ? n : (int)nx; }
    }
    const int nblk = ceil_div(n, 1024);
    cl_keep_count_kernel<<<nblk, 1024, 0, st>>>(c.state, n, c.blk);
    cl_keep_scan_kernel<<<1, 1024, 0, st>>>(c.blk, nblk, n_keep);
    cl_keep_emit_kernel<<<nblk, 1024, 0, st>>>(c.state, w.keys, n, c.blk, keep);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

size_t nms_workspace_bytes(int n) {
    if (n <= 0) return 256;
    return nms_layout(nullptr, n).total + (n >= cell_min_boxes() ? cl_layout(nullptr, n, nullptr) : 0) + 256;
}

int nms_run(const float* boxes, int box_dim, const float* scores, const int32_t* group, int n, float thr, int ignore_group,
            int64_t* keep, int32_t* n_keep, void* ws, size_t ws_bytes, cudaStream_t st, int max_group) {
    if (max_group <= 0 || max_group > n) max_group = n;
    if (n == 0) { NRPN_CUDA_TRY(cudaMemsetAsync(n_keep, 0, 4, st)); return NRPN_OK; }
    if (n > kNmsMaxBoxes) return NRPN_ERR_UNSUPPORTED;
    if (ws_bytes < nms_workspace_bytes(n)) return NRPN_ERR_WORKSPACE;
    void* base = (void*)align_up((size_t)ws, 256);
    NmsWs w = nms_layout(base, n);
    // Cull mode (nrpn_set_nms_cull_mode).  The exact-zero culls (bounding circles / z ranges disjoint -> the reference computes exactly 0) are always
    // on.  The RATIO culls (volume ratio, z-overlap ratio, footprint lens; box_iou.cuh) bound the GEOMETRIC IoU -- but the reference's vertex sort
    // replaces an unsortable vertex (mean-centred y == 0.0f, coincident points) by corner 0 of the first box, and then reports MORE than the geometric
    // value (DESIGN.md 3.3: ~1e-8 of the touching pairs; 1-3 of 85 702 kept boxes at 256 000 boxes).  They are therefore opt-in (bit 0: volume /
    // depth ratios, bit 1: + footprint lens), only ever applied from 16 384 boxes up, and the default keep set is provably the sequential loop's.
    const int cull_mode = g_nms_cull_mode.load(std::memory_order_relaxed);
    const float thr_m = ((cull_mode & 1) && n >= kRatioCullMinBoxes) ? thr - 1e-3f : 0.0f;
    {
        static std::atomic<int> applied{-1};
        const int lens = (cull_mode >> 1) & 1;
        if (applied.load(std::memory_order_relaxed) != lens) {
            NRPN_CUDA_TRY(cudaMemcpyToSymbolAsync(g_lens_cull, &lens, sizeof(int), 0, cudaMemcpyHostToDevice, st));
            NRPN_CUDA_TRY(cudaStreamSynchronize(st));
            applied.store(lens, std::memory_order_relaxed);
        }
    }
    if (n >= cell_min_boxes() && thr >= 0.0f) {
        static const bool cells_off = [] { const char* e = getenv("NRPN_NMS_CELLS"); return e && e[0] == '0'; }();
        cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
        cudaStreamIsCapturing(st, &cap);                    // the level loop reads counters back: not capturable
        if (!cells_off && cap == cudaStreamCaptureStatusNone) {
            CellWs c;
            cl_layout((char*)base + w.total, n, &c);
            bool declined = false;
            const int rc = nms_run_cells(boxes, box_dim, scores, group, n, thr, ignore_group, keep, n_keep, w, c, st, &declined, thr_m);
            if (rc || !declined) return rc;
        }
    }
    const int n_pad = next_pow2(n < 2 ? 2 : n);
    const int W = ceil_div(n, 64);
    NRPN_CUDA_TRY(cudaMemsetAsync(w.seg, 0, 512 * 4, st));
    NRPN_CUDA_TRY(cudaMemsetAsync(w.keepbits, 0, (size_t)W * 8, st));
    nms_keys_kernel<<<ceil_div(n_pad, 256), 256, 0, st>>>(scores, group, n, n_pad, w.keys);
    NRPN_LAUNCH_CHECK();
    int rc = bitonic_sort_u64(w.keys, n_pad, st);
    if (rc) return rc;
    nms_prep_kernel<<<ceil_div(n, 128), 128, 0, st>>>(w.keys, boxes, box_dim, n, w.prep, w.sgroup, w.seg);
    NRPN_LAUNCH_CHECK();
    if (nms_use_matrix(n, max_group)) {
        nms_mask_kernel<<<dim3(W, W), kMaskThreads, 0, st>>>(w.prep, w.sgroup, n, W, box_dim, thr, thr_m, ignore_group, w.mask);
        NRPN_LAUNCH_CHECK();
        nms_resolve_kernel<<<256, 256, 0, st>>>(w.mask, W, n, w.seg, ignore_group, w.keepbits);
        NRPN_LAUNCH_CHECK();
    } else {
        NRPN_CUDA_TRY(cudaMemsetAsync(w.removed0, 0, 64 * 8, st));
        nms_state_init_kernel<<<1, 256, 0, st>>>(w.state);
        NRPN_LAUNCH_CHECK();
        const int chunk = nms_chunk_size(n);
        static const bool bin_off = [] { const char* e = getenv("NRPN_NMS_BINNED"); return e && e[0] == '0'; }();
        const bool binned = n >= kBinMinBoxes && !bin_off;
        int* filed = w.state + 257;
        if (binned) {
            // grid of the kept-box index: extents -> classes -> per-class cell sizes -> cell of every box -> segment capacities
            nms_bin_stats_init_kernel<<<1, 64, 0, st>>>(w.bstats);
            NRPN_LAUNCH_CHECK();
            nms_bin_stats_kernel<<<ceil_div(n, 256), 256, 0, st>>>(w.prep, n, 0, w.grid, w.bstats);
            NRPN_LAUNCH_CHECK();
            nms_bin_grid_kernel<<<1, 32, 0, st>>>(w.bstats, thr_m, 0, w.grid);
            NRPN_LAUNCH_CHECK();
            nms_bin_stats_kernel<<<ceil_div(n, 256), 256, 0, st>>>(w.prep, n, 1, w.grid, w.bstats);
            NRPN_LAUNCH_CHECK();
            nms_bin_grid_kernel<<<1, 32, 0, st>>>(w.bstats, thr_m, 1, w.grid);
            NRPN_LAUNCH_CHECK();
            NRPN_CUDA_TRY(cudaMemsetAsync(w.cell_fill, 0, (size_t)kBinCells * 4, st));
            nms_bin_assign_kernel<<<ceil_div(n, 256), 256, 0, st>>>(w.prep, n, w.grid, w.box_cell, w.cell_fill);
            NRPN_LAUNCH_CHECK();
            nms_bin_scan_kernel<<<1, 1024, 0, st>>>(w.cell_fill, w.cell_start);
            NRPN_LAUNCH_CHECK();
            NRPN_CUDA_TRY(cudaMemsetAsync(w.cell_fill, 0, (size_t)kBinCells * 4, st));
            NRPN_CUDA_TRY(cudaMemsetAsync(filed, 0, 4, st));
        }
        for (int cb = 0; cb < n; cb += chunk) {
            const int cn = n - cb < chunk ? n - cb : chunk;
            const int Wc = ceil_div(cn, 64);
            if (binned) {
                nms_bin_file_kernel<<<8, 256, 0, st>>>(w.kept_pos, w.state, filed, w.box_cell, w.prep, w.sgroup, w.cell_start, w.cell_fill, w.cell_recs);
                NRPN_LAUNCH_CHECK();
                nms_bin_filed_kernel<<<1, 1, 0, st>>>(w.state, filed);
                NRPN_LAUNCH_CHECK();
                nms_cross_binned_kernel<<<ceil_div(cn, 8), 256, 0, st>>>(w.prep, w.sgroup, box_dim, thr, thr_m, ignore_group, cb, cn, w.grid,
                                                                         w.cell_start, w.cell_fill, w.cell_recs, w.removed0);
            } else
            nms_cross_kernel<<<ceil_div(cn, 8), 256, 0, st>>>(w.prep, w.sgroup, box_dim, thr, thr_m, ignore_group, cb, cn,
                                                                     w.kept_pos, w.state, w.removed0);
            NRPN_LAUNCH_CHECK();
            nms_mask_kernel<<<dim3(Wc, Wc), kMaskThreads, 0, st>>>(w.prep + (size_t)cb * kPrepFloats, w.sgroup + cb, cn, Wc, box_dim, thr, thr_m,
                                                        ignore_group, w.mask);
            NRPN_LAUNCH_CHECK();
            nms_chunk_resolve_kernel<<<1, 256, 0, st>>>(w.mask, Wc, cb, cn, w.sgroup, w.removed0, w.kept_pos, w.state, w.keepbits);
            NRPN_LAUNCH_CHECK();
        }
    }
    nms_keys2_kernel<<<ceil_div(n_pad, 256), 256, 0, st>>>(w.keys, w.keepbits, n, n_pad, w.keys2);
    NRPN_LAUNCH_CHECK();
    rc = bitonic_sort_u64(w.keys2, n_pad, st);
    if (rc) return rc;
    nms_emit_kernel<<<ceil_div(n, 256), 256, 0, st>>>(w.keys2, n, keep, n_keep);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

}  // namespace nrpn

using namespace nrpn;

extern "C" {
#pragma GCC visibility push(default)

void nrpn_set_nms_cull_mode(int mode) { g_nms_cull_mode.store(mode & 3, std::memory_order_relaxed); }
int nrpn_get_nms_cull_mode(void) { return g_nms_cull_mode.load(std::memory_order_relaxed); }

int nrpn_nms_cells_stats(unsigned long long* out16, int reset) {
    if (out16) NRPN_CUDA_TRY(cudaMemcpyFromSymbol(out16, g_cl_stats, 16 * sizeof(unsigned long long)));
    if (reset) { const unsigned long long z[16] = {0}; NRPN_CUDA_TRY(cudaMemcpyToSymbol(g_cl_stats, z, sizeof(z))); }
    return NRPN_OK;
}

int nrpn_iou3d_pairs(const float* a, const float* b, int n, int box_dim, float* iou, nrpn_stream_t stream) {
    if (n < 0 || (box_dim != 6 && box_dim != 7)) return NRPN_ERR_INVALID;
    if (n == 0) return NRPN_OK;
    if (!a || !b || !iou) return NRPN_ERR_INVALID;
    iou_pairs_kernel<<<ceil_div(n, 128), 128, 0, (cudaStream_t)stream>>>(a, b, n, box_dim, iou);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

int nrpn_iou3d_pairs_verbose(const float* a, const float* b, int n, float* iou, float* corners1, float* corners2, float* z_range, float* u3d,
                             nrpn_stream_t stream) {
    if (n < 0) return NRPN_ERR_INVALID;
    if (n == 0) return NRPN_OK;
    if (!a || !b || !iou || !corners1 || !corners2 || !z_range || !u3d) return NRPN_ERR_INVALID;
    iou_pairs_verbose_kernel<<<ceil_div(n, 128), 128, 0, (cudaStream_t)stream>>>(a, b, n, iou, corners1, corners2, z_range, u3d);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

int nrpn_iou3d_pairs_backward(const float* a, const float* b, int n, const float* grad_iou, const float* grad_u3d, float* grad_a, float* grad_b,
                              nrpn_stream_t stream) {
    if (n < 0) return NRPN_ERR_INVALID;
    if (n == 0) return NRPN_OK;
    if (!a || !b || !grad_a || !grad_b || (!grad_iou && !grad_u3d)) return NRPN_ERR_INVALID;
    iou_pairs_grad_kernel<<<ceil_div(n * 14, 128), 128, 0, (cudaStream_t)stream>>>(a, b, n, grad_iou, grad_u3d, grad_a, grad_b);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

int nrpn_iou3d_matrix(const float* a, int n, const float* b, int m, int box_dim, float* out, nrpn_stream_t stream) {
    if (n < 0 || m < 0 || (box_dim != 6 && box_dim != 7)) return NRPN_ERR_INVALID;
    if (n == 0 || m == 0) return NRPN_OK;
    if (!a || !b || !out) return NRPN_ERR_INVALID;
    dim3 grid(ceil_div(m, 32), ceil_div(n, 8));
    if (grid.y > 65535) return NRPN_ERR_UNSUPPORTED;
    iou_matrix_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a, n, b, m, box_dim, out);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

int nrpn_sort_vertices(const float* vertices, const uint8_t* mask, const int32_t* num_valid, int b, int n, int m,
                       int32_t* idx, nrpn_stream_t stream) {
    if (b < 0 || n < 0 || m < 9 || m > 32) return NRPN_ERR_INVALID;
    const long total = (long)b * n;
    if (total == 0) return NRPN_OK;
    if (!vertices || !mask || !num_valid || !idx) return NRPN_ERR_INVALID;
    sort_vertices_kernel<<<(unsigned)ceil_div(total, 128L), 128, 0, (cudaStream_t)stream>>>(vertices, mask, num_valid, total, m, idx);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

static int g_iou_mode_host = 3;
int nrpn_set_iou_mode(int mode) {
    if (mode < 0 || mode > 3) return NRPN_ERR_INVALID;
    NRPN_CUDA_TRY(cudaMemcpyToSymbol(nrpn::g_iou_mode, &mode, sizeof(int)));
    g_iou_mode_host = mode;
    return NRPN_OK;
}
int nrpn_get_iou_mode(void) { return g_iou_mode_host; }

int nrpn_nms_max_boxes(void) { return kNmsMaxBoxes; }

size_t nrpn_nms_workspace_bytes(int n) { return nms_workspace_bytes(n); }

int nrpn_nms(const float* boxes, int box_dim, const float* scores, const int32_t* group, int n, float thr, int64_t* keep,
             int32_t* n_keep, void* workspace, size_t workspace_bytes, nrpn_stream_t stream) {
    if (n < 0 || (box_dim != 6 && box_dim != 7) || !n_keep) return NRPN_ERR_INVALID;
    if (n > 0 && (!boxes || !scores || !keep || !workspace)) return NRPN_ERR_INVALID;
    return nms_run(boxes, box_dim, scores, group, n, thr, /*ignore_group=*/-1, keep, n_keep, workspace, workspace_bytes,
                   (cudaStream_t)stream);
}

#pragma GCC visibility pop
}  // extern "C"
