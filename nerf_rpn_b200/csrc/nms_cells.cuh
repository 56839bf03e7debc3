// Cell-list greedy NMS for tens of thousands to millions of boxes (BASELINE config 5: utils.py:215-265 at 1 k .. 1 M proposals).
// Included by nms.cu inside namespace nrpn (uses its prepared records and culls).
//
// The greedy loop "keep the best remaining box, drop what it overlaps" decides box i from the boxes j that score higher AND overlap it:
//     i is dropped  <=>  some such j is kept.
// That is a dependency graph, not a sequence.  This path resolves it without walking the boxes one chunk after another:
//   * boxes are sorted by score once (position = rank; groups only filter pairs) and assigned to the cells of a uniform grid per volume
//     class (BinGrid, below);
//   * positions are processed in a handful of LEVELS [b, e) of geometrically growing size.  Per level
//       (1) cross:      every box of the level is tested against the KEPT boxes of the earlier levels (early exit on the first hit);
//       (2) adjacency:  the survivors are tested against each other; hits (j before i) go to a short per-box list;
//       (3) rounds:     a survivor with a kept predecessor is dropped, one whose predecessors are all dropped is kept -- repeated
//                       until nothing is undecided (the earliest undecided box always resolves, so it terminates; random scores give
//                       chains of a dozen rounds).
//   * (1) and (2) are the same kernel: a CTA takes one grid cell's boxes as queries (in shared memory), streams the records of the cells
//     their circles / z ranges can reach -- stored cell by cell, so a window row is one contiguous range -- one record per thread, and
//     every thread loops over the queries: cheap necessary conditions first, the exact polygon clip only on full warps of queued pairs.
// Every decision is the exact IoU of the sequential loop (same operand order), so the keep set is the reference's bit for bit; the
// chunked path stays as the fallback for what this path declines (adjacency overflow, round cap, thr < 0, stream capture).

// ---- the grid
// Whether box j can suppress box k is bounded by two necessary conditions that can be INDEXED: (a) their volumes are within a factor 1 / thr_m
// of each other (IoU <= min V / max V), (b) their bounding circles and z ranges intersect.  Boxes are therefore filed in a uniform grid per
// volume class -- class width log2(1 / thr_m), so partners sit in the same or an adjacent class; cells half of the class's largest diameter /
// depth -- and a box only visits the cells its circle and z range can reach in its three classes.  Every candidate still goes through the
// same culls and exact polygon clip.
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

__device__ __forceinline__ float ordered_to_float(unsigned u) { return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u); }
__device__ __forceinline__ int bin_clampi(int v, int n) { return v < 0 ? 0 : (v >= n ? n - 1 : v); }

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

// cell of every box (kBinCells - 1 = the "everywhere" cell of boxes without a usable cull record)
__global__ void nms_bin_assign_kernel(const float* __restrict__ prep, int n, const BinGrid* __restrict__ g, int* __restrict__ box_cell) {
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
}

// ---- the cell lists
constexpr int kAdjSlots = 32;             // inline predecessors per box; more -> fallback
constexpr int kQB = 256;                  // queries per work item
constexpr int kPairThreads = 256;
constexpr int kMaxRows = 2048;            // window rows per item: <= 3 classes x 32 x 16 + 1
constexpr int kLevel0 = 8192, kLevelGrowth = 4;
constexpr int kRoundBatch = 8, kRoundCap = 4096;
constexpr int kScanTile = 1024;
constexpr int kScanBlocks = (kBinCells + kScanTile - 1) / kScanTile;
enum : signed char { ST_UNDECIDED = 0, ST_KEPT = 1, ST_REMOVED = 2 };

struct CellIndex {
    int* start;          // kBinCells + 1: first record of every cell
    int* cursor;         // kBinCells: scratch counters (zero between builds)
    float4* recs;        // 3 float4 per record: cull tail (8 floats), {position, group, -, -}
    int* item_start;     // kBinCells + 1 (query index only): first work item of every cell
    int2* items;         // (cell, batch of kQB queries)
};

__global__ void cl_state_init_kernel(const int* __restrict__ sgroup, int n, int ignore_group, signed char* __restrict__ state, int* __restrict__ adj_cnt) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    state[p] = sgroup[p] == ignore_group ? ST_REMOVED : ST_UNDECIDED;
    adj_cnt[p] = 0;
}

__global__ void cl_count_kernel(const signed char* __restrict__ state, const int* __restrict__ box_cell, int b, int e, int want, int* __restrict__ cursor) {
    const int p = b + blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= e || state[p] != want) return;
    atomicAdd(&cursor[box_cell[p]], 1);
}

// block-local exclusive scan of (records, work items) per cell, packed as (items << 32 | records); block totals -> totals[]
__global__ void __launch_bounds__(kScanTile) cl_scan_local_kernel(const int* __restrict__ cnt, int* __restrict__ start, int* __restrict__ item_start,
                                                                  unsigned long long* __restrict__ totals) {
    __shared__ unsigned long long wtot[32];
    const int t = threadIdx.x, cell = blockIdx.x * kScanTile + t, lane = t & 31, wid = t >> 5;
    const int c = cell < kBinCells ? cnt[cell] : 0;
    const unsigned long long v = ((unsigned long long)((c + kQB - 1) / kQB) << 32) | (unsigned long long)c;
    unsigned long long s = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned long long u = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += u; }
    if (lane == 31) wtot[wid] = s;
    __syncthreads();
    if (wid == 0) {
        unsigned long long w = wtot[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const unsigned long long u = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += u; }
        wtot[lane] = w;
    }
    __syncthreads();
    const unsigned long long ex = s - v + (wid ? wtot[wid - 1] : 0ull);
    if (cell < kBinCells) { start[cell] = (int)(ex & 0xffffffffull); item_start[cell] = (int)(ex >> 32); }
    if (t == kScanTile - 1) totals[blockIdx.x] = wtot[31];
}

// adds the totals of the preceding blocks; the last block writes the end markers; meta[0] = work counter of the next pairs launch
__global__ void __launch_bounds__(kScanTile) cl_scan_add_kernel(int* __restrict__ start, int* __restrict__ item_start,
                                                                const unsigned long long* __restrict__ totals, int* __restrict__ meta) {
    __shared__ unsigned long long red[32];
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
    unsigned long long s = 0;
    for (int k = t; k < (int)blockIdx.x; k += kScanTile) s += totals[k];
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) red[wid] = s;
    __syncthreads();
    unsigned long long off = 0;
    for (int k = 0; k < 32; ++k) off += red[k];
    const int cell = blockIdx.x * kScanTile + t;
    if (cell < kBinCells) { start[cell] += (int)(off & 0xffffffffull); item_start[cell] += (int)(off >> 32); }
    if (blockIdx.x == kScanBlocks - 1 && t == 0) {
        const unsigned long long all = off + totals[kScanBlocks - 1];
        start[kBinCells] = (int)(all & 0xffffffffull);
        item_start[kBinCells] = (int)(all >> 32);
        meta[0] = 0;
    }
}

__global__ void cl_items_kernel(const int* __restrict__ item_start, int2* __restrict__ items) {
    const int cell = blockIdx.x * blockDim.x + threadIdx.x;
    if (cell >= kBinCells) return;
    const int b = item_start[cell], e = item_start[cell + 1];
    for (int k = b; k < e; ++k) items[k] = make_int2(cell, k - b);
}

__global__ void cl_scatter_kernel(const signed char* __restrict__ state, const int* __restrict__ box_cell, const float* __restrict__ prep,
                                  const int* __restrict__ sgroup, int b, int e, int want, const int* __restrict__ start, int* __restrict__ cursor,
                                  float4* __restrict__ recs) {
    const int p = b + blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= e || state[p] != want) return;
    const int cell = box_cell[p];
    const int slot = start[cell] + atomicSub(&cursor[cell], 1) - 1;          // the counters return to zero for the next build
    const float4* t = reinterpret_cast<const float4*>(prep + (size_t)p * kPrepFloats + 8);
    float4* r = recs + (size_t)slot * 3;
    r[0] = t[0]; r[1] = t[1];
    r[2] = make_float4(__int_as_float(p), __int_as_float(sgroup[p]), 0.f, 0.f);
}

// diagnostics (nrpn_nms_cells_stats): [0] records streamed, [1] pair slots (records x queries of the item, before the group / order / already-dropped filters), [2] exact IoU evaluations, [3] hits,
// [4] work items; per mode: +0 cross, +8 adjacency
static __device__ unsigned long long g_cl_stats[16];

// obb_surely_not_above (box_iou.cuh) on two cull records held in registers / shared memory as float4 pairs {area, vol, zmin, zmax}, {cx, cy, rad,
// cullable}: the same tests in the same order, written on scalars so that nothing is addressed through a pointer (the pointer form put both
// records in local memory inside the pair loop: 16 G local-load sectors in one pass at 1 M boxes, profiles/r02_nms_cells_ncu.md).
__device__ __forceinline__ bool cl_needs_exact(const float4 a0, const float4 a1, const float4 b0, const float4 b1, const float thr_m) {
    if (!(__float_as_int(a1.w) && __float_as_int(b1.w))) return true;
    const float dx = a1.x - b1.x, dy = a1.y - b1.y, rr = a1.z + b1.z;
    const float d2 = dx * dx + dy * dy;
    if (d2 > rr * rr) return false;
    const float oz = fminf(a0.w, b0.w) - fmaxf(a0.z, b0.z);
    if (!(oz >= 0.0f)) return false;
    if (thr_m > 0.0f) {
        const float vmax = fmaxf(a0.y, b0.y);
        if (fminf(a0.y, b0.y) <= thr_m * vmax) return false;
        if (oz <= thr_m * fmaxf(a0.w - a0.z, b0.w - b0.z)) return false;
        const float lens = 2.0f * fminf(a1.z, b1.z) * (rr - sqrtf(d2));
        if (NRPN_LENS_CULL && fminf(fminf(a0.x, b0.x), lens) * oz <= thr_m * vmax) return false;
    }
    return true;
}

// obb_footprints_surely_disjoint (box_iou.cuh) straight on two prepared records (16 floats: 8 corner coordinates, area, vol, zmin, zmax, cx, cy, rad,
// cullable): the second filter stage, run on full warps of queued pairs before the exact clip
__device__ __forceinline__ bool cl_sat_disjoint(const float* __restrict__ pa, const float* __restrict__ pb) {
    ObbPrep a, b;
    const float4 a0 = __ldg(reinterpret_cast<const float4*>(pa)), a1 = __ldg(reinterpret_cast<const float4*>(pa) + 1), a3 = __ldg(reinterpret_cast<const float4*>(pa) + 3);
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(pb)), b1 = __ldg(reinterpret_cast<const float4*>(pb) + 1), b3 = __ldg(reinterpret_cast<const float4*>(pb) + 3);
    a.c[0] = a0.x; a.c[1] = a0.y; a.c[2] = a0.z; a.c[3] = a0.w; a.c[4] = a1.x; a.c[5] = a1.y; a.c[6] = a1.z; a.c[7] = a1.w;
    b.c[0] = b0.x; b.c[1] = b0.y; b.c[2] = b0.z; b.c[3] = b0.w; b.c[4] = b1.x; b.c[5] = b1.y; b.c[6] = b1.z; b.c[7] = b1.w;
    a.cx = a3.x; a.cy = a3.y; a.rad = a3.z; a.cullable = __float_as_int(a3.w);
    b.cx = b3.x; b.cy = b3.y; b.rad = b3.z; b.cullable = __float_as_int(b3.w);
    return obb_footprints_surely_disjoint(a, b);
}

// the decision of the sequential loop for one pair: a = the higher-scored ("picked") box, b = the candidate (operand order matters: the reference's
// vertex sort is not symmetric).  Kept out of line so that the polygon clip's registers and stack stay out of the pair loop.
__device__ __noinline__ bool cl_exact(const float* __restrict__ prep, int box_dim, float thr, int pj, int pq) {
    const float* ap = prep + (size_t)pj * kPrepFloats;
    const float* bp = prep + (size_t)pq * kPrepFloats;
    if (box_dim == 7) { ObbPrep a, b; load_prep(ap, a); load_prep(bp, b); return !(iou3d_obb_full(a, b) <= thr); }      // the SAT stage ran before
    float aa[6], bb[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) { aa[i] = ap[i]; bb[i] = bp[i]; }
    return !(iou3d_aabb(aa, bb) <= thr);
}

struct PairArgs {
    const float* prep; int box_dim; float thr, thr_m;
    const BinGrid* grid;
    const int* qstart; const float4* qrecs; const int* item_start; const int2* items; int* work;
    const int* rstart; const float4* rrecs;
    signed char* state; int* adj_cnt; int* adj; int* fail;
};

// MODE 0 = cross (records: kept boxes of earlier levels; a hit drops the query), MODE 1 = adjacency (records == queries' own index; a hit with
// j before i is appended to i's predecessor list)
template <int MODE>
__global__ void __launch_bounds__(kPairThreads, 2) cl_pairs_kernel(const PairArgs A) {
    __shared__ float4 q_t0[kQB], q_t1[kQB];
    __shared__ int q_pos[kQB], q_grp[kQB], q_dead[kQB];
    __shared__ int r_beg[kMaxRows], r_pre[kMaxRows + 1];
    __shared__ int2 queue[kPairThreads / 32][64];        // stage 1: survivors of the cheap necessary conditions
    __shared__ int2 queue2[kPairThreads / 32][64];       // stage 2: survivors of the separating-axis test, waiting for the exact clip
    __shared__ int s_item, s_dead, s_scan[kPairThreads], s_win[3][6];
    const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31;
    const BinGrid& G = *A.grid;
    const int n_items = A.item_start[kBinCells];
    const float thr = A.thr, thr_m = A.thr_m;
    const int box_dim = A.box_dim;
    const float* __restrict__ prep = A.prep;

    auto exact = [&](int pj, int pq) -> bool { return cl_exact(prep, box_dim, thr, pj, pq); };
    auto on_hit = [&](int q, int pj) {
        if (MODE == 0) {
            if (atomicExch(&q_dead[q], 1) == 0) atomicAdd(&s_dead, 1);
        } else {
            const int pq = q_pos[q];
            const int slot = atomicAdd(&A.adj_cnt[pq], 1);
            if (slot < kAdjSlots) A.adj[(size_t)pq * kAdjSlots + slot] = pj;
            else *A.fail = 1;
        }
    };

    unsigned long long st_rec = 0, st_pair = 0, st_exact = 0, st_hit = 0, st_item = 0;
    for (;;) {
        __syncthreads();
        if (tid == 0) { s_item = atomicAdd(A.work, 1); s_dead = 0; }
        __syncthreads();
        const int item = s_item;
        if (item >= n_items) break;
        if (tid == 0) ++st_item;
        const int2 it = A.items[item];
        const int cell = it.x;
        const int qb = A.qstart[cell] + it.y * kQB;
        const int nq = min(kQB, A.qstart[cell + 1] - qb);
        if (tid < nq) {
            const float4* r = A.qrecs + (size_t)(qb + tid) * 3;
            q_t0[tid] = __ldg(r); q_t1[tid] = __ldg(r + 1);
            const float4 r2 = __ldg(r + 2);
            q_pos[tid] = __float_as_int(r2.x); q_grp[tid] = __float_as_int(r2.y); q_dead[tid] = 0;
        }
        // ---- window rows of this cell: contiguous record ranges [beg, beg + len)
        int nrows;
        if (cell == kBinCells - 1) {                       // boxes without a usable cull record: against everything
            nrows = 1;
            if (tid == 0) { r_beg[0] = 0; r_pre[0] = A.rstart[kBinCells]; }
        } else {
            const int c = cell / kBinCellsPerClass, rem = cell - c * kBinCellsPerClass;
            const int hx = rem % kBinMaxXY, hy = (rem / kBinMaxXY) % kBinMaxXY, hz = rem / (kBinMaxXY * kBinMaxXY);
            const float big = 3.0e38f;
            const float lox = hx == 0 ? -big : G.x0 + (float)hx * G.S[c], hix = hx == G.nx[c] - 1 ? big : G.x0 + (float)(hx + 1) * G.S[c];
            const float loy = hy == 0 ? -big : G.y0 + (float)hy * G.S[c], hiy = hy == G.ny[c] - 1 ? big : G.y0 + (float)(hy + 1) * G.S[c];
            const float loz = hz == 0 ? -big : G.z0 + (float)hz * G.Sz[c], hiz = hz == G.nz[c] - 1 ? big : G.z0 + (float)(hz + 1) * G.Sz[c];
            // per neighbour class (c - 1, c, c + 1): the cells the queries' circles / z ranges can reach -> s_win[ci] = {rows, wy, ix0, ix1, iy0, iz0}
            if (tid < 3) {
                const int ci = tid, cc = c - 1 + ci;
                int rows = 0, wy = 1, x0 = 0, x1 = 0, y0 = 0, z0 = 0;
                if (cc >= 0 && cc < G.n_cls) {
                    const float R = (G.rmax[c] + G.rmax[cc]) * 1.0005f + 1e-3f, Rz = 0.5f * (G.dmax[c] + G.dmax[cc]) * 1.0005f + 1e-3f;
                    const float S = G.S[cc], Sz = G.Sz[cc];
                    x0 = bin_clampi((int)floorf(fmaxf((lox - R - G.x0) / S, -1.0f)), G.nx[cc]);
                    x1 = bin_clampi((int)floorf(fminf((hix + R - G.x0) / S, 1.0e6f)), G.nx[cc]);
                    y0 = bin_clampi((int)floorf(fmaxf((loy - R - G.y0) / S, -1.0f)), G.ny[cc]);
                    const int y1 = bin_clampi((int)floorf(fminf((hiy + R - G.y0) / S, 1.0e6f)), G.ny[cc]);
                    z0 = bin_clampi((int)floorf(fmaxf((loz - Rz - G.z0) / Sz, -1.0f)), G.nz[cc]);
                    const int z1 = bin_clampi((int)floorf(fminf((hiz + Rz - G.z0) / Sz, 1.0e6f)), G.nz[cc]);
                    wy = y1 - y0 + 1;
                    rows = wy * (z1 - z0 + 1);
                }
                s_win[ci][0] = rows; s_win[ci][1] = wy; s_win[ci][2] = x0; s_win[ci][3] = x1; s_win[ci][4] = y0; s_win[ci][5] = z0;
            }
            __syncthreads();
            const int rows0 = s_win[0][0], rows1 = s_win[1][0], rows2 = s_win[2][0];
            const int off1 = rows0, off2 = rows0 + rows1, off3 = off2 + rows2;
            nrows = off3 + 1;                              // + the "everywhere" cell
            for (int r = tid; r < nrows; r += kPairThreads) {
                int beg, end;
                if (r == off3) { beg = A.rstart[kBinCells - 1]; end = A.rstart[kBinCells]; }
                else {
                    const int ci = r >= off2 ? 2 : (r >= off1 ? 1 : 0);
                    const int local = r - (ci == 2 ? off2 : (ci == 1 ? off1 : 0));
                    const int wy = s_win[ci][1], iy = s_win[ci][4] + local % wy, iz = s_win[ci][5] + local / wy;
                    const int base = (c - 1 + ci) * kBinCellsPerClass + (iz * kBinMaxXY + iy) * kBinMaxXY;
                    beg = A.rstart[base + s_win[ci][2]]; end = A.rstart[base + s_win[ci][3] + 1];
                }
                r_beg[r] = beg; r_pre[r] = end - beg;
            }
        }
        __syncthreads();
        // ---- exclusive scan of the row lengths (8 per thread)
        {
            int loc[kMaxRows / kPairThreads], s = 0;
#pragma unroll
            for (int k = 0; k < kMaxRows / kPairThreads; ++k) { const int r = tid * (kMaxRows / kPairThreads) + k; loc[k] = r < nrows ? r_pre[r] : 0; s += loc[k]; }
            s_scan[tid] = s;
            __syncthreads();
            for (int o = 1; o < kPairThreads; o <<= 1) { const int v = tid >= o ? s_scan[tid - o] : 0; __syncthreads(); s_scan[tid] += v; __syncthreads(); }
            int run = s_scan[tid] - s;
#pragma unroll
            for (int k = 0; k < kMaxRows / kPairThreads; ++k) { const int r = tid * (kMaxRows / kPairThreads) + k; if (r < nrows) r_pre[r] = run; run += loc[k]; }
            if (tid == kPairThreads - 1) r_pre[nrows] = s_scan[tid];
            __syncthreads();
        }
        const int total = r_pre[nrows];
        // ---- stream the records: one per thread and step; warps run independently from here
        int qn = 0, qn2 = 0;
        const bool obb = box_dim == 7 && thr >= 0.0f;
        auto drain2 = [&](int count) {                       // exact clip on the first `count` (<= 32) entries of stage 2
            if (lane < count) {
                const int2 e = queue2[wid][lane];
                if (!(MODE == 0 && *(volatile int*)&q_dead[e.x])) { ++st_exact; if (exact(e.y, q_pos[e.x])) { on_hit(e.x, e.y); ++st_hit; } }
            }
            __syncwarp();
            const int rest = qn2 - count;
            const int2 moved = lane < rest ? queue2[wid][count + lane] : make_int2(0, 0);
            __syncwarp();
            if (lane < rest) queue2[wid][lane] = moved;
            qn2 = rest;
            __syncwarp();
        };
        auto drain1 = [&](int count) {                       // separating-axis test on the first `count` (<= 32) entries of stage 1 -> stage 2
            bool keep = false;
            int2 e = make_int2(0, 0);
            if (lane < count) {
                e = queue[wid][lane];
                keep = !(MODE == 0 && *(volatile int*)&q_dead[e.x]);
                if (keep && obb) keep = !cl_sat_disjoint(prep + (size_t)e.y * kPrepFloats, prep + (size_t)q_pos[e.x] * kPrepFloats);
            }
            const unsigned m = __ballot_sync(0xffffffffu, keep);
            if (keep) queue2[wid][qn2 + __popc(m & ((1u << lane) - 1u))] = e;
            qn2 += __popc(m);
            const int rest = qn - count;
            const int2 moved = lane < rest ? queue[wid][count + lane] : make_int2(0, 0);
            __syncwarp();
            if (lane < rest) queue[wid][lane] = moved;
            qn = rest;
            __syncwarp();
            if (qn2 >= 32) drain2(32);
        };
        for (int base = 0; base < total; base += kPairThreads) {
            if (MODE == 0 && *(volatile int*)&s_dead >= nq) break;
            const int gidx = base + tid;
            const bool have = gidx < total;
            float4 t0 = make_float4(0.f, 0.f, 0.f, 0.f), t1 = t0;
            int pj = 0, gj = -1;
            if (have) {
                int lo = 0, hi = nrows;                     // largest row with r_pre[row] <= gidx
                while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (r_pre[mid] <= gidx) lo = mid; else hi = mid; }
                const float4* r = A.rrecs + (size_t)(r_beg[lo] + gidx - r_pre[lo]) * 3;
                t0 = __ldg(r); t1 = __ldg(r + 1);
                const float4 r2 = __ldg(r + 2);
                pj = __float_as_int(r2.x); gj = __float_as_int(r2.y);
            }
            if (!__any_sync(0xffffffffu, have)) continue;
            st_rec += have; st_pair += have ? nq : 0;
            for (int q = 0; q < nq; ++q) {
                if (MODE == 0 && *(volatile int*)&q_dead[q]) continue;
                bool c = false;
                if (have && gj == q_grp[q] && (MODE == 0 || pj < q_pos[q])) {
                    c = cl_needs_exact(t0, t1, q_t0[q], q_t1[q], thr_m);
                }
                const unsigned m = __ballot_sync(0xffffffffu, c);
                if (!m) continue;
                if (c) queue[wid][qn + __popc(m & ((1u << lane) - 1u))] = make_int2(q, pj);
                qn += __popc(m);
                __syncwarp();
                if (qn >= 32) drain1(32);
            }
        }
        if (qn > 0) drain1(qn);
        if (qn2 > 0) drain2(qn2);
        if (MODE == 0) {
            __syncthreads();
            if (tid < nq && q_dead[tid]) A.state[q_pos[tid]] = ST_REMOVED;
        }
    }
    {   // one atomic per warp and counter
        unsigned long long v[5] = {st_rec, st_pair, st_exact, st_hit, st_item};
#pragma unroll
        for (int k = 0; k < 5; ++k) {
#pragma unroll
            for (int o = 16; o; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
            if (lane == 0 && v[k]) atomicAdd(&g_cl_stats[MODE * 8 + k], v[k]);
        }
    }
}

// one round of the dependency resolution over the level's survivors (records of the level index); und[r] counts what stays undecided
__global__ void cl_round_kernel(const float4* __restrict__ recs, const int* __restrict__ start, const int* __restrict__ adj_cnt, const int* __restrict__ adj,
                                signed char* __restrict__ state, int* __restrict__ und, int round) {
    if (round > 0 && und[round - 1] == 0) return;
    const int total = start[kBinCells];
    int mine = 0;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
        const int p = __float_as_int(__ldg(&recs[(size_t)e * 3 + 2]).x);
        volatile signed char* vs = state;
        if (vs[p] != ST_UNDECIDED) continue;
        const int cnt = min(adj_cnt[p], kAdjSlots);
        bool done = false;
        for (int attempt = 0; attempt < 4 && !done; ++attempt) {      // neighbours decided a moment ago (same launch) unblock this one right away
            bool kept_pred = false, open = false;
            for (int k = 0; k < cnt; ++k) {
                const signed char s = vs[adj[(size_t)p * kAdjSlots + k]];
                kept_pred = kept_pred || s == ST_KEPT;
                open = open || s == ST_UNDECIDED;
            }
            if (kept_pred) { vs[p] = ST_REMOVED; done = true; }
            else if (!open) { vs[p] = ST_KEPT; done = true; }
        }
        if (!done) ++mine;
    }
    mine = __reduce_add_sync(0xffffffffu, mine);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(&und[round], mine);
}

// ---- ordered compaction of the kept positions into original indices
__global__ void __launch_bounds__(1024) cl_keep_count_kernel(const signed char* __restrict__ state, int n, int* __restrict__ blk) {
    const int p = blockIdx.x * 1024 + threadIdx.x;
    const int c = __syncthreads_count(p < n && state[p] == ST_KEPT);
    if (threadIdx.x == 0) blk[blockIdx.x] = c;
}
__global__ void __launch_bounds__(1024) cl_keep_scan_kernel(int* __restrict__ blk, int nblk, int32_t* __restrict__ n_keep) {
    __shared__ int part[1024];
    const int t = threadIdx.x;
    const int per = (nblk + 1023) / 1024;
    int s = 0;
    for (int i = t * per; i < min(nblk, t * per + per); ++i) s += blk[i];
    part[t] = s;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) { const int v = t >= o ? part[t - o] : 0; __syncthreads(); part[t] += v; __syncthreads(); }
    int run = part[t] - s;
    for (int i = t * per; i < min(nblk, t * per + per); ++i) { const int c = blk[i]; blk[i] = run; run += c; }
    if (t == 1023) *n_keep = part[1023];
}
__global__ void __launch_bounds__(1024) cl_keep_emit_kernel(const signed char* __restrict__ state, const unsigned long long* __restrict__ keys, int n,
                                                            const int* __restrict__ blk, int64_t* __restrict__ keep) {
    __shared__ int wcnt[32];
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
    const int p = blockIdx.x * 1024 + t;
    const bool k = p < n && state[p] == ST_KEPT;
    const unsigned m = __ballot_sync(0xffffffffu, k);
    if (lane == 0) wcnt[wid] = __popc(m);
    __syncthreads();
    int off = blk[blockIdx.x];
    for (int w = 0; w < wid; ++w) off += wcnt[w];
    if (k) keep[off + __popc(m & ((1u << lane) - 1u))] = (int64_t)(keys[p] & 0xFFFFFFull);
}

struct CellWs {
    BinGrid* grid;       // grid parameters
    unsigned* bstats;    // kBinStatWords: reduction scratch of the grid (ordered-uint min / max)
    int* box_cell;       // n: cell of every box
    signed char* state; int* adj_cnt; int* adj;
    CellIndex A, B;
    unsigned long long* totals; int* meta; int* und; int* fail; int* blk;
};

// the grid of the n prepared records: extents -> volume classes -> per-class cell sizes -> cell of every box
static int cl_build_grid(const CellWs& c, const float* prep, int n, float thr_m, cudaStream_t st) {
    nms_bin_stats_init_kernel<<<1, 64, 0, st>>>(c.bstats);
    nms_bin_stats_kernel<<<ceil_div(n, 256), 256, 0, st>>>(prep, n, 0, c.grid, c.bstats);
    nms_bin_grid_kernel<<<1, 32, 0, st>>>(c.bstats, thr_m, 0, c.grid);
    nms_bin_stats_kernel<<<ceil_div(n, 256), 256, 0, st>>>(prep, n, 1, c.grid, c.bstats);
    nms_bin_grid_kernel<<<1, 32, 0, st>>>(c.bstats, thr_m, 1, c.grid);
    NRPN_LAUNCH_CHECK();
    nms_bin_assign_kernel<<<ceil_div(n, 256), 256, 0, st>>>(prep, n, c.grid, c.box_cell);
    NRPN_LAUNCH_CHECK();
    return NRPN_OK;
}

static void cl_build_index(const CellIndex& X, const CellWs& c, const NmsWs& w, int b, int e, int want, bool with_items, cudaStream_t st) {
    if (e > b) cl_count_kernel<<<ceil_div(e - b, 256), 256, 0, st>>>(c.state, c.box_cell, b, e, want, X.cursor);
    cl_scan_local_kernel<<<kScanBlocks, kScanTile, 0, st>>>(X.cursor, X.start, X.item_start, c.totals);
    cl_scan_add_kernel<<<kScanBlocks, kScanTile, 0, st>>>(X.start, X.item_start, c.totals, c.meta);
    if (with_items) cl_items_kernel<<<ceil_div(kBinCells, 256), 256, 0, st>>>(X.item_start, X.items);
    if (e > b) cl_scatter_kernel<<<ceil_div(e - b, 256), 256, 0, st>>>(c.state, c.box_cell, w.prep, w.sgroup, b, e, want, X.start, X.cursor, X.recs);
}
