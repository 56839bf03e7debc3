// Device functions for 3-D box overlap -- the fused replacement of the reference's ~40-kernel ATen chain
// plus its native vertex sort:
//   oriented_iou_loss.py:6-57,82-107, box_intersection_2d.py:11-176, cuda_op/sort_vert_kernel.cu:15-134,
//   utils.py:418-458 (axis-aligned).
// One thread evaluates one pair entirely in registers; nothing (24-vertex arrays, masks, sort indices)
// is materialised in HBM.
//
// Arithmetic contract: every fp32 operation is an explicitly rounded intrinsic in the reference's operation order.  Three steps
// of the reference chain round differently on its CPU and CUDA builds; NRPN_IOU_MODE selects which build is reproduced
// (measured on the GPU against the unmodified reference + its own K1 binary: tools/ref_gpu_probe.py):
//   bit 0 (operation order of the torch-CUDA kernels): box2corners_th's 4x2 * 2x2 torch.bmm = fma(y4, r1, x4 * r0); torch.sum over
//         the 24 masked vertices = four interleaved accumulators, ((a0 + a1) + a2) + a3; torch.sum over the 8 shoelace terms =
//         (t0+t4 + t2+t6) + (t1+t5 + t3+t7).  Mode bit clear: separately rounded mul/mul/add and left-to-right sums, the order of
//         oracle/box_oracle.c's default (== the reference's CPU build on the golden vectors).
//   bit 1 (libm): sin / cos through CUDA's sinf / cosf like ATen's CUDA kernels; clear: fp64 sin / cos rounded once (oracle).
// The library default is 3 = "what the reference computes on this GPU" (nrpn_set_iou_mode); tests against the CPU oracle use 0.
// Independent of the mode, K1's pseudo-angle denominator is fma(x, x, y * y): that is what nvcc makes of `x1*x1 + y1*y1` in the
// reference's sort_vert_kernel.cu:25 (SASS of its own build: FMUL y*y; FFMA x*x + .).
#pragma once
#ifndef NRPN_SKIP_COMMON
#include "common.cuh"
#endif
#ifndef NRPN_IOU_MODE
#define NRPN_IOU_MODE 3
#endif

namespace nrpn {

// smallest fp32 >= 1e-8 (EPSILON in the reference is the double 1e-8; comparisons of an fp32 value v
// against it satisfy  v < 1e-8 <=> v < kEpsUp  and  v > 1e-8 <=> v >= kEpsUp).
__device__ __forceinline__ float eps_up() { return __uint_as_float(0x322BCC78u); }   // 1.000000082740371e-08, first fp32 above 1e-8
__device__ __forceinline__ float eps_f()  { return __uint_as_float(0x322BCC77u); }   // (float)1e-8 = 9.99999993922529e-09

struct ObbPrep {          // per-box derived data, computed once per box
    float c[8];           // corners (x0,y0,...,x3,y3)   box2corners_th
    float area;           // w*h
    float vol;            // (w*h)*d
    float zmin, zmax;
    float cx, cy, rad;    // conservative bounding circle for exact-zero culling
    int cullable;         // 1 when w,h,d are positive and everything is finite
};

__device__ __forceinline__ void obb_prepare(const float* __restrict__ b, ObbPrep& p) {
    const float x = b[0], y = b[1], z = b[2], w = b[3], h = b[4], d = b[5], alpha = b[6];
    const int mode = NRPN_IOU_MODE;
    float s, co;
    if (mode & 2) { s = sinf(alpha); co = cosf(alpha); }
    else { s = (float)sin((double)alpha); co = (float)cos((double)alpha); }
    const float ns = -s;
    const float sx[4] = {0.5f, -0.5f, -0.5f, 0.5f};
    const float sy[4] = {0.5f, 0.5f, -0.5f, -0.5f};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float x4 = __fmul_rn(sx[i], w);
        const float y4 = __fmul_rn(sy[i], h);
        float rx, ry;
        if (mode & 1) { rx = __fmaf_rn(y4, ns, __fmul_rn(x4, co)); ry = __fmaf_rn(y4, co, __fmul_rn(x4, s)); }
        else { rx = __fadd_rn(__fmul_rn(x4, co), __fmul_rn(y4, ns)); ry = __fadd_rn(__fmul_rn(x4, s), __fmul_rn(y4, co)); }
        p.c[2 * i] = __fadd_rn(rx, x);
        p.c[2 * i + 1] = __fadd_rn(ry, y);
    }
    p.area = __fmul_rn(w, h);
    p.vol = __fmul_rn(p.area, d);
    const float hd = __fmul_rn(d, 0.5f);
    p.zmax = __fadd_rn(z, hd);
    p.zmin = __fsub_rn(z, hd);
    p.cx = x; p.cy = y;
    p.rad = 0.5f * sqrtf(w * w + h * h) * 1.001f + 1e-3f;
    const bool fin = isfinite(x) && isfinite(y) && isfinite(z) && isfinite(w) && isfinite(h) && isfinite(d) && isfinite(alpha);
    p.cullable = (fin && w > 0.f && h > 0.f && d > 0.f) ? 1 : 0;
}

// compare_vertices (sort_vert_kernel.cu:15-40) on pre-computed pseudo-angles q = |x|*x / (x*x + y*y + eps).
__device__ __forceinline__ bool vert_less(float x1, float y1, float q1, float x2, float y2, float q2) {
    const float e = eps_up();
    if (fabsf(__fsub_rn(x1, x2)) < e && fabsf(__fsub_rn(y2, y1)) < e) return false;
    if (y1 > 0.f && y2 < 0.f) return true;
    if (y1 < 0.f && y2 > 0.f) return false;
    const float dq = __fsub_rn(q1, q2);
    if (y1 > 0.f && y2 > 0.f) return dq >= e;   // (double)dq > 1e-8
    if (y1 < 0.f && y2 < 0.f) return dq < e;    // (double)dq < 1e-8
    return false;                               // the reference falls off the end of the function here
}

__device__ __forceinline__ float pseudo_angle(float x, float y) {
    const float n = (float)((double)__fmaf_rn(x, x, __fmul_rn(y, y)) + 1e-8);       // nvcc contracts x1*x1 + y1*y1 in K1 (see header)
    return __fdiv_rn(__fmul_rn(fabsf(x), x), n);
}

// Intersection area of two rectangles given as corner lists (oriented_box_intersection_2d,
// box_intersection_2d.py:161-176).
__device__ __forceinline__ float rect_inter_area(const float* __restrict__ c1, const float* __restrict__ c2) {
    float vx[24], vy[24];
    uint32_t mk = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) { vx[i] = c1[2 * i]; vy[i] = c1[2 * i + 1]; vx[4 + i] = c2[2 * i]; vy[4 + i] = c2[2 * i + 1]; }
    // edge x edge (box_intersection_th, :11-52)
    const float epsf = eps_f();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float x1 = c1[2 * i], y1 = c1[2 * i + 1], x2 = c1[2 * ((i + 1) & 3)], y2 = c1[2 * ((i + 1) & 3) + 1];
        const float dx12 = __fsub_rn(x1, x2), dy12 = __fsub_rn(y1, y2);
        const float ex = __fsub_rn(x2, x1), ey = __fsub_rn(y2, y1);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float x3 = c2[2 * j], y3 = c2[2 * j + 1], x4 = c2[2 * ((j + 1) & 3)], y4 = c2[2 * ((j + 1) & 3) + 1];
            const float dx34 = __fsub_rn(x3, x4), dy34 = __fsub_rn(y3, y4);
            const float dx13 = __fsub_rn(x1, x3), dy13 = __fsub_rn(y1, y3);
            const float num = __fsub_rn(__fmul_rn(dx12, dy34), __fmul_rn(dy12, dx34));
            const float den_t = __fsub_rn(__fmul_rn(dx13, dy34), __fmul_rn(dy13, dx34));
            float t = __fdiv_rn(den_t, num);
            if (num == 0.0f) t = -1.0f;
            const bool mt = (t > 0.0f) && (t < 1.0f);
            const float den_u = __fsub_rn(__fmul_rn(dx12, dy13), __fmul_rn(dy12, dx13));
            float u = __fdiv_rn(-den_u, num);
            if (num == 0.0f) u = -1.0f;
            const bool mu = (u > 0.0f) && (u < 1.0f);
            const bool mm = mt && mu;
            const float t2 = __fdiv_rn(den_t, __fadd_rn(num, epsf));
            const float px = __fadd_rn(x1, __fmul_rn(t2, ex));
            const float py = __fadd_rn(y1, __fmul_rn(t2, ey));
            const float mf = mm ? 1.0f : 0.0f;
            vx[8 + 4 * i + j] = __fmul_rn(px, mf);
            vy[8 + 4 * i + j] = __fmul_rn(py, mf);
            mk |= (mm ? 1u : 0u) << (8 + 4 * i + j);
        }
    }
    // corner-in-box both ways (box1_in_box2, :54-79)
#pragma unroll
    for (int dir = 0; dir < 2; ++dir) {
        const float* p = dir == 0 ? c1 : c2;
        const float* q = dir == 0 ? c2 : c1;
        const float ax = q[0], ay = q[1];
        const float abx = __fsub_rn(q[2], ax), aby = __fsub_rn(q[3], ay);
        const float adx = __fsub_rn(q[6], ax), ady = __fsub_rn(q[7], ay);
        const float nab = __fadd_rn(__fmul_rn(abx, abx), __fmul_rn(aby, aby));
        const float nad = __fadd_rn(__fmul_rn(adx, adx), __fmul_rn(ady, ady));
        const float lo = (float)(-1e-6), hi = (float)(1.0 + 1e-6);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float amx = __fsub_rn(p[2 * i], ax), amy = __fsub_rn(p[2 * i + 1], ay);
            const float pab = __fadd_rn(__fmul_rn(abx, amx), __fmul_rn(aby, amy));
            const float pad = __fadd_rn(__fmul_rn(adx, amx), __fmul_rn(ady, amy));
            const float r1 = __fdiv_rn(pab, nab), r2 = __fdiv_rn(pad, nad);
            const bool ok = (r1 > lo) && (r1 < hi) && (r2 > lo) && (r2 < hi);
            mk |= (ok ? 1u : 0u) << (dir * 4 + i);
        }
    }
    // mean of the valid vertices (sort_indices, :121-141)
    int nv = __popc(mk);
    const int mode = NRPN_IOU_MODE;
    float sxm = 0.f, sym = 0.f;
    if (mode & 1) {                             // ATen CUDA reduce: 4 interleaved accumulators, combined left to right
        float ax[4] = {0.f, 0.f, 0.f, 0.f}, ay[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int k = 0; k < 24; ++k) {
            const float mf = ((mk >> k) & 1u) ? 1.0f : 0.0f;
            ax[k & 3] = __fadd_rn(ax[k & 3], __fmul_rn(vx[k], mf));
            ay[k & 3] = __fadd_rn(ay[k & 3], __fmul_rn(vy[k], mf));
        }
        sxm = __fadd_rn(__fadd_rn(__fadd_rn(ax[0], ax[1]), ax[2]), ax[3]);
        sym = __fadd_rn(__fadd_rn(__fadd_rn(ay[0], ay[1]), ay[2]), ay[3]);
    } else {
#pragma unroll
        for (int k = 0; k < 24; ++k) {
            const float mf = ((mk >> k) & 1u) ? 1.0f : 0.0f;
            sxm = __fadd_rn(sxm, __fmul_rn(vx[k], mf));
            sym = __fadd_rn(sym, __fmul_rn(vy[k], mf));
        }
    }
    const float mx = __fdiv_rn(sxm, (float)nv), my = __fdiv_rn(sym, (float)nv);
    // pad vertex: first masked-out intersection point
    const uint32_t inv = (~mk) & 0x00FFFF00u;
    const int pad = inv ? (__ffs(inv) - 1) : 0;
    float padx = 0.f, pady = 0.f;
#pragma unroll
    for (int k = 0; k < 24; ++k) if (k == pad) { padx = vx[k]; pady = vy[k]; }
    const float tpp = __fsub_rn(__fmul_rn(padx, pady), __fmul_rn(pady, padx));   // pad x pad term

    // the 8 shoelace terms t[i] = sel[i] x sel[i+1] of the gathered 9-vertex list (calculate_area, :143-159)
    float t[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) t[i] = tpp;     // nv < 3: every index is the pad vertex
    if (nv >= 3) {
        // normalised coordinates and pseudo-angles of the valid vertices
        float nx[24], ny[24], qq[24];
#pragma unroll
        for (int k = 0; k < 24; ++k) {
            nx[k] = __fsub_rn(vx[k], mx); ny[k] = __fsub_rn(vy[k], my);
            qq[k] = (((mk >> k) & 1u) || k == 0) ? pseudo_angle(nx[k], ny[k]) : 0.f;   // vertex 0 is the default pick
        }
        // selection sort by angle (sort_vertices_kernel, :70-106), shoelace terms recorded on the fly
        const int nsel = nv < 9 ? nv : 9;
        float pnx = 0.f, pny = 0.f, pq = 0.f;       // previous pick, normalised
        float fx = 0.f, fy = 0.f;                   // first pick, raw
        float lx = 0.f, ly = 0.f;                   // last pick, raw
        float s3x = 0.f, s3y = 0.f;                 // fourth pick (identical-box special case)
        unsigned long long takes = 0ull;
        for (int j = 0; j < nsel; ++j) {
            float bx = 1.0f, by = -eps_f(), bq = 1.0f;   // "big" start value (1, -EPSILON): q = 1*1/(1+1e-16+1e-8) -> 1.0f
            int take = 0;
            float rx = vx[0], ry = vy[0], tnx = nx[0], tny = ny[0], tq = qq[0];   // default pick is vertex 0
#pragma unroll
            for (int k = 0; k < 24; ++k) {
                if ((mk >> k) & 1u) {
                    bool ok = vert_less(nx[k], ny[k], qq[k], bx, by, bq);
                    if (ok && j > 0) ok = vert_less(pnx, pny, pq, nx[k], ny[k], qq[k]);
                    if (ok) { bx = nx[k]; by = ny[k]; bq = qq[k]; take = k; rx = vx[k]; ry = vy[k]; tnx = nx[k]; tny = ny[k]; tq = qq[k]; }
                }
            }
            // (when nothing qualified the reference leaves idx = 0 and reads vertex 0, valid or not, next round)
            takes |= (unsigned long long)take << (8 * (j & 7));
            if (j == 0) { fx = rx; fy = ry; }
            else {
                const float term = __fsub_rn(__fmul_rn(lx, ry), __fmul_rn(ly, rx));
#pragma unroll
                for (int q = 0; q < 8; ++q) if (q == j - 1) t[q] = term;
            }
            if (j == 3) { s3x = rx; s3y = ry; }
            lx = rx; ly = ry; pnx = tnx; pny = tny; pq = tq;
        }
        bool special = false;
        if (nv == 8) {                              // identical boxes (:114-129)
            int counter = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int check = (int)((takes >> (8 * j)) & 0xFF);
#pragma unroll
                for (int k = 4; k < 8; ++k) counter += ((int)((takes >> (8 * k)) & 0xFF) == check) ? 1 : 0;
            }
            special = counter == 4;
        }
        const float t_first_pad = __fsub_rn(__fmul_rn(fx, pady), __fmul_rn(fy, padx));          // first pick -> pad
        if (special) {                              // idx = p0 p1 p2 p3 p0 pad pad pad pad
            t[3] = __fsub_rn(__fmul_rn(s3x, fy), __fmul_rn(s3y, fx));
            t[4] = t_first_pad;
            t[5] = tpp; t[6] = tpp; t[7] = tpp;
        } else if (nv < 9) {                        // idx = p0 .. p(nv-1) p0 pad ...
            const float t_close = __fsub_rn(__fmul_rn(lx, fy), __fmul_rn(ly, fx));
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                if (q == nv - 1) t[q] = t_close;
                else if (q == nv) t[q] = t_first_pad;
                else if (q > nv) t[q] = tpp;
            }
        }
    }
    float total;
    if (mode & 1) {                                 // ATen CUDA reduce over 8 contiguous elements: (t0+t4 + t2+t6) + (t1+t5 + t3+t7)
        total = __fadd_rn(__fadd_rn(__fadd_rn(t[0], t[4]), __fadd_rn(t[2], t[6])), __fadd_rn(__fadd_rn(t[1], t[5]), __fadd_rn(t[3], t[7])));
    } else {
        total = t[0];
#pragma unroll
        for (int i = 1; i < 8; ++i) total = __fadd_rn(total, t[i]);
    }
    return __fdiv_rn(fabsf(total), 2.0f);
}

// Exact-zero test on the tail of a prepared record (floats 8..15: area, vol, zmin, zmax, cx, cy, rad, cullable): true only
// when the reference arithmetic yields exactly 0 for the pair (disjoint bounding circles -> no vertex of the intersection
// polygon; disjoint z ranges -> z_overlap clamps to 0).  Cheap enough to run on every pair before the full clip.
__device__ __forceinline__ bool obb_surely_zero(const float* __restrict__ ta, const float* __restrict__ tb) {
    if (!(__float_as_int(ta[7]) && __float_as_int(tb[7]))) return false;
    const float dx = ta[4] - tb[4], dy = ta[5] - tb[5], rr = ta[6] + tb[6];
    if (dx * dx + dy * dy > rr * rr) return true;
    return ta[2] > tb[3] || tb[2] > ta[3];
}

// NMS-only shortcut: true only when IoU(a, b) <= thr is CERTAIN, so that the suppression test `!(iou <= thr)` is false without
// evaluating the polygon clip.  On top of the exact-zero tests:  IoU = I / U with I <= min(V_a, V_b), U >= max(V_a, V_b) and
// I = A_int * z_overlap <= A_i * z_overlap, hence
//     IoU <= min(V) / max(V)          (boxes of very different volume cannot suppress each other)
//     IoU <= z_overlap / max(depth)   (a thin slab of z overlap cannot either)
//     IoU <= min(A_a, A_b, lens) * z_overlap / max(V)   (footprints that only graze each other cannot either).
// thr_m = thr - 1e-3: the margin dwarfs every rounding error of the reference's fp32 chain (its value never exceeds the exact IoU by
// more than ~1e-5: mis-sorted or missing vertices only ever SHRINK the polygon), so the skipped decisions are the reference's.
#ifndef NRPN_LENS_CULL
#define NRPN_LENS_CULL 1
#endif
__device__ __forceinline__ bool obb_surely_not_above(const float* __restrict__ ta, const float* __restrict__ tb, float thr_m) {
    if (!(__float_as_int(ta[7]) && __float_as_int(tb[7]))) return false;
    const float dx = ta[4] - tb[4], dy = ta[5] - tb[5], rr = ta[6] + tb[6];
    const float d2 = dx * dx + dy * dy;
    if (d2 > rr * rr) return true;
    const float oz = fminf(ta[3], tb[3]) - fmaxf(ta[2], tb[2]);
    if (!(oz >= 0.0f)) return true;                                           // disjoint z ranges (ta[2] > tb[3] || tb[2] > ta[3])
    if (thr_m > 0.0f) {
        const float vmax = fmaxf(ta[1], tb[1]);
        if (fminf(ta[1], tb[1]) <= thr_m * vmax) return true;
        if (oz <= thr_m * fmaxf(ta[3] - ta[2], tb[3] - tb[2])) return true;
        // intersection = footprint overlap x z overlap, union >= the larger volume; the footprint overlap is at most the smaller footprint and at
        // most the bounding rectangle of the lens the two bounding circles share: (r_a + r_b - distance) x 2 min(r)
        const float lens = 2.0f * fminf(ta[6], tb[6]) * (rr - sqrtf(d2));
        if (NRPN_LENS_CULL && fminf(fminf(ta[0], tb[0]), lens) * oz <= thr_m * vmax) return true;
    }
    return false;
}

// cal_iou_3d for one pair without the shortcut (oriented_iou_loss.py:82-107). a = "box1" (the picked box in NMS).
__device__ __forceinline__ float iou3d_obb_full(const ObbPrep& a, const ObbPrep& b) {
    float zo = __fsub_rn(fminf(a.zmax, b.zmax), fmaxf(a.zmin, b.zmin));
    if (!(zo >= 0.0f)) zo = (zo != zo) ? zo : 0.0f;
    const float inter = rect_inter_area(a.c, b.c);
    const float u = __fsub_rn(__fadd_rn(a.area, b.area), inter);
    const float iou2d = __fdiv_rn(inter, u);
    const float i3 = __fmul_rn(__fmul_rn(iou2d, u), zo);
    const float u3 = __fsub_rn(__fadd_rn(a.vol, b.vol), i3);
    return __fdiv_rn(i3, u3);
}

// Separating-axis test with a margin: true only when, along an edge direction of one of the two rectangles, the projections of the two corner sets are
// further apart than 1e-3 of the boxes' size (+ 8e-6 of the coordinate magnitude) -- three orders of magnitude above anything fp32 rounding or the
// reference's 1e-6 corner tolerance can move.  Then no edge pair crosses (t or u is far outside (0, 1), or the edges are parallel), no corner lies
// inside the other rectangle, every mask of the reference is false, its vertex list is empty and it returns exactly 0 (box_intersection_2d.py:11-79,
// sort_vert_kernel.cu:62: num_valid < 3 -> pad vertex only).  An exact-zero cull like the bounding-circle test, ~40 % sharper on touching circles.
__device__ __forceinline__ bool obb_footprints_surely_disjoint(const ObbPrep& a, const ObbPrep& b) {
    if (!(a.cullable && b.cullable)) return false;
    const float scale = fmaxf(fmaxf(fabsf(a.cx), fabsf(a.cy)), fmaxf(fabsf(b.cx), fabsf(b.cy)));
    const float margin = 1e-3f * (a.rad + b.rad) + 8e-6f * scale;
#pragma unroll
    for (int ax = 0; ax < 4; ++ax) {
        const float* s = ax < 2 ? a.c : b.c;
        const int k = (ax & 1) ? 3 : 1;                         // edge corner0 -> corner1 and corner0 -> corner3
        const float ex = s[2 * k] - s[0], ey = s[2 * k + 1] - s[1];
        const float len = sqrtf(ex * ex + ey * ey);
        float amin = 3.0e38f, amax = -3.0e38f, bmin = 3.0e38f, bmax = -3.0e38f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float pa = a.c[2 * i] * ex + a.c[2 * i + 1] * ey, pb = b.c[2 * i] * ex + b.c[2 * i + 1] * ey;
            amin = fminf(amin, pa); amax = fmaxf(amax, pa); bmin = fminf(bmin, pb); bmax = fmaxf(bmax, pb);
        }
        const float gap = fmaxf(bmin - amax, amin - bmax);
        if (len > 0.0f && gap > margin * len) return true;
    }
    return false;
}

// NMS decision for one pair: does the picked box a suppress the candidate b at threshold thr?  (`!(iou <= thr)` keeps the reference's NaN behaviour.)
__device__ __forceinline__ bool obb_suppresses(const ObbPrep& a, const ObbPrep& b, float thr) {
    if (thr >= 0.0f && obb_footprints_surely_disjoint(a, b)) return false;      // the reference computes exactly 0, and !(0 <= thr) is false
    return !(iou3d_obb_full(a, b) <= thr);
}

__device__ __forceinline__ float iou3d_obb(const ObbPrep& a, const ObbPrep& b, bool allow_cull) {
    if (allow_cull && a.cullable && b.cullable) {
        const float dx = a.cx - b.cx, dy = a.cy - b.cy, rr = a.rad + b.rad;
        if (dx * dx + dy * dy > rr * rr) return 0.0f;           // footprints cannot touch -> reference yields exactly 0
        if (a.zmin > b.zmax || b.zmin > a.zmax) return 0.0f;     // z_overlap clamps to 0
        if (obb_footprints_surely_disjoint(a, b)) return 0.0f;    // no vertex at all -> intersection exactly 0
    }
    return iou3d_obb_full(a, b);
}

// box_iou_3d AABB branch for one pair (utils.py:418-458).
__device__ __forceinline__ float iou3d_aabb(const float* __restrict__ a, const float* __restrict__ b) {
    const float va = __fmul_rn(__fmul_rn(__fsub_rn(a[3], a[0]), __fsub_rn(a[4], a[1])), __fsub_rn(a[5], a[2]));
    const float vb = __fmul_rn(__fmul_rn(__fsub_rn(b[3], b[0]), __fsub_rn(b[4], b[1])), __fsub_rn(b[5], b[2]));
    float w = __fsub_rn(fminf(a[3], b[3]), fmaxf(a[0], b[0])); if (w < 0.f) w = 0.f;
    float h = __fsub_rn(fminf(a[4], b[4]), fmaxf(a[1], b[1])); if (h < 0.f) h = 0.f;
    float d = __fsub_rn(fminf(a[5], b[5]), fmaxf(a[2], b[2])); if (d < 0.f) d = 0.f;
    const float inter = __fmul_rn(__fmul_rn(w, h), d);
    const float uni = __fsub_rn(__fadd_rn(va, vb), inter);
    return __fdiv_rn(inter, uni);
}

}  // namespace nrpn
