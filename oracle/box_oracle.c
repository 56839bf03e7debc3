/*
 * oracle/box_oracle.c -- TEST INFRASTRUCTURE ONLY (not product code).
 *
 * CPU restatement, in plain C, of the reference's box-overlap path:
 *   - oriented (yaw-only) 3-D box IoU        nerf_rpn/model/rotated_iou/oriented_iou_loss.py:6-57,82-107
 *   - edge/edge + corner-in-box + vertices    nerf_rpn/model/rotated_iou/box_intersection_2d.py:11-159
 *   - convex-polygon vertex sort (native K1)  nerf_rpn/model/rotated_iou/cuda_op/sort_vert_kernel.cu:15-134
 *   - axis-aligned IoU                         nerf_rpn/model/utils.py:418-458
 *   - greedy NMS / per-level NMS               nerf_rpn/model/utils.py:215-265
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load this library. The product path (nerf_rpn_b200/csrc) never links it.
 *
 * Arithmetic conventions (shared with the CUDA kernels so that CUDA == oracle bit-for-bit):
 *   - every fp32 operation is a separately rounded IEEE op (build with -ffp-contract=off);
 *   - sin/cos are evaluated in double precision and rounded once to fp32;
 *   - reductions (mean of valid vertices, shoelace sum) are plain left-to-right sums.
 * The reference itself runs this chain through ATen kernels whose reduction trees and
 * libm differ between its CPU and GPU builds; parity with it is therefore pinned by the
 * golden vectors in tests/golden/ (IoU to 2e-6, NMS keep sets exactly).
 *
 * Pinning status: the Python part of the chain is pinned by golden vectors generated from
 * the unmodified reference imported on CPU (tools/make_golden.py). The native kernel K1
 * cannot be executed without a GPU next to /root/reference, so orc_sort_vertices is
 * "parity unpinned" w.r.t. K1's own binary; it follows the source line by line, returns
 * false where compare_vertices() falls off its end (sort_vert_kernel.cu:15-40), and drops
 * writes past slot 8 where the reference would write out of bounds (num_valid > 8).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_EPS_D 1e-8          /* EPSILON, box_intersection_2d.py:9 / sort_vert_kernel.cu:8 */

/* Arithmetic mode (orc_set_mode), mirrors NRPN_IOU_MODE of csrc/box_iou.cuh:
 *   0 (default)  the conventions above == the reference's CPU build on the golden vectors;
 *   bit 0        operation ORDER of the reference's torch-CUDA build, measured on the GPU by tools/ref_gpu_probe.py against the
 *                unmodified reference: box2corners_th's bmm = fma(y4, r1, x4*r0); torch.sum over the 24 masked vertices = four
 *                interleaved accumulators ((a0+a1)+a2)+a3; torch.sum over the 8 shoelace terms = (t0+t4 + t2+t6) + (t1+t5 + t3+t7);
 *   bit 1        sin / cos through float sinf / cosf (the CUDA build calls CUDA's; a CPU libm can only approximate that, so
 *                this bit exists for structural cross-checks of the kernel logic, not for bit-parity with a GPU).
 * K1's pseudo-angle denominator is fma(x, x, y*y) in every mode: nvcc contracts `x1*x1 + y1*y1` (sort_vert_kernel.cu:25) -- SASS
 * of the reference's own build (FMUL y*y; FFMA x*x + .), confirmed bit-for-bit against that binary on 600 000 polygons. */
static int orc_mode = 0;
void orc_set_mode(int m) { orc_mode = m; }
int orc_get_mode(void) { return orc_mode; }
#define ORC_MAXV 24
#define ORC_NIDX 9

/* ---------------------------------------------------------------- corners */
/* box2corners_th, oriented_iou_loss.py:6-35: (x,y,w,h,alpha) -> 4 corners.
 * The reference multiplies a (4,2) corner matrix with rot_T = [[c,s],[-s,c]] via bmm. */
static void orc_corners(float x, float y, float w, float h, float alpha, float c[8])
{
    static const float sx[4] = {0.5f, -0.5f, -0.5f, 0.5f};
    static const float sy[4] = {0.5f, 0.5f, -0.5f, -0.5f};
    float s = (orc_mode & 2) ? sinf(alpha) : (float)sin((double)alpha);
    float co = (orc_mode & 2) ? cosf(alpha) : (float)cos((double)alpha);
    float ns = -s;
    for (int i = 0; i < 4; ++i) {
        float x4 = sx[i] * w;
        float y4 = sy[i] * h;
        float rx, ry;
        if (orc_mode & 1) {
            float t = x4 * co; rx = fmaf(y4, ns, t);
            t = x4 * s;        ry = fmaf(y4, co, t);
        } else {
            rx = x4 * co;  float t = y4 * ns;  rx = rx + t;   /* row . rot_T[:,0] */
            ry = x4 * s;   t = y4 * co;        ry = ry + t;   /* row . rot_T[:,1] */
        }
        c[2 * i + 0] = rx + x;
        c[2 * i + 1] = ry + y;
    }
}

/* compare_vertices, sort_vert_kernel.cu:15-40 */
static int orc_cmp(float x1, float y1, float x2, float y2)
{
    if ((double)fabsf(x1 - x2) < ORC_EPS_D && (double)fabsf(y2 - y1) < ORC_EPS_D) return 0;
    if (y1 > 0 && y2 < 0) return 1;
    if (y1 < 0 && y2 > 0) return 0;
    float n1 = (float)((double)fmaf(x1, x1, y1 * y1) + ORC_EPS_D);     /* nvcc's contraction of x1*x1 + y1*y1 (see orc_mode note) */
    float n2 = (float)((double)fmaf(x2, x2, y2 * y2) + ORC_EPS_D);
    float q1 = fabsf(x1) * x1 / n1;
    float q2 = fabsf(x2) * x2 / n2;
    float d = q1 - q2;
    if (y1 > 0 && y2 > 0) return (double)d > ORC_EPS_D;
    if (y1 < 0 && y2 < 0) return (double)d < ORC_EPS_D;
    return 0; /* reference falls off the end here (UB); convention: false */
}

/* sort_vertices_kernel body for one polygon, sort_vert_kernel.cu:52-132.
 * v: m x 2 mean-centred vertices, mask: m flags, nv: number of valid; idx: 9 outputs. */
static void orc_sort_one(const float *v, const uint8_t *mask, int nv, int m, int32_t *idx)
{
    int pad = 0;
    for (int j = 8; j < m; ++j) if (!mask[j]) { pad = j; break; }
    if (nv < 3) { for (int j = 0; j < ORC_NIDX; ++j) idx[j] = pad; return; }
    int32_t tmp[ORC_MAXV + 2];
    for (int j = 0; j < nv; ++j) {
        float x_min = 1.0f, y_min = (float)(-ORC_EPS_D);
        int take = 0;
        float x2 = 0.f, y2 = 0.f;
        if (j > 0) { int i2 = tmp[j - 1]; x2 = v[2 * i2]; y2 = v[2 * i2 + 1]; }
        for (int k = 0; k < m; ++k) {
            float x = v[2 * k], y = v[2 * k + 1];
            if (!mask[k]) continue;
            if (j == 0) {
                if (orc_cmp(x, y, x_min, y_min)) { x_min = x; y_min = y; take = k; }
            } else {
                if (orc_cmp(x, y, x_min, y_min) && orc_cmp(x2, y2, x, y)) { x_min = x; y_min = y; take = k; }
            }
        }
        tmp[j] = take;
    }
    for (int j = 0; j < ORC_NIDX; ++j) idx[j] = pad;
    for (int j = 0; j < nv && j < ORC_NIDX; ++j) idx[j] = tmp[j];
    if (nv < ORC_NIDX) idx[nv] = tmp[0];
    /* identical-box corner case, sort_vert_kernel.cu:114-129 */
    if (nv == 8) {
        int counter = 0;
        for (int j = 0; j < 4; ++j) { int check = idx[j]; for (int k = 4; k < 8; ++k) if (idx[k] == check) counter++; }
        if (counter == 4) { idx[4] = idx[0]; for (int j = 5; j < ORC_NIDX; ++j) idx[j] = pad; }
    }
}

/* Public: batched K1 restatement. vertices (b,n,m,2) f32, mask (b,n,m) u8, num_valid (b,n) i32 -> idx (b,n,9) */
void orc_sort_vertices(const float *vertices, const uint8_t *mask, const int32_t *num_valid,
                       int b, int n, int m, int32_t *idx)
{
    for (long p = 0; p < (long)b * n; ++p)
        orc_sort_one(vertices + p * m * 2, mask + p * m, num_valid[p], m, idx + p * ORC_NIDX);
}

/* oriented_box_intersection_2d, box_intersection_2d.py:161-176, on two corner sets. */
static float orc_inter_area(const float c1[8], const float c2[8])
{
    float vx[ORC_MAXV], vy[ORC_MAXV];
    uint8_t mk[ORC_MAXV];
    for (int i = 0; i < 4; ++i) { vx[i] = c1[2 * i]; vy[i] = c1[2 * i + 1]; vx[4 + i] = c2[2 * i]; vy[4 + i] = c2[2 * i + 1]; }
    /* box_intersection_th, :11-52 */
    const float epsf = (float)ORC_EPS_D;
    for (int i = 0; i < 4; ++i) {
        float x1 = c1[2 * i], y1 = c1[2 * i + 1], x2 = c1[2 * ((i + 1) & 3)], y2 = c1[2 * ((i + 1) & 3) + 1];
        for (int j = 0; j < 4; ++j) {
            float x3 = c2[2 * j], y3 = c2[2 * j + 1], x4 = c2[2 * ((j + 1) & 3)], y4 = c2[2 * ((j + 1) & 3) + 1];
            float a = (x1 - x2) * (y3 - y4), bb = (y1 - y2) * (x3 - x4);
            float num = a - bb;
            a = (x1 - x3) * (y3 - y4); bb = (y1 - y3) * (x3 - x4);
            float den_t = a - bb;
            float t = den_t / num;
            if (num == 0.0f) t = -1.0f;
            int mt = (t > 0.0f) && (t < 1.0f);
            a = (x1 - x2) * (y1 - y3); bb = (y1 - y2) * (x1 - x3);
            float den_u = a - bb;
            float u = -den_u / num;
            if (num == 0.0f) u = -1.0f;
            int mu = (u > 0.0f) && (u < 1.0f);
            int mm = mt && mu;
            float t2 = den_t / (num + epsf);
            float px = t2 * (x2 - x1); px = x1 + px;
            float py = t2 * (y2 - y1); py = y1 + py;
            float mf = mm ? 1.0f : 0.0f;
            vx[8 + 4 * i + j] = px * mf;
            vy[8 + 4 * i + j] = py * mf;
            mk[8 + 4 * i + j] = (uint8_t)mm;
        }
    }
    /* box1_in_box2, :54-79 (both directions, :81-94) */
    for (int dir = 0; dir < 2; ++dir) {
        const float *p = dir == 0 ? c1 : c2;   /* points tested */
        const float *q = dir == 0 ? c2 : c1;   /* containing box */
        float ax = q[0], ay = q[1];
        float abx = q[2] - ax, aby = q[3] - ay;
        float adx = q[6] - ax, ady = q[7] - ay;
        float nab = abx * abx; { float t = aby * aby; nab = nab + t; }
        float nad = adx * adx; { float t = ady * ady; nad = nad + t; }
        const float lo = (float)(-1e-6), hi = (float)(1.0 + 1e-6);
        for (int i = 0; i < 4; ++i) {
            float amx = p[2 * i] - ax, amy = p[2 * i + 1] - ay;
            float pab = abx * amx; { float t = aby * amy; pab = pab + t; }
            float pad_ = adx * amx; { float t = ady * amy; pad_ = pad_ + t; }
            float r1 = pab / nab, r2 = pad_ / nad;
            int ok = (r1 > lo) && (r1 < hi) && (r2 > lo) && (r2 < hi);
            mk[dir * 4 + i] = (uint8_t)ok;
        }
    }
    /* sort_indices, :121-141 */
    int nv = 0; float sxm = 0.f, sym = 0.f;
    if (orc_mode & 1) {
        float ax[4] = {0.f, 0.f, 0.f, 0.f}, ay[4] = {0.f, 0.f, 0.f, 0.f};
        for (int k = 0; k < ORC_MAXV; ++k) {
            float mf = mk[k] ? 1.0f : 0.0f;
            nv += mk[k];
            float px = vx[k] * mf, py = vy[k] * mf;
            ax[k & 3] = ax[k & 3] + px;
            ay[k & 3] = ay[k & 3] + py;
        }
        sxm = ax[0] + ax[1]; sxm = sxm + ax[2]; sxm = sxm + ax[3];
        sym = ay[0] + ay[1]; sym = sym + ay[2]; sym = sym + ay[3];
    } else {
        for (int k = 0; k < ORC_MAXV; ++k) {
            float mf = mk[k] ? 1.0f : 0.0f;
            nv += mk[k];
            sxm = sxm + vx[k] * mf;
            sym = sym + vy[k] * mf;
        }
    }
    float mx = sxm / (float)nv, my = sym / (float)nv;
    float vn[2 * ORC_MAXV];
    for (int k = 0; k < ORC_MAXV; ++k) { vn[2 * k] = vx[k] - mx; vn[2 * k + 1] = vy[k] - my; }
    int32_t idx[ORC_NIDX];
    orc_sort_one(vn, mk, nv, ORC_MAXV, idx);
    /* calculate_area, :143-159 (gathers the un-normalised vertices) */
    float t[8];
    for (int i = 0; i < 8; ++i) {
        float a = vx[idx[i]] * vy[idx[i + 1]];
        float bb = vy[idx[i]] * vx[idx[i + 1]];
        t[i] = a - bb;
    }
    float total;
    if (orc_mode & 1) {
        float a0 = t[0] + t[4], a1 = t[1] + t[5], a2 = t[2] + t[6], a3 = t[3] + t[7];
        float l = a0 + a2, r = a1 + a3;
        total = l + r;
    } else {
        total = 0.f;
        for (int i = 0; i < 8; ++i) total = total + t[i];
    }
    return fabsf(total) / 2.0f;
}

/* cal_iou_3d, oriented_iou_loss.py:82-107 for one pair of (x,y,z,w,h,d,alpha) boxes. */
float orc_iou3d_obb(const float *a, const float *b)
{
    float c1[8], c2[8];
    orc_corners(a[0], a[1], a[3], a[4], a[6], c1);
    orc_corners(b[0], b[1], b[3], b[4], b[6], c2);
    float zmax1 = a[2] + a[5] * 0.5f, zmin1 = a[2] - a[5] * 0.5f;
    float zmax2 = b[2] + b[5] * 0.5f, zmin2 = b[2] - b[5] * 0.5f;
    float zo = fminf(zmax1, zmax2) - fmaxf(zmin1, zmin2);
    if (!(zo >= 0.0f)) zo = (zo != zo) ? zo : 0.0f;     /* clamp_min(0) keeps NaN */
    float inter = orc_inter_area(c1, c2);
    float area1 = a[3] * a[4], area2 = b[3] * b[4];
    float u = area1 + area2; u = u - inter;
    float iou2d = inter / u;
    float i3 = iou2d * u; i3 = i3 * zo;
    float v1 = a[3] * a[4]; v1 = v1 * a[5];
    float v2 = b[3] * b[4]; v2 = v2 * b[5];
    float u3 = v1 + v2; u3 = u3 - i3;
    return i3 / u3;
}

/* _aabb_inter_union_3d + box_iou_3d, utils.py:387-458 for one pair of (x1,y1,z1,x2,y2,z2). */
float orc_iou3d_aabb(const float *a, const float *b)
{
    float va = (a[3] - a[0]) * (a[4] - a[1]); va = va * (a[5] - a[2]);
    float vb = (b[3] - b[0]) * (b[4] - b[1]); vb = vb * (b[5] - b[2]);
    float w = fminf(a[3], b[3]) - fmaxf(a[0], b[0]); if (w < 0.f) w = 0.f;
    float h = fminf(a[4], b[4]) - fmaxf(a[1], b[1]); if (h < 0.f) h = 0.f;
    float d = fminf(a[5], b[5]) - fmaxf(a[2], b[2]); if (d < 0.f) d = 0.f;
    float inter = w * h; inter = inter * d;
    float uni = va + vb; uni = uni - inter;
    return inter / uni;
}

float orc_iou3d(const float *a, const float *b, int box_dim)
{
    return box_dim == 7 ? orc_iou3d_obb(a, b) : orc_iou3d_aabb(a, b);
}

/* box_iou_3d: full (n x m) matrix, first argument is "boxes1". */
void orc_iou_matrix(const float *a, int n, const float *b, int m, int box_dim, float *out)
{
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < m; ++j)
            out[(long)i * m + j] = orc_iou3d(a + (long)i * box_dim, b + (long)j * box_dim, box_dim);
}

/* element-wise pairs (cal_iou_3d on (1,n,7) x (1,n,7)) */
void orc_iou_pairs(const float *a, const float *b, int n, int box_dim, float *out)
{
    for (int i = 0; i < n; ++i) out[i] = orc_iou3d(a + (long)i * box_dim, b + (long)i * box_dim, box_dim);
}

/* stable descending argsort of scores: ties keep ascending index (the convention both the
 * oracle and the CUDA path use; torch.argsort leaves tie order unspecified). */
typedef struct { float s; int32_t i; } orc_si;
static int orc_si_cmp(const void *pa, const void *pb)
{
    const orc_si *a = (const orc_si *)pa, *b = (const orc_si *)pb;
    if (a->s > b->s) return -1;
    if (a->s < b->s) return 1;
    return (a->i > b->i) - (a->i < b->i);
}

/* Exactness-preserving shortcut for large inputs: 1 when the reference chain is certain to return an IoU of exactly 0
 * (positive finite extents and either disjoint z ranges or bounding circles / boxes further apart than their radii plus a
 * 0.1 % + 1e-3 margin). Used by orc_nms only; the IoU functions above never take it. */
static int orc_surely_zero(const float *a, const float *b, int box_dim)
{
    for (int i = 0; i < box_dim; ++i) if (!isfinite(a[i]) || !isfinite(b[i])) return 0;
    if (box_dim == 7) {
        if (!(a[3] > 0 && a[4] > 0 && a[5] > 0 && b[3] > 0 && b[4] > 0 && b[5] > 0)) return 0;
        double za0 = (double)a[2] - 0.5 * a[5], za1 = (double)a[2] + 0.5 * a[5];
        double zb0 = (double)b[2] - 0.5 * b[5], zb1 = (double)b[2] + 0.5 * b[5];
        if (za0 > zb1 * 1.0 + 1e-3 + 1e-6 * fabs(zb1) || zb0 > za1 + 1e-3 + 1e-6 * fabs(za1)) return 1;
        double ra = 0.5 * sqrt((double)a[3] * a[3] + (double)a[4] * a[4]) * 1.001 + 1e-3;
        double rb = 0.5 * sqrt((double)b[3] * b[3] + (double)b[4] * b[4]) * 1.001 + 1e-3;
        double dx = (double)a[0] - b[0], dy = (double)a[1] - b[1];
        return dx * dx + dy * dy > (ra + rb) * (ra + rb);
    }
    return 0;
}

/* nms(), utils.py:215-230. keep[] receives indices in pick order (score-descending). */
int orc_nms(const float *boxes, int box_dim, const float *scores, int n, float thr, int64_t *keep)
{
    if (n <= 0) return 0;
    orc_si *ord = (orc_si *)malloc(sizeof(orc_si) * (size_t)n);
    uint8_t *dead = (uint8_t *)calloc((size_t)n, 1);
    for (int i = 0; i < n; ++i) { ord[i].s = scores[i]; ord[i].i = i; }
    qsort(ord, (size_t)n, sizeof(orc_si), orc_si_cmp);
    int nk = 0;
    for (int p = 0; p < n; ++p) {
        if (dead[p]) continue;
        int i = ord[p].i;
        keep[nk++] = i;
        for (int q = p + 1; q < n; ++q) {
            if (dead[q]) continue;
            const float *bi = boxes + (long)i * box_dim, *bq = boxes + (long)ord[q].i * box_dim;
            if (thr >= 0.0f && orc_surely_zero(bi, bq, box_dim)) continue;     /* IoU is exactly 0 <= thr: kept */
            float iou = orc_iou3d(bi, bq, box_dim);
            if (!(iou <= thr)) dead[q] = 1;      /* reference keeps iou <= thr, utils.py:228 */
        }
    }
    free(ord); free(dead);
    return nk;
}

/* batched_nms(), utils.py:233-265: NMS per group id, result sorted by score descending
 * (ties: ascending index). */
int orc_batched_nms(const float *boxes, int box_dim, const float *scores, const int32_t *group,
                    int n, float thr, int64_t *keep)
{
    if (n <= 0) return 0;
    uint8_t *mask = (uint8_t *)calloc((size_t)n, 1);
    int32_t *sel = (int32_t *)malloc(sizeof(int32_t) * (size_t)n);
    float *bsub = (float *)malloc(sizeof(float) * (size_t)n * box_dim);
    float *ssub = (float *)malloc(sizeof(float) * (size_t)n);
    int64_t *ksub = (int64_t *)malloc(sizeof(int64_t) * (size_t)n);
    uint8_t *done = (uint8_t *)calloc((size_t)n, 1);
    for (int s = 0; s < n; ++s) {
        if (done[s]) continue;
        int g = group[s], cnt = 0;
        for (int i = s; i < n; ++i) if (group[i] == g) {
            done[i] = 1; sel[cnt] = i;
            memcpy(bsub + (long)cnt * box_dim, boxes + (long)i * box_dim, sizeof(float) * box_dim);
            ssub[cnt] = scores[i]; cnt++;
        }
        int nk = orc_nms(bsub, box_dim, ssub, cnt, thr, ksub);
        for (int k = 0; k < nk; ++k) mask[sel[ksub[k]]] = 1;
    }
    int total = 0;
    orc_si *ord = (orc_si *)malloc(sizeof(orc_si) * (size_t)n);
    for (int i = 0; i < n; ++i) if (mask[i]) { ord[total].s = scores[i]; ord[total].i = i; total++; }
    qsort(ord, (size_t)total, sizeof(orc_si), orc_si_cmp);
    for (int i = 0; i < total; ++i) keep[i] = ord[i].i;
    free(ord); free(mask); free(sel); free(bsub); free(ssub); free(ksub); free(done);
    return total;
}
