"""CPU stand-in for the reference's pybind module `sort_vertices` (tools only, never shipped).

A literal, numpy-vectorised restatement of nerf_rpn/model/rotated_iou/cuda_op/sort_vert_kernel.cu:15-134
so that the UNMODIFIED reference Python (box_intersection_2d.py:141 -> cuda_ext.py:8) can be imported and
run on a GPU-less box to generate golden vectors (tools/make_golden.py).  It is deliberately independent
of oracle/box_oracle.c so the two restatements cross-check each other.
"""
import numpy as np
import torch

EPS = 1e-8


def _cmp(x1, y1, x2, y2):
    x1 = x1.astype(np.float32); y1 = y1.astype(np.float32)
    x2 = x2.astype(np.float32); y2 = y2.astype(np.float32)
    out = np.zeros(x1.shape, dtype=bool)
    decided = np.zeros(x1.shape, dtype=bool)
    eq = (np.abs(x1 - x2).astype(np.float64) < EPS) & (np.abs(y2 - y1).astype(np.float64) < EPS)
    decided |= eq
    c = (~decided) & (y1 > 0) & (y2 < 0)
    out |= c; decided |= c
    c = (~decided) & (y1 < 0) & (y2 > 0)
    decided |= c
    with np.errstate(all="ignore"):
        # nvcc contracts `x1*x1 + y1*y1` (sort_vert_kernel.cu:25) into fma(x1, x1, y1*y1): SASS of the reference's own build, and
        # bit-for-bit agreement with that binary on the GPU (tests/test_gpu_reference.py)
        n1 = ((x1.astype(np.float64) * x1 + (y1 * y1).astype(np.float64)).astype(np.float32).astype(np.float64) + EPS).astype(np.float32)
        n2 = ((x2.astype(np.float64) * x2 + (y2 * y2).astype(np.float64)).astype(np.float32).astype(np.float64) + EPS).astype(np.float32)
        d = (np.abs(x1) * x1 / n1 - np.abs(x2) * x2 / n2).astype(np.float32).astype(np.float64)
    c = (~decided) & (y1 > 0) & (y2 > 0)
    out |= c & (d > EPS); decided |= c
    c = (~decided) & (y1 < 0) & (y2 < 0)
    out |= c & (d < EPS); decided |= c
    return out  # undecided (falls off the end in the CUDA source) -> False


def sort_vertices_forward(vertices, mask, num_valid):
    v = vertices.detach().cpu().numpy().astype(np.float32)
    mk = mask.detach().cpu().numpy().astype(bool)
    nv = num_valid.detach().cpu().numpy().astype(np.int64)
    b, n, m, _ = v.shape
    P = b * n
    v = v.reshape(P, m, 2); mk = mk.reshape(P, m); nv = nv.reshape(P)
    inv = ~mk[:, 8:]
    pad = np.where(inv.any(1), inv.argmax(1) + 8, 0)
    idx = np.zeros((P, 9), dtype=np.int32)
    tmp = np.zeros((P, m + 1), dtype=np.int64)
    ar = np.arange(P)
    for j in range(min(int(nv.max()) if P else 0, m)):
        active = (nv >= 3) & (j < nv)
        x_min = np.full(P, 1.0, np.float32); y_min = np.full(P, np.float32(-EPS), np.float32)
        take = np.zeros(P, dtype=np.int64)
        if j > 0:
            x2 = v[ar, tmp[:, j - 1], 0]; y2 = v[ar, tmp[:, j - 1], 1]
        for k in range(m):
            x = v[:, k, 0]; y = v[:, k, 1]
            ok = mk[:, k] & _cmp(x, y, x_min, y_min)
            if j > 0:
                ok &= _cmp(x2, y2, x, y)
            ok &= active
            x_min = np.where(ok, x, x_min); y_min = np.where(ok, y, y_min); take = np.where(ok, k, take)
        tmp[:, j] = take
    for p in range(P):
        if nv[p] < 3:
            idx[p, :] = pad[p]
            continue
        idx[p, :] = pad[p]
        k = min(nv[p], 9)
        idx[p, :k] = tmp[p, :k]
        if nv[p] < 9:
            idx[p, nv[p]] = tmp[p, 0]
        if nv[p] == 8:
            counter = sum(int(idx[p, kk] == idx[p, j]) for j in range(4) for kk in range(4, 8))
            if counter == 4:
                idx[p, 4] = idx[p, 0]
                idx[p, 5:] = pad[p]
    return torch.from_numpy(idx.reshape(b, n, 9))
