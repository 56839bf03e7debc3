"""GPU parity tests (through the C ABI) for box overlap, vertex sort, NMS and RPN post-processing.
Bar: bit-exact against the oracle (oracle/box_oracle.c, oracle/rpn_post.py) on the same seeded inputs; against
the reference's golden vectors within the tolerance the oracle itself is held to (tests/test_oracle_golden.py)."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import box as obox
from oracle import rpn_post as rp

pytestmark = pytest.mark.gpu

SIZES = ((8,), (16,), (32,), (64,))
ASPECT = ((1., 1., 1.), (1., 1., 2.), (1., 2., 2.), (1., 1., 3.), (1., 3., 3.))


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from nerf_rpn_b200 import ops as _ops
    return _ops


@pytest.fixture(scope="module")
def G(golden_dir):
    return {n: np.load(os.path.join(golden_dir, n + ".npz")) for n in
            ("iou", "nms", "decode", "sort_vertices", "rpn_small_aabb", "rpn_small_obb")}


def cu(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).cuda().contiguous()


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def rand_obb(n, rng, extent, smin=0.5, smax=10.5):
    return np.concatenate([rng.random((n, 3)) * extent, rng.random((n, 3)) * (smax - smin) + smin,
                           (rng.random((n, 1)) - .5) * math.pi], 1).astype(np.float32)


def rand_aabb(n, rng, extent, smin=0.5, smax=12.0):
    lo = rng.random((n, 3)) * extent
    return np.concatenate([lo, lo + rng.random((n, 3)) * (smax - smin) + smin], 1).astype(np.float32)


def test_iou_pairs_bit_exact_vs_oracle_and_golden(ops, G):
    g = G["iou"]
    for a, b, ref in ((g["kat_a"], g["kat_b"], g["kat_iou"]), (g["rand_a"], g["rand_b"], g["rand_iou"])):
        got = ops.iou3d_pairs(cu(a), cu(b)).cpu().numpy()
        np.testing.assert_array_equal(bits(got), bits(obox.iou_pairs(a, b)))
        np.testing.assert_allclose(got, ref, rtol=0, atol=2e-6)
    rng = np.random.default_rng(5)
    n = 100000
    a, b = rand_obb(n, rng, 8), rand_obb(n, rng, 8)
    a[:2000] = b[:2000]; b[2000:4000, 6] = a[2000:4000, 6]; a[6000:8000, 6] = 0; b[6000:8000, 6] = 0
    got = ops.iou3d_pairs(cu(a), cu(b)).cpu().numpy()
    np.testing.assert_array_equal(bits(got), bits(obox.iou_pairs(a, b)))
    a, b = rand_aabb(n, rng, 10), rand_aabb(n, rng, 10)
    np.testing.assert_array_equal(bits(ops.iou3d_pairs(cu(a), cu(b)).cpu().numpy()), bits(obox.iou_pairs(a, b)))


def test_iou_matrix(ops, G):
    g = G["iou"]
    for key in ("mat_boxes", "aabb_boxes"):
        m = ops.iou3d_matrix(cu(g[key]), cu(g[key])).cpu().numpy()
        np.testing.assert_array_equal(bits(m), bits(obox.iou_matrix(g[key], g[key])))
    np.testing.assert_array_equal(ops.iou3d_matrix(cu(g["aabb_boxes"]), cu(g["aabb_boxes"])).cpu().numpy(), g["aabb_iou"])
    rng = np.random.default_rng(6)
    a, b = rand_obb(37, rng, 12), rand_obb(301, rng, 12)          # ragged tile edges
    np.testing.assert_array_equal(bits(ops.iou3d_matrix(cu(a), cu(b)).cpu().numpy()), bits(obox.iou_matrix(a, b)))
    assert ops.iou3d_matrix(cu(a[:0]), cu(b)).shape == (0, 301)


def test_sort_vertices_dropin(ops, G):
    g = G["sort_vertices"]
    idx = ops.sort_vertices_forward(cu(g["vertices"]), cu(g["mask"], torch.bool), cu(g["num_valid"], torch.int32))
    assert idx.dtype == torch.int32 and tuple(idx.shape) == g["idx"].shape
    np.testing.assert_array_equal(idx.cpu().numpy(), g["idx"])
    np.testing.assert_array_equal(idx.cpu().numpy(), obox.sort_vertices(g["vertices"], g["mask"], g["num_valid"]))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.sort_vertices_forward(torch.zeros(1, 1, 24, 2), torch.zeros(1, 1, 24, dtype=torch.bool), torch.zeros(1, 1, dtype=torch.int32))


def run_nms(ops, boxes, scores, groups, thr):
    keep, nk = ops.nms_device(cu(boxes), cu(scores), None if groups is None else cu(groups, torch.int32), thr)
    return keep[: int(nk.item())].cpu().numpy()


@pytest.mark.parametrize("name", ["s64", "o700", "a1500"])
def test_nms_golden_sets(ops, G, name):
    g = G["nms"]
    b, s, lv = g[f"{name}_boxes"], g[f"{name}_scores"], g[f"{name}_levels"]
    np.testing.assert_array_equal(run_nms(ops, b, s, None, 0.3), g[f"{name}_keep"])
    np.testing.assert_array_equal(run_nms(ops, b, s, lv, 0.3), g[f"{name}_bkeep"])


def test_nms_vs_oracle_larger_and_edges(ops, G):
    rng = np.random.default_rng(7)
    for n, dim, ext in ((5000, 7, 60.0), (10000, 6, 90.0), (9999, 7, 40.0), (6000, 7, 12.0), (3072, 7, 30.0), (3073, 7, 30.0),
                        (65, 7, 5.0), (64, 6, 5.0), (1, 7, 5.0)):      # 6000 @ 12: heavy suppression (few survivors, long kept-list scans)
        boxes = rand_obb(n, rng, ext, 2, 14) if dim == 7 else rand_aabb(n, rng, ext, 2, 16)
        scores = rng.random(n).astype(np.float32)
        scores[: n // 10] = scores[n // 10: 2 * (n // 10)]           # exact score ties
        groups = rng.integers(0, 4, n).astype(np.int32)
        np.testing.assert_array_equal(run_nms(ops, boxes, scores, groups, 0.3), obox.batched_nms(boxes, scores, groups, 0.3))
        np.testing.assert_array_equal(run_nms(ops, boxes, scores, None, 0.5), obox.nms(boxes, scores, 0.5))
    keep, nk = ops.nms_device(torch.zeros((0, 7), device="cuda"), torch.zeros((0,), device="cuda"), None, 0.3)
    assert int(nk.item()) == 0 and keep.numel() == 0
    g = G["nms"]
    np.testing.assert_array_equal(run_nms(ops, g["o700_boxes"], g["o700_scores"], None, 0.5), g["o700_keep_t5"])


def test_nms_chunked_path_large_inputs(ops):
    """BASELINE config 5 sizes (beyond the 32 768-box bit-matrix path): exact against the oracle at 40k-70k boxes,
    size-independent properties at 300k (sorted by score, idempotent, kept set pairwise below the threshold)."""
    rng = np.random.default_rng(17)
    for n, dim, ext, ngroups in ((40000, 7, 200.0, 1), (50000, 7, 160.0, 4), (70000, 6, 260.0, 1), (66000, 7, 130.0, 1), (72000, 7, 180.0, 3)):   # >= 12 288: cell-list path
        boxes = rand_obb(n, rng, ext, 3, 24) if dim == 7 else rand_aabb(n, rng, ext, 3, 28)
        if dim == 7:
            boxes[:, 2] = rng.random(n) * ext * 0.625
        scores = rng.random(n).astype(np.float32)
        groups = rng.integers(0, ngroups, n).astype(np.int32) if ngroups > 1 else None
        got = run_nms(ops, boxes, scores, groups, 0.3)
        ref = obox.batched_nms(boxes, scores, groups, 0.3) if groups is not None else obox.nms(boxes, scores, 0.3)
        np.testing.assert_array_equal(got, ref)
    n = 300000
    boxes = rand_obb(n, rng, 256.0, 4, 48)
    boxes[:, 2] = rng.random(n) * 160.0
    scores = rng.random(n).astype(np.float32)
    keep = run_nms(ops, boxes, scores, None, 0.3)
    s = scores[keep]
    assert 1000 < keep.shape[0] < n and np.all(s[:-1] >= s[1:]) and np.unique(keep).shape[0] == keep.shape[0]
    again = run_nms(ops, boxes[keep], scores[keep], None, 0.3)
    np.testing.assert_array_equal(again, np.arange(keep.shape[0]))                   # idempotent
    sub = keep[:: max(1, keep.shape[0] // 1500)]
    m = obox.iou_matrix(boxes[sub], boxes[sub]); np.fill_diagonal(m, 0)
    assert np.nanmax(m) <= 0.3                                                        # survivors do not overlap beyond thr


def test_nms_cell_list_path_equals_chunked_kept_list_scan(ops, tmp_path):
    """n >= 12 288 runs the cell-list path (levels: cross against the kept boxes, adjacency among the survivors, dependency rounds); the keep
    list must equal the plain chunk-by-chunk kept-list scan (NRPN_NMS_CELLS=0, read when the library initialises: run in a second process)
    at 300 000 boxes, 2 groups, 40 degenerate boxes."""
    import subprocess, sys, textwrap
    rng = np.random.default_rng(23)
    n = 300000
    boxes = rand_obb(n, rng, 256.0, 4, 48)
    boxes[:, 2] = rng.random(n) * 160.0
    boxes[:40, 3] = 0.0                                       # degenerate boxes have no usable cull record: the "everywhere" cell
    scores = rng.random(n).astype(np.float32)
    groups = rng.integers(0, 2, n).astype(np.int32)
    np.savez(str(tmp_path / "in.npz"), boxes=boxes, scores=scores, groups=groups)
    keep = run_nms(ops, boxes, scores, groups, 0.3)
    code = textwrap.dedent(f"""
        import sys, numpy as np, torch
        sys.path.insert(0, {os.path.dirname(os.path.dirname(os.path.abspath(__file__)))!r})
        from nerf_rpn_b200 import ops
        from nerf_rpn_b200._lib import lib
        lib().nrpn_set_iou_mode(0)
        d = np.load({str(tmp_path / 'in.npz')!r})
        k, nk = ops.nms_device(torch.from_numpy(d['boxes']).cuda(), torch.from_numpy(d['scores']).cuda(), torch.from_numpy(d['groups']).cuda(), 0.3)
        np.save({str(tmp_path / 'ref.npy')!r}, k[: int(nk.item())].cpu().numpy())
    """)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, env={**os.environ, "NRPN_NMS_CELLS": "0"})
    assert r.returncode == 0, r.stderr[-2000:]
    ref = np.load(str(tmp_path / "ref.npy"))
    assert 1000 < ref.shape[0] < n
    np.testing.assert_array_equal(keep, ref)


def test_nms_cell_list_path_declines_crowds_and_handles_ties(ops):
    """More than 32 higher-scored overlapping survivors per box overflow the inline predecessor lists: the path must hand over to the chunked
    one (same keep set as the oracle), with 1 024-box chunks at 20 000 boxes and 4 096-box chunks at 70 000.  Exact score ties and long
    suppression chains stay on the cell-list path."""
    rng = np.random.default_rng(29)
    base = rand_obb(40, rng, 120.0, 8, 20)
    crowd = np.repeat(base, 500, axis=0) + rng.normal(0, 0.05, (20000, 7)).astype(np.float32)      # 500 near-copies of each of 40 boxes
    crowd[:, 3:6] = np.abs(crowd[:, 3:6])
    scores = rng.random(20000).astype(np.float32)
    np.testing.assert_array_equal(run_nms(ops, crowd, scores, None, 0.3), obox.nms(crowd, scores, 0.3))
    n = 18000                                                   # a chain: neighbours overlap at IoU ~ 0.54, scores fall along the chain
    chain = np.zeros((n, 7), np.float32)
    chain[:, 0] = np.arange(n) * 3.0; chain[:, 3:6] = 10.0
    s2 = np.linspace(1.0, 0.0, n).astype(np.float32)
    k = min(s2[::7].shape[0], s2[1::7].shape[0])
    s2[::7][:k] = s2[1::7][:k]                                  # ties
    np.testing.assert_array_equal(run_nms(ops, chain, s2, None, 0.3), obox.nms(chain, s2, 0.3))
    groups = rng.integers(0, 3, n).astype(np.int32)
    np.testing.assert_array_equal(run_nms(ops, chain, s2, groups, 0.3), obox.batched_nms(chain, s2, groups, 0.3))
    base = rand_obb(140, rng, 180.0, 8, 20)                     # a crowd above 65 536 boxes: 500 near-copies of each of 140 boxes
    crowd = np.repeat(base, 500, axis=0) + rng.normal(0, 0.05, (70000, 7)).astype(np.float32)
    crowd[:, 3:6] = np.abs(crowd[:, 3:6])
    scores = rng.random(70000).astype(np.float32)
    np.testing.assert_array_equal(run_nms(ops, crowd, scores, None, 0.3), obox.nms(crowd, scores, 0.3))


def test_nms_geometric_cull_modes_stay_within_a_few_boxes_of_the_exact_set(ops):
    """Cull modes 1 / 3 (opt-in, >= 16 384 boxes) bound the geometric IoU; the reference's vertex-sort quirk makes them differ from the exact keep set
    (mode 0) in ~1e-5 of the boxes.  100 000 boxes: symmetric difference of at most 5 boxes, and mode 0 is restored."""
    rng = np.random.default_rng(41)
    n = 100000
    boxes = rand_obb(n, rng, 256.0, 4, 48)
    boxes[:, 2] = rng.random(n) * 160.0
    scores = rng.random(n).astype(np.float32)
    exact = run_nms(ops, boxes, scores, None, 0.3)
    try:
        for mode in (1, 3):
            ops.set_nms_cull_mode(mode)
            got = run_nms(ops, boxes, scores, None, 0.3)
            assert np.setxor1d(got, exact).shape[0] <= 5, mode
    finally:
        ops.set_nms_cull_mode(0)
    assert lib_mode() == 0


def lib_mode():
    from nerf_rpn_b200._lib import lib
    return int(lib().nrpn_get_nms_cull_mode())


def _rpn_inputs_from_golden(r, rot):
    code = 8 if rot else 6
    A = 13
    preds, logits, deltas = [], [], []
    for l in range(4):
        lg, dl = r[f"logits{l}"], r[f"deltas{l}"]
        lg = np.transpose(lg, (1, 2, 3, 0)).reshape(-1, A)
        dl = np.transpose(dl.reshape(A, code, *dl.shape[1:]), (2, 3, 4, 0, 1)).reshape(-1, A * code)
        pad = np.zeros((lg.shape[0], 128 - A * (1 + code)), np.float32)
        preds.append(np.ascontiguousarray(np.concatenate([lg, dl, pad], 1)))
        logits.append(lg.reshape(-1)); deltas.append(dl.reshape(-1, code))
    return preds, logits, deltas


@pytest.mark.parametrize("name,rot", [("rpn_small_aabb", False), ("rpn_small_obb", True)])
def test_rpn_proposals_small(ops, G, name, rot):
    r = G[name]
    grids = [(8, 12, 10), (4, 6, 5), (2, 3, 3), (1, 2, 2)]
    mesh = (32, 48, 40)
    strides = [tuple(mesh[i] // gr[i] for i in range(3)) for gr in grids]
    cells = [rp.cell_anchors(s, ASPECT) for s in SIZES]
    preds, logits, deltas = _rpn_inputs_from_golden(r, rot)
    d = ops.make_rpn_desc([cu(p) for p in preds], grids, strides, cells, 13, rot, 2500, 2500, 0.3, 0.0, 1e-3, mesh)
    boxes, scores, levels, count = ops.rpn_proposals(d, torch.device("cuda"))
    k = int(count.item())
    ob, os_, ol = rp.rpn_proposals(logits, deltas, grids, strides, cells, mesh, rot)
    assert k == ob.shape[0] == r["proposals"].shape[0]
    np.testing.assert_array_equal(bits(boxes[:k].cpu().numpy()), bits(ob))          # bit-identical to the oracle
    np.testing.assert_array_equal(bits(scores[:k].cpu().numpy()), bits(os_))
    np.testing.assert_array_equal(levels[:k].cpu().numpy(), ol)
    np.testing.assert_allclose(boxes[:k].cpu().numpy(), r["proposals"], rtol=1e-5, atol=1e-4)   # and matches the reference
    np.testing.assert_array_equal(levels[:k].cpu().numpy(), r["level_index"])


@pytest.mark.parametrize("rot", [False, True])
def test_rpn_proposals_full_size_vs_oracle(ops, rot):
    """BASELINE config-2 sizes: 160x256x256 mesh, 2 433 600 anchors, top-2500 per level, NMS 0.3."""
    grids = [(40, 64, 64), (20, 32, 32), (10, 16, 16), (5, 8, 8)]
    mesh = (160, 256, 256)
    strides = [tuple(mesh[i] // gr[i] for i in range(3)) for gr in grids]
    cells = [rp.cell_anchors(s, ASPECT) for s in SIZES]
    code = 8 if rot else 6
    gen = torch.Generator(device="cuda").manual_seed(3)
    preds = []
    for gr in grids:
        v = gr[0] * gr[1] * gr[2]
        p = torch.zeros((v, 128), device="cuda")
        p[:, :13] = torch.randn((v, 13), device="cuda", generator=gen) * 2.0
        p[:, 13:13 + 13 * code] = torch.randn((v, 13 * code), device="cuda", generator=gen) * 0.3
        p[::7, 3] = p[::5, 3][: p[::7, 3].numel()]                   # exact logit ties
        preds.append(p.contiguous())
    d = ops.make_rpn_desc(preds, grids, strides, cells, 13, rot, 2500, 2500, 0.3, 0.0, 1e-3, mesh)
    boxes, scores, levels, count = ops.rpn_proposals(d, torch.device("cuda"))
    k = int(count.item())
    logits = [p[:, :13].reshape(-1).cpu().numpy() for p in preds]
    deltas = [p[:, 13:13 + 13 * code].reshape(-1, code).cpu().numpy() for p in preds]
    ob, os_, ol = rp.rpn_proposals(logits, deltas, grids, strides, cells, mesh, rot)
    assert k == ob.shape[0] and k > 100
    np.testing.assert_array_equal(bits(boxes[:k].cpu().numpy()), bits(ob))
    np.testing.assert_array_equal(bits(scores[:k].cpu().numpy()), bits(os_))
    np.testing.assert_array_equal(levels[:k].cpu().numpy(), ol)
    s = scores[:k].cpu().numpy()
    assert np.all(s[:-1] >= s[1:])                                   # size-independent property: sorted by score
