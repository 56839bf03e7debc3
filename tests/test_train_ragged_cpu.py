"""CPU: the per-anchor padding mask of a batch of differently sized scenes (nerf_rpn_b200/csrc/anchor_mask.cuh, the arithmetic of
nrpn_anchor_padding_mask) compiled for the host, element for element against the reference's own AnchorGenerator3D.get_padding_masks +
permute_and_flatten (RegionProposalNetwork.get_padding_masks) from the staged copy."""
import ctypes
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ref():
    from oracle import ref_gpu
    if not ref_gpu.available():
        pytest.skip("oracle/_ref not staged")
    stub = os.path.join(ROOT, "tools", "ref_stub")                 # import-time stand-in for the reference's native op on a CPU-only host
    sys.path.insert(0, stub)
    try:
        return ref_gpu.load(need_k1=False)
    finally:
        sys.path.remove(stub)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("shim") / "libanchor_mask_shim.so")
    subprocess.check_call(["g++", "-O1", "-shared", "-fPIC", "-o", out, os.path.join(ROOT, "tests", "host_shim", "anchor_mask_host.cpp")])
    lib = ctypes.CDLL(out)
    lib.shim_anchor_padding_mask.restype = ctypes.c_longlong
    return lib


def _levels(padded):
    """ResNet_FPN_256's P2..P5 extents for a padded grid: stem (s2), max-pool (s2), then stages 2..4 (s2 each)."""
    from nerf_rpn_b200.engine import _down
    d = _down(_down(tuple(padded)))
    out = [d]
    for _ in range(3):
        d = _down(d)
        out.append(d)
    return out


def _shim_masks(shim, ori_sizes, padded, grids, A):
    ori = np.ascontiguousarray(np.array(ori_sizes, np.int32).reshape(-1))
    gd = np.ascontiguousarray(np.array(grids, np.int32).reshape(-1))
    total = shim.shim_anchor_padding_mask(ori.ctypes.data_as(ctypes.c_void_p), len(ori_sizes), *padded, gd.ctypes.data_as(ctypes.c_void_p),
                                          len(grids), A, None)
    out = np.zeros((len(ori_sizes), total), np.uint8)
    shim.shim_anchor_padding_mask(ori.ctypes.data_as(ctypes.c_void_p), len(ori_sizes), *padded, gd.ctypes.data_as(ctypes.c_void_p), len(grids), A,
                                  out.ctypes.data_as(ctypes.c_void_p))
    return out


CASES = {
    # padded depth 130: the P2 grid is 33, so the reference's stride is 130 // 33 = 3 (not 4); one scene equals the padded size
    "depth130": [(130, 96, 64), (101, 96, 57)],
    # padded depth 65: P2 grid 17, stride 65 // 17 = 3; a scene of ONE voxel along x
    "depth65": [(40, 65, 30), (1, 20, 65)],
    # three scenes, odd extents, one voxel along z and along y
    "three": [(47, 33, 1), (20, 1, 41), (9, 12, 13)],
    # the longest side 160 of the reference's --resolution 160, two dataset-like scenes
    "res160": [(160, 124, 96), (112, 160, 80)],
}


@pytest.mark.parametrize("name", list(CASES))
def test_padding_mask_matches_reference(shim, name):
    ref = _ref()
    sizes = CASES[name]
    padded = tuple(max(s[a] for s in sizes) for a in range(3))
    grids = _levels(padded)
    ag = ref.anchor.AnchorGenerator3D(((8,), (16,), (32,), (64,)), (((1., 1., 1.), (1., 1., 2.), (1., 2., 2.), (1., 1., 3.), (1., 3., 3.)),) * 4)
    A = ag.num_anchors_per_location()[0]
    meshes = torch.empty((len(sizes), 4, *padded))
    feats = [torch.empty((len(sizes), 1, *g)) for g in grids]
    rpn_like = types.SimpleNamespace(anchor_generator=ag)
    want = ref.rpn.RegionProposalNetwork.get_padding_masks(rpn_like, meshes, feats, [torch.Size(s) for s in sizes]).numpy().astype(np.uint8)
    got = _shim_masks(shim, sizes, padded, grids, A)
    assert got.shape == want.shape
    assert np.array_equal(got, want), f"{int((got != want).sum())} of {got.size} anchors differ"
    # non-trivial: a padded scene has masked anchors, a scene of the padded size has none
    for i, s in enumerate(sizes):
        assert (got[i] == 0).any() == (tuple(s) != padded)
    if name in ("depth130", "depth65"):
        assert padded[0] // grids[0][0] == 3 or padded[1] // grids[0][1] == 3 or padded[2] // grids[0][2] == 3
