"""CPU: the C-ABI library loads without a GPU, exports every entry point include/nerf_rpn_b200.h declares, and the
ctypes mirror of its structs has the C layout.  No compute calls here."""
import ctypes
import os
import re
import subprocess
import tempfile

import pytest

from nerf_rpn_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "nerf_rpn_b200.h")


def test_library_loads_and_exports_header_symbols():
    L = _lib.lib()
    src = open(HEADER).read()
    declared = sorted(set(re.findall(r"\b(nrpn_[a-z0-9_]+)\s*\(", src)))
    assert len(declared) >= 16
    for name in declared:
        assert hasattr(L, name), f"{name} declared in the header but not exported"
    assert sorted(_lib.exported_symbols()) == declared            # the ctypes table covers exactly the header
    assert L.nrpn_version() >= 100
    assert L.nrpn_status_string(0) == b"ok" and L.nrpn_status_string(-3) == b"workspace too small"


def test_host_only_queries():
    L = _lib.lib()
    assert [L.nrpn_conv3d_block_n(c) for c in (8, 64, 72, 128, 256, 2048)] == [64, 64, 128, 128, 256, 256]
    assert L.nrpn_nms_max_boxes() >= 10000
    assert L.nrpn_nms_workspace_bytes(10000) > 10000 * 157 * 8
    assert L.nrpn_nms_workspace_bytes(0) > 0


def test_conv_variant_query_needs_no_device():
    """nrpn_conv3d_variant names the exact instance nrpn_conv3d_fprop launches (the epilogue included) and refuses what it refuses."""
    L = _lib.lib()
    d = _lib.ConvDesc()
    d.cin, d.cout, d.stride, d.n_levels = 256, 256, 1, 1
    taps = [(a, b, c) for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1)]
    d.n_taps = len(taps)
    for t, off in enumerate(taps):
        d.tap_off[t][0], d.tap_off[t][1], d.tap_off[t][2] = off
    d.w, d.shift = 1 << 32, 2 << 32                                 # pointers are checked, never dereferenced
    lv = d.level[0]
    lv.x, lv.y, lv.n, lv.ldy = 3 << 32, 4 << 32, 1, 256
    lv.xi, lv.yi, lv.zi = lv.xo, lv.yo, lv.zo = (40, 48, 64)
    name = lambda: L.nrpn_conv3d_variant(ctypes.byref(d)).decode()
    assert name() == "igemm<256,4,1,tma-epilogue>"
    d.out_fp32 = 1
    assert name() == "igemm<256,4,1>"
    d.stride = 2                                                    # strided taps must not move
    assert name() == "unsupported"
    d.stride, lv.x = 1, 0
    assert name() == "invalid"


def test_ctypes_struct_layouts_match_header():
    code = r'''
#include <stdio.h>
#include <stddef.h>
#include "nerf_rpn_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", offsetof(nrpn_conv_desc, act_fp16), offsetof(nrpn_conv_desc, wsplit),
         sizeof(nrpn_conv_level), sizeof(nrpn_conv_desc), offsetof(nrpn_conv_desc, stride),
         offsetof(nrpn_conv_desc, w), offsetof(nrpn_conv_desc, level), sizeof(nrpn_rpn_level), sizeof(nrpn_rpn_desc),
         offsetof(nrpn_rpn_desc, cell_anchors), offsetof(nrpn_rpn_desc, nms_thresh), offsetof(nrpn_rpn_desc, valid));
  printf("%zu %zu %zu %zu %zu %zu\n", sizeof(nrpn_wgrad_level), sizeof(nrpn_wgrad_desc), offsetof(nrpn_wgrad_desc, level),
         offsetof(nrpn_wgrad_desc, dw), offsetof(nrpn_wgrad_desc, workspace_bytes), offsetof(nrpn_wgrad_desc, dw_layout));
  printf("%zu %zu %zu %d %d %d %d\n", sizeof(nrpn_stem_src), offsetof(nrpn_stem_src, x), offsetof(nrpn_stem_src, layout),
         NRPN_STEM_MAX_SCENES, NRPN_STEM_F32_NCDHW, NRPN_STEM_F32_XYZC, NRPN_STEM_U8_XYZC);
  return 0; }'''
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "t.c"), os.path.join(d, "t")
        open(src, "w").write(code)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
        vals = [int(v) for v in subprocess.check_output([exe]).split()]
    C, R, W, S = _lib.ConvDesc, _lib.RpnDesc, _lib.WgradDesc, _lib.StemSrc
    mine = [C.act_fp16.offset, C.wsplit.offset, ctypes.sizeof(_lib.ConvLevel), ctypes.sizeof(C), C.stride.offset, C.w.offset, C.level.offset,
            ctypes.sizeof(_lib.RpnLevel), ctypes.sizeof(R), R.cell_anchors.offset, R.nms_thresh.offset, R.valid.offset,
            ctypes.sizeof(_lib.WgradLevel), ctypes.sizeof(W), W.level.offset, W.dw.offset, W.workspace_bytes.offset, W.dw_layout.offset,
            ctypes.sizeof(S), S.x.offset, S.layout.offset, _lib.STEM_MAX_SCENES, _lib.STEM_F32_NCDHW, _lib.STEM_F32_XYZC, _lib.STEM_U8_XYZC]
    assert mine == vals


def test_stem_pack_validates_every_scene_before_launching():
    """nrpn_pack_stem_input refuses a bad scene anywhere in the table (here the second) on the host: the pointers are checked, never
    dereferenced, and nothing is launched."""
    L = _lib.lib()
    base = 1 << 32

    def status(layout, grid=base, extent=(4, 4, 4), alpha=0):
        src = (_lib.StemSrc * 2)()
        src[0].grid, src[0].layout, src[0].x, src[0].y, src[0].z = base, _lib.STEM_F32_XYZC, 6, 6, 6
        src[1].grid, src[1].layout = grid, layout
        src[1].x, src[1].y, src[1].z = extent
        before = L.nrpn_launch_count()
        st = L.nrpn_pack_stem_input(src, 2, base, 0, alpha, None)
        assert L.nrpn_launch_count() == before
        return st

    assert status(_lib.STEM_U8_XYZC, alpha=1) == -1                      # uint8 grids hold alphas already
    assert status(_lib.STEM_U8_XYZC, grid=base + 2) == -1                # 32-bit voxel loads
    assert status(_lib.STEM_F32_XYZC, grid=base + 4) == -1               # 128-bit voxel loads
    assert status(3) == -1                                               # no such layout
    assert status(_lib.STEM_F32_NCDHW, grid=0) == -1
    assert status(_lib.STEM_F32_NCDHW, extent=(4, 0, 4)) == -1


def test_missing_library_fails_loudly(monkeypatch):
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", "/nonexistent/libnerf_rpn_b200.so")
    with pytest.raises(_lib.NativeLibraryError, match="no CPU / PyTorch fallback"):
        _lib.lib()


def test_ops_reject_cpu_tensors():
    import torch
    from nerf_rpn_b200 import ops
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.iou3d_pairs(torch.zeros(2, 7), torch.zeros(2, 7))
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.pack_stem_input(torch.zeros(1, 4, 4, 4, 4))
