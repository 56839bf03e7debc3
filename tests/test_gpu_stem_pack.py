"""GPU: the stem packing (nrpn_pack_stem_input) of every input layout against the pure-torch statement of its row layout,
tests/emulate.py:emulate_pack_stem, bit for bit after 16-bit rounding, at odd extents."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.emulate import emulate_pack_stem
from tests.test_gpu_train_ragged import _alpha, _pad_stack, _scene

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]


def _rand(shape, seed):
    """fp32 on the host: RGB-like values and signed densities of either sign, so both roundings see varied bits."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g) * 3.0


def _check(got, grid_f32, dtype):
    """got: the packed rows on the device; grid_f32: the (N,4,X,Y,Z) fp32 host grid they must equal after 16-bit rounding."""
    want = emulate_pack_stem(grid_f32.contiguous()).to(dtype)
    torch.cuda.synchronize()
    assert got.dtype == dtype and tuple(got.shape) == tuple(want.shape)
    assert torch.equal(got.cpu().view(torch.int16), want.view(torch.int16))


@pytest.mark.parametrize("dtype", DTYPES)
def test_stacked_ncdhw(dtype):
    from nerf_rpn_b200 import ops
    x = _rand((2, 4, 21, 19, 27), 1)
    _check(ops.pack_stem_input(x.cuda(), dtype=dtype), x, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_stacked_channels_last_view(dtype):
    from nerf_rpn_b200 import ops
    xyzc = _rand((2, 21, 19, 27, 4), 2)                                  # the dataset's view: memory (N,X,Y,Z,4)
    _check(ops.pack_stem_input(xyzc.cuda().permute(0, 4, 1, 2, 3), dtype=dtype), xyzc.permute(0, 4, 1, 2, 3), dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_stacked_uint8(dtype):
    from nerf_rpn_b200 import ops
    g = torch.Generator().manual_seed(3)
    raw = torch.randint(0, 256, (2, 21, 19, 27, 4), generator=g, dtype=torch.uint8)
    ref = raw.permute(0, 4, 1, 2, 3).float() / 255.0                     # datasets.py:59-61, correctly rounded fp32 division on the host
    _check(ops.pack_stem_input(raw.cuda().permute(0, 4, 1, 2, 3), dtype=dtype), ref, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_ragged_list_mixed_layouts(dtype):
    """Differently sized scenes, NCDHW and channels-last views mixed, against the batch the reference builds: zero-padded with torch and stacked."""
    from nerf_rpn_b200 import ops
    dims = [(13, 20, 9), (17, 11, 15), (7, 19, 21)]
    host = [_rand((*d, 4), 10 + i).permute(3, 0, 1, 2) for i, d in enumerate(dims)]
    scenes = [h.contiguous().cuda() if i == 1 else h.permute(1, 2, 3, 0).cuda().permute(3, 0, 1, 2) for i, h in enumerate(host)]
    assert ops.is_channels_last_grid(scenes[0]) and scenes[1].is_contiguous() and ops.is_channels_last_grid(scenes[2])
    X, Y, Z = ops.padded_extent(host)
    padded = torch.stack([F.pad(h, (0, Z - h.shape[3], 0, Y - h.shape[2], 0, X - h.shape[1])) for h in host])
    _check(ops.pack_stem_input(scenes, dtype=dtype), padded, dtype)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("alpha", [False, True])
def test_ragged_stem_packing_bit_identical(dtype, alpha):
    """The list path against the stacked path on the batch padded with torch, with and without the fused density_to_alpha map."""
    from nerf_rpn_b200 import ops
    dims = [(13, 20, 9), (17, 11, 15), (7, 19, 21)]
    scenes = [_scene(d, 10 + i, cl) for i, (d, cl) in enumerate(zip(dims, (True, False, True)))]
    got = ops.pack_stem_input(scenes, dtype=dtype, density_to_alpha=alpha)
    if alpha:
        # the fused map on the stacked padded batch whose padding maps to exactly 0 (density -inf): the same bits.  (A map computed
        # on the host -- torch or numpy exp -- differs from the kernel's expf in the last fp32 bit now and then, which can flip a 16-bit rounding.)
        want = ops.pack_stem_input(_pad_stack(scenes, value_density=-math.inf), dtype=dtype, density_to_alpha=True)
    else:
        want = ops.pack_stem_input(_pad_stack(scenes), dtype=dtype)          # F.pad -> torch.stack -> the stacked packing
    torch.cuda.synchronize()
    assert got.shape == want.shape == (3, 9, 10, 12, 64)
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))
    if alpha:
        torch_map = ops.pack_stem_input(_pad_stack([_alpha(s) for s in scenes]), dtype=dtype)
        assert (got.float() - torch_map.float()).abs().max().item() <= (2.0 ** -10 if dtype == torch.float16 else 2.0 ** -7)
        # numpy's map (BaseDataset.density_to_alpha on the host): within one 16-bit ulp of values in [0, 1]
        host = []
        for s in scenes:
            a = s.cpu().numpy().copy()
            a[3] = np.clip(1.0 - np.exp(-np.exp(a[3]) / 100.0), 0.0, 1.0)
            host.append(torch.from_numpy(a).cuda())
        ref_np = ops.pack_stem_input(_pad_stack(host), dtype=dtype)
        assert (got.float() - ref_np.float()).abs().max().item() <= (2.0 ** -10 if dtype == torch.float16 else 2.0 ** -7)
    # the padding is exactly zero: scene 2 (x extent 7 -> 4 packed rows of 9) has nothing beyond x row 4, scene 1 (y 11) nothing beyond y row 6
    assert not got[2, 4:].any() and not got[1, :, 6:].any()
    assert got[2, :4].any() and got[1, :, :6].any()


@pytest.mark.parametrize("dtype", DTYPES)
def test_more_scenes_than_one_launch_holds(dtype):
    """A stacked batch has no scene limit: 33 scenes take two launches and equal the scenes packed one at a time."""
    from nerf_rpn_b200 import ops
    from nerf_rpn_b200._lib import STEM_MAX_SCENES, lib
    n = STEM_MAX_SCENES + 1
    x = _rand((n, 5, 6, 7, 4), 4).cuda().permute(0, 4, 1, 2, 3)
    before = lib().nrpn_launch_count()
    got = ops.pack_stem_input(x, dtype=dtype)
    assert lib().nrpn_launch_count() - before == 2
    one_by_one = torch.cat([ops.pack_stem_input(x[i:i + 1], dtype=dtype) for i in range(n)])
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int16), one_by_one.view(torch.int16))


def test_uint8_refuses_density_to_alpha():
    from nerf_rpn_b200 import ops
    raw = torch.zeros((1, 6, 6, 6, 4), dtype=torch.uint8, device="cuda").permute(0, 4, 1, 2, 3)
    with pytest.raises(NotImplementedError, match="uint8 grids hold alphas already"):
        ops.pack_stem_input(raw, density_to_alpha=True)
