"""tests/emulate.py:reference_conv64 -- the float64 reference of the convolution kernel tests -- against F.conv3d and
F.interpolate in float64, so that the GPU tests rest on a reference that was itself checked."""
import math

import pytest
import torch
import torch.nn.functional as F

from nerf_rpn_b200 import packing
from tests.emulate import nearest_source_index, reference_conv64


def _torch_conv64(x, w, bias, k, stride, act, res):
    """Channels-last float64 F.conv3d ('same' padding for odd k) + bias + residual (nearest, size=...) + activation."""
    y = F.conv3d(x.double().permute(0, 4, 1, 2, 3), w.double(), bias.double(), stride=stride, padding=k // 2)
    if res is not None:
        r = res.float().permute(0, 4, 1, 2, 3)                # 16-bit values: exact in float32
        if r.shape[2:] != y.shape[2:]:
            r = F.interpolate(r, size=y.shape[2:], mode="nearest")      # float32 data: float32 scale, as the kernel
        y = y + r.double()
    if act == 1:
        y = F.relu(y)
    elif act == 2:
        y = F.gelu(y)                                        # exact (erf) form
    return y.permute(0, 2, 3, 4, 1)


@pytest.mark.parametrize("dims,cin,cout,k,stride,act,res_dims,dtype", [
    ((5, 7, 3), 64, 24, 3, 1, 0, None, torch.bfloat16),          # padding taps on every face, odd extents
    ((7, 5, 9), 64, 40, 3, 2, 1, None, torch.float16),           # stride 2 on odd extents (3^3 taps)
    ((9, 6, 1), 128, 16, 1, 2, 2, None, torch.bfloat16),         # stride-2 1^3 layer, extent 1
    ((13, 9, 4), 64, 16, 1, 1, 2, (7, 5, 2), torch.float16),     # residual up-sampled 7/13, 5/9, 2/4
    ((9, 13, 2), 64, 32, 3, 1, 1, (5, 7, 1), torch.bfloat16),    # 5/9, 7/13, 1/2
    ((4, 6, 5), 64, 32, 3, 1, 0, (4, 6, 5), torch.float16),      # same-extent residual
])
def test_reference_conv64_matches_torch(dims, cin, cout, k, stride, act, res_dims, dtype):
    g = torch.Generator().manual_seed(sum(dims) * 131 + cout)
    x = torch.randn((2, *dims, cin), generator=g).to(dtype)
    w = (torch.randn((cout, cin, k, k, k), generator=g) / math.sqrt(cin * k ** 3)).to(dtype)
    bias = torch.randn((cout,), generator=g)
    res = None if res_dims is None else torch.randn((2, *res_dims, cout), generator=g).to(dtype)
    wp, taps = packing.pack_conv_weight(w.float(), dtype=dtype)                      # exact: w is already 16-bit
    shift = packing.pad_shift(bias, wp.shape[1])
    od = tuple((d - 1) // stride + 1 for d in dims)
    ref, mag = reference_conv64(x, wp, taps, shift, od, stride=stride, act=act, res=res)
    assert ref.dtype == torch.float64 and ref.shape == (2, *od, wp.shape[1])
    want = _torch_conv64(x, w, bias, k, stride, act, res)
    torch.testing.assert_close(ref[..., :cout], want, rtol=1e-12, atol=1e-12)
    assert torch.equal(ref[..., cout:], torch.zeros_like(ref[..., cout:]))          # zero weight / shift padding
    # mag is the same sum over |terms|: it bounds the pre-activation value and equals the conv of the absolute operands
    pre, _ = reference_conv64(x, wp, taps, shift, od, stride=stride, act=0, res=res)
    assert bool((pre.abs() <= mag * (1 + 1e-12)).all())
    want_mag = _torch_conv64(x.abs(), w.abs(), bias.abs(), k, stride, 0, None if res is None else res.abs())
    torch.testing.assert_close(mag[..., :cout], want_mag, rtol=1e-12, atol=1e-12)


def test_reference_conv64_sums_split_weight_planes():
    """wsplit weights (taps, 2, CoutPad, Cin): the kernel multiplies both planes with the same activations, so the reference is
    the conv with hi + lo summed in float64 (not the 16-bit sum)."""
    g = torch.Generator().manual_seed(5)
    x = torch.randn((1, 4, 5, 3, 64), generator=g).to(torch.float16)
    w = torch.randn((32, 64, 3, 3, 3), generator=g) / math.sqrt(64 * 27)
    ws, taps = packing.pack_conv_weight(w, dtype=torch.float16, split=True)
    shift = torch.zeros(ws.shape[-2])
    ref, mag = reference_conv64(x, ws, taps, shift, (4, 5, 3))
    wsum = ws[:, 0].double() + ws[:, 1].double()                                 # (27 taps, CoutPad 64, Cin 64)
    assert not torch.equal(wsum, ws[:, 0].double())
    want = _torch_conv64(x, wsum.view(3, 3, 3, 64, 64).permute(3, 4, 0, 1, 2)[:32], torch.zeros(32), 3, 1, 0, None)
    torch.testing.assert_close(ref[..., :32], want, rtol=1e-12, atol=1e-12)
    absw = ws[:, 0].double().abs() + ws[:, 1].double().abs()
    m2, _ = reference_conv64(x.abs(), absw, taps, shift, (4, 5, 3))
    torch.testing.assert_close(mag, m2, rtol=0, atol=0)


@pytest.mark.parametrize("out_size,in_size", [(13, 7), (9, 5), (46, 14), (16, 8), (10, 3), (6, 6), (5, 1)])
def test_nearest_source_index_matches_interpolate(out_size, in_size):
    """The residual gather index equals F.interpolate(size=...) on float32 data, whose scale is float32 as in the kernel.  At
    14 -> 46 an exact (float64) scale picks voxel 7 for output 23 instead of 6."""
    def interp(dtype):
        src = torch.arange(in_size, dtype=dtype).view(1, 1, in_size, 1, 1)
        return F.interpolate(src, size=(out_size, 1, 1), mode="nearest").view(-1).to(torch.int64)
    got = nearest_source_index(out_size, in_size)
    assert torch.equal(got, interp(torch.float32))
    if (out_size, in_size) == (46, 14):
        exact = [min(math.floor(o * in_size / out_size), in_size - 1) for o in range(out_size)]
        assert got[23] == 6 and exact[23] == 7
