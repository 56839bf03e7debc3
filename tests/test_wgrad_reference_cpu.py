"""The float64 reference of the weight-gradient tests (tests/emulate.py:reference_wgrad64) against float64 torch.autograd of
F.conv3d, and negative controls: the bound of tests/test_gpu_wgrad_variants.py, 2^-24 |ref| + GAMMA mag, must reject a reference
with one deliberate mistake many times over on a small version (fewer channels, the same extents, levels and taps) of the table row
the mistake is aimed at."""
import dataclasses

import pytest
import torch
import torch.nn.functional as F

from tests import test_gpu_wgrad_variants as K
from tests.emulate import reference_wgrad64


def _close(a, b):
    torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)


def _autograd_wgrad(dys, xs, taps):
    """dW (taps, Cout, Cin) by float64 autograd.  Each level is a convolution of X with a (2P+1)^3 kernel that is zero outside the
    taps, cropped to dY's extent; a 'same' k^3 filter is F.conv3d(padding=k // 2) as it stands."""
    cout, cin = dys[0].shape[-1], xs[0].shape[-1]
    P = max(max(abs(v) for v in t) for t in taps)
    cube = len(taps) == (2 * P + 1) ** 3 and all(dy.shape[1:4] == x.shape[1:4] for dy, x in zip(dys, xs))
    w = torch.zeros((cout, cin, 2 * P + 1, 2 * P + 1, 2 * P + 1), dtype=torch.float64, requires_grad=True)
    for dy, x in zip(dys, xs):
        xc, g = x.double().permute(0, 4, 1, 2, 3), dy.double().permute(0, 4, 1, 2, 3)
        if cube:
            y = F.conv3d(xc, w, padding=P)
        else:
            ext = dy.shape[1:4]
            hi = [max(0, P + e - xe) for e, xe in zip(ext, x.shape[1:4])]
            y = F.conv3d(F.pad(xc, (P, hi[2], P, hi[1], P, hi[0])), w)[:, :, :ext[0], :ext[1], :ext[2]]
        y.backward(g)
    return torch.stack([w.grad[:, :, P + a, P + b, P + c] for a, b, c in taps])


CASES = {
    # name: cout, cin, taps, dY extents per level, X extent (one level) when it differs
    "k1_odd": (24, 16, 1, ((5, 3, 7),), None),
    "k3_odd": (16, 24, 3, ((5, 4, 3),), None),
    "k3_two_levels": (16, 8, 3, ((4, 5, 3), (3, 2, 2)), None),
    "k3_extent_1": (8, 16, 3, ((7, 1, 1),), None),
    "stem_taps_x_longer_along_z": (16, 16, "stem", ((3, 4, 3),), (3, 4, 4)),
    "two_taps_x_shorter": (8, 8, K.TWO_TAPS, ((4, 3, 5),), (3, 3, 4)),
}


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_reference_matches_autograd(name, dtype):
    cout, cin, taps, levels, x_ext = CASES[name]
    taps = K.row_taps(K.Row("", cout, cin, taps, levels))
    g = torch.Generator().manual_seed(len(name) * 31 + cout)
    dys = [torch.randn((2, *d, cout), generator=g).to(dtype) for d in levels]
    xs = [torch.randn((2, *(x_ext or d), cin), generator=g).to(dtype) for d in levels]
    x_dims = None if x_ext is None else [x_ext]
    ref, mag = reference_wgrad64(dys, xs, taps, x_dims)
    assert ref.dtype == torch.float64 and ref.shape == (len(taps), cout, cin)
    _close(ref, _autograd_wgrad(dys, xs, taps))
    want, _ = reference_wgrad64([d.abs() for d in dys], [x.abs() for x in xs], taps, x_dims)
    _close(mag, want)
    assert bool((ref.abs() <= mag).all())


def test_reference_refuses_an_x_extent_it_was_not_told():
    dy, x = torch.zeros((1, 3, 4, 5, 8)), torch.zeros((1, 3, 4, 6, 8))
    with pytest.raises(AssertionError, match="X extent"):
        reference_wgrad64([dy], [x], [(0, 0, 0)])
    reference_wgrad64([dy], [x], [(0, 0, 0)], x_dims=[(3, 4, 6)])


# ------------------------------------------------------------------------------------------------ negative controls
def _pick_box(extent, cap):
    """wgrad_plan's brick edge along one axis (csrc/conv3d_wgrad.cu: pick_box): the power of two in [1, cap] with the least
    overhang over `extent`, the larger one on ties."""
    best, waste, b = 1, None, 1
    while b <= cap:
        w = -(-extent // b) * b
        if waste is None or w <= waste:
            waste, best = w, b
        b *= 2
    return best


def _drop_brick(dys):
    """dY with one 64-voxel brick of the kernel's tiling (level 0, sample 0, the middle brick) zeroed; returns it and the number of
    real voxels the brick held."""
    dy = dys[0].clone()
    X, Y, Z = dy.shape[1:4]
    bz = _pick_box(Z, 64)
    by = _pick_box(Y, 64 // bz)
    bx = 64 // (bz * by)
    x0, y0, z0 = (-(-X // bx) // 2) * bx, (-(-Y // by) // 2) * by, (-(-Z // bz) // 2) * bz
    blk = dy[0, x0:x0 + bx, y0:y0 + by, z0:z0 + bz]
    real = blk.shape[0] * blk.shape[1] * blk.shape[2]
    blk.zero_()
    return [dy] + list(dys[1:]), real


CONTROLS = [
    # (flaw, row of tests/test_gpu_wgrad_variants.py it is aimed at)
    ("drop_brick", "c2_64_fp16"),
    ("drop_brick", "two_levels"),
    ("tap_shifted_along_z", "c2_64_fp16"),
    ("tap_shifted_along_z", "stem_like"),
    ("input_channels_swapped", "k1_64_256"),
    ("input_channels_swapped", "cin32_cout40"),
    ("level_left_out", "head_4_levels"),
    ("level_left_out", "predictor_fp16"),
    ("last_tap_group_dropped", "c2_64_fp16"),
    ("last_tap_group_dropped", "c2_128"),
    ("last_tap_group_dropped", "m2_t2_fp16"),
]


def _control_ratio(flaw, row):
    """Largest |flawed - ref| / bound over the row's dW, operands drawn on the CPU as the GPU test draws them."""
    taps = K.row_taps(row)
    dys, xs = K.operands(row, "cpu")
    ref, mag = K.reference(row, dys, xs, taps)
    if flaw == "drop_brick":
        bad_dys, real = _drop_brick(dys)
        assert real >= 8, f"the dropped brick holds {real} real voxels"
        bad, _ = K.reference(row, bad_dys, xs, taps)
    elif flaw == "tap_shifted_along_z":
        i = len(taps) // 2
        bad, _ = K.reference(row, dys, xs, taps[:i] + [(taps[i][0], taps[i][1], taps[i][2] + 1)] + taps[i + 1:])
    elif flaw == "input_channels_swapped":
        bad_xs = [x.clone() for x in xs]
        for x in bad_xs:
            x[..., [0, 1]] = x[..., [1, 0]]
        bad, _ = K.reference(row, dys, bad_xs, taps)
    elif flaw == "level_left_out":                   # the smallest level, the one with the least weight
        bad, _ = K.reference(dataclasses.replace(row, levels=row.levels[:-1]), dys[:-1], xs[:-1], taps)
    else:
        t_group = int(row.variant.split("/t")[1])
        last = len(taps) % t_group
        assert last, f"{row.variant} with {len(taps)} taps has no partial last group"
        bad = ref.clone()
        bad[-last:] = 0
    return float(((bad - ref).abs() / K.bound(ref, mag)).max())


@pytest.mark.parametrize("flaw,name", CONTROLS)
def test_bound_rejects_flawed_reference(flaw, name):
    row = K.ROWS[name]
    small = dataclasses.replace(row, cout=min(row.cout, 16), cin=min(row.cin, 16))
    ratio = _control_ratio(flaw, small)
    print(f"\n[control] {flaw:24s} on {name:16s} worst |flawed - ref| / bound {ratio:.3g}")
    assert ratio >= 16.0, f"{flaw} on {name}: only {ratio:.3g}x the bound"
