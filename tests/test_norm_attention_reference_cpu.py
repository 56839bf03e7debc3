"""The float64 references of the Swin-3D and GroupNorm kernel tests (tests/emulate.py) against oracle/net.py and torch in
float64, and negative controls: each bound of tests/test_gpu_swin_gn_kernels.py, evaluated on the reference's own scale, must
reject a reference with one deliberate mistake by at least 4x on the row the mistake is aimed at."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import net as onet
from tests import test_gpu_swin_gn_kernels as K
from tests.emulate import (MERGE_PARITY, _relative_position_index, reference_groupnorm64, reference_layernorm64,
                           reference_patch_embed, reference_patch_merge64, reference_window_attention64)

EPS = K.EPS


def _close(a, b):
    torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)


def _oracle_attention(qkv, bias16, table, heads, shift):
    """oracle/net.py:_window_attention in float64 with identity projections, fed so that its q / k / v are exactly the given
    16-bit ones: the input is qkv - bias (3C wide), so that the Linear gives qkv on real tokens and the bias on the zero padding.
    The oracle splits its qkv output into 3 heads-of-32 groups as wide as its input, so it runs 3 * heads heads: its qkv weight
    selects [q q q | k k k | v v v] and its table is the given one three times; each copy of a head computes the same output."""
    C = heads * 32
    eye = torch.eye(C, dtype=torch.float64)
    sel = torch.zeros((9 * C, 3 * C), dtype=torch.float64)
    for part in range(3):
        for r in range(3):
            sel[(3 * part + r) * C:(3 * part + r + 1) * C, part * C:(part + 1) * C] = eye
    sd = {"a.qkv.weight": sel, "a.qkv.bias": sel @ bias16, "a.proj.weight": torch.eye(3 * C, dtype=torch.float64),
          "a.proj.bias": torch.zeros(3 * C, dtype=torch.float64), "a.relative_position_bias_table": torch.cat([table.double()] * 3, 1),
          "a.relative_position_index": _relative_position_index()}
    out = onet._window_attention(qkv[..., :3 * C].double() - bias16, sd, "a", 3 * heads, shift)
    assert torch.equal(out[..., :C], out[..., C:2 * C]) and torch.equal(out[..., :C], out[..., 2 * C:])
    return out[..., :C]


@pytest.mark.parametrize("dims,heads,shift,dtype", [
    ((8, 8, 8), 2, 0, torch.bfloat16),
    ((8, 12, 8), 1, 2, torch.float16),          # shifted on every axis, no padding
    ((5, 7, 3), 2, 2, torch.float16),           # padding on every axis, shifted on every axis
    ((5, 7, 4), 1, 0, torch.float16),           # padding, no shift
    ((3, 4, 2), 1, 2, torch.bfloat16),          # every padded extent is 4: the shift is dropped on every axis
    ((7, 7, 4), 2, 2, torch.float16),           # config 3 stage 4: shifted on H and W, not on D
    ((9, 3, 4), 1, 2, torch.bfloat16),          # only H shifted
])
def test_attention_reference_matches_oracle(dims, heads, shift, dtype):
    C = heads * 32
    g = torch.Generator().manual_seed(sum(dims) * 7 + heads + shift)
    qkv = torch.full((2, *dims, 3 * C + 8), float("nan"), dtype=dtype)               # columns past 3C are never read
    qkv[..., :3 * C] = torch.randn((2, *dims, 3 * C), generator=g).to(dtype)
    bias = torch.randn(3 * C, generator=g) * 0.3
    table = torch.randn((343, heads), generator=g) * 0.5
    ref, scale = reference_window_attention64(qkv, bias, table, heads, shift, dtype)
    assert ref.dtype == torch.float64 and ref.shape == (2, *dims, C)
    _close(ref, _oracle_attention(qkv, bias.to(dtype).double(), table, heads, shift))
    # scale = sum_j p_j |v_j|: p does not depend on v, so it is the output for |v| (and |v| padding tokens)
    qkv_abs, bias_abs = qkv.clone(), bias.clone()
    qkv_abs[..., 2 * C:3 * C] = qkv_abs[..., 2 * C:3 * C].abs()
    bias_abs[2 * C:] = bias_abs[2 * C:].abs()
    want, _ = reference_window_attention64(qkv_abs, bias_abs, table, heads, shift, dtype)
    _close(scale, want)
    assert bool((ref.abs() <= scale * (1 + 1e-12)).all())


@pytest.mark.parametrize("C,ld,dtype", [(96, 128, torch.float16), (192, 192, torch.bfloat16), (384, 448, torch.float16)])
def test_layernorm_reference_matches_torch(C, ld, dtype):
    g = torch.Generator().manual_seed(C)
    x = torch.full((2, 5, 3, 4, ld), float("nan"), dtype=dtype)
    x[..., :C] = (torch.randn((2, 5, 3, 4, C), generator=g) * 2 + 0.3).to(dtype)
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    ref, scale = reference_layernorm64(x, C, gamma, beta, EPS)
    _close(ref, F.layer_norm(x[..., :C].double(), (C,), gamma.double(), beta.double(), EPS))
    assert bool((ref.abs() <= scale).all())


@pytest.mark.parametrize("dims,C,dtype", [((4, 6, 2), 96, torch.bfloat16), ((5, 6, 4), 96, torch.float16),
                                          ((4, 7, 4), 192, torch.float16), ((4, 6, 3), 96, torch.bfloat16),
                                          ((5, 7, 3), 384, torch.float16)])
def test_patch_merge_reference_matches_oracle(dims, C, dtype):
    """Against oracle/net.py's PatchMerging front half (pad odd extents with zeros, gather in parity order, LayerNorm(8C))."""
    g = torch.Generator().manual_seed(sum(dims) + C)
    x = torch.full((2, *dims, C + 64), float("nan"), dtype=dtype)
    x[..., :C] = (torch.randn((2, *dims, C), generator=g) * 2 + 0.3).to(dtype)
    gamma, beta = torch.rand(8 * C, generator=g) + 0.5, torch.randn(8 * C, generator=g)
    ref, scale = reference_patch_merge64(x, C, gamma, beta, EPS)
    h = x[..., :C].double()
    H, W, D = h.shape[1:4]
    hp = F.pad(h, (0, 0, 0, D % 2, 0, W % 2, 0, H % 2))
    parts = [hp[:, i::2, j::2, k::2, :] for (i, j, k) in ((0, 0, 0), (1, 0, 0), (0, 1, 0), (1, 1, 0), (0, 0, 1), (1, 0, 1), (0, 1, 1), (1, 1, 1))]
    assert tuple(MERGE_PARITY) == ((0, 0, 0), (1, 0, 0), (0, 1, 0), (1, 1, 0), (0, 0, 1), (1, 0, 1), (0, 1, 1), (1, 1, 1))
    _close(ref, F.layer_norm(torch.cat(parts, -1), (8 * C,), gamma.double(), beta.double(), EPS))
    assert bool((ref.abs() <= scale).all())


@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_groupnorm_reference_matches_torch(dtype, relu):
    g = torch.Generator().manual_seed(11 + int(relu))
    levels = [(torch.randn((2, *d, 256), generator=g) * 3 + 0.7).to(dtype) for d in ((6, 5, 4), (3, 2, 2), (1, 2, 2))]
    gamma, beta = torch.rand(256, generator=g) + 0.5, torch.randn(256, generator=g)
    refs, scales = reference_groupnorm64(levels, gamma, beta, EPS, relu)
    for x, ref, scale in zip(levels, refs, scales):
        want = F.group_norm(x.double().permute(0, 4, 1, 2, 3), 32, gamma.double(), beta.double(), EPS).permute(0, 2, 3, 4, 1)
        _close(ref, F.relu(want) if relu else want)
        assert bool((ref.abs() <= scale).all())


def test_patch_embed_reference_is_the_conv_as_a_gemm():
    """reference_patch_embed rows times the Conv3d(4, C, 4, stride 4) weight flattened to (C, 256) give the convolution."""
    g = torch.Generator().manual_seed(3)
    grid = torch.randn((2, 4, 21, 18, 14), generator=g)
    w = torch.randn((40, 4, 4, 4, 4), generator=g, dtype=torch.float64)
    rows = reference_patch_embed(grid)
    assert rows.shape == (2, 5, 4, 3, 256) and rows.dtype == torch.float64
    _close(rows @ w.reshape(40, 256).t(), F.conv3d(grid.double(), w, stride=4).permute(0, 2, 3, 4, 1))
    i, j, k, c, px, py, pz = 4, 2, 1, 3, 1, 2, 3
    assert rows[1, i, j, k, ((c * 4 + px) * 4 + py) * 4 + pz] == grid[1, c, 4 * i + px, 4 * j + py, 4 * k + pz]


# ------------------------------------------------------------------------------------------------ negative controls
CONTROLS = [
    # (flaw, row of tests/test_gpu_swin_gn_kernels.py it is aimed at)
    ("mask_h_omitted", "attn_s7_c768_mixed_shift_bf16"),
    ("mask_unshifted_axes", "attn_s7_c768_mixed_shift_bf16"),
    ("index_transposed", "attn_s7_c768_mixed_shift_bf16"),
    ("pad_zero", "attn_s7_c768_mixed_shift_bf16"),
    ("no_scale", "attn_s7_c768_mixed_shift_bf16"),
    ("unbiased", "ln_c96_bf16"),
    ("swap_100_010", "merge_c96_odd_all_bf16"),
    ("edge_replicate", "merge_c96_odd_all_bf16"),
    ("unbiased", "gn_4_voxels"),
    ("group_mod32", "gn_small_bf16"),
    ("pooled", "gn_small_bf16"),
]


def _control_ratio(flaw, row):
    """Largest |flawed - ref| / bound over the row's outputs, operands drawn on the CPU as the GPU test draws them."""
    dt = K.DTYPE[row.dtype]
    if isinstance(row, K.Attn):
        C = row.heads * 32
        qkv, bias, table = K.attention_operands(row, "cpu")
        ref, scale = reference_window_attention64(qkv, bias, table, row.heads, row.shift, dt)
        bad, _ = reference_window_attention64(qkv, bias, table, row.heads, row.shift, dt, flaw=flaw)
        return float(((bad - ref).abs() / K.attention_bound(ref, scale, dt, K.attention_vmax(qkv, bias, C, dt))).max())
    if isinstance(row, K.LayerNorm):
        x, gamma, beta = K.layernorm_operands(row, "cpu")
        ref, scale = reference_layernorm64(x, row.c, gamma, beta, EPS)
        bad, _ = reference_layernorm64(x, row.c, gamma, beta, EPS, flaw=flaw)
        return float(((bad - ref).abs() / K.norm_bound(ref, scale, dt, K.layernorm_terms(row.c))).max())
    if isinstance(row, K.Merge):
        x, gamma, beta = K.merge_operands(row, "cpu")
        ref, scale = reference_patch_merge64(x, row.c, gamma, beta, EPS)
        bad, _ = reference_patch_merge64(x, row.c, gamma, beta, EPS, flaw=flaw)
        return float(((bad - ref).abs() / K.norm_bound(ref, scale, dt, K.layernorm_terms(8 * row.c))).max())
    levels, gamma, beta = K.groupnorm_operands(row, "cpu")
    refs, scales = reference_groupnorm64(levels, gamma, beta, EPS, row.relu)
    bads, _ = reference_groupnorm64(levels, gamma, beta, EPS, row.relu, flaw=flaw)
    return max(float(((b - r).abs() / K.norm_bound(r, s, dt, K.groupnorm_terms(math.prod(d)))).max())
               for b, r, s, d in zip(bads, refs, scales, row.levels))


@pytest.mark.parametrize("flaw,name", CONTROLS)
def test_bound_rejects_flawed_reference(flaw, name):
    row = K.ROWS[name]
    ratio = _control_ratio(flaw, row)
    print(f"\n[control] {flaw:20s} on {name:32s} worst |flawed - ref| / bound {ratio:.3g}")
    assert ratio >= 4.0, f"{flaw} on {name}: only {ratio:.3g}x the bound"


def test_control_rows_exercise_their_flaw():
    """The mixed-shift row is shifted on H and W only and pads H and W; the GroupNorm unbiased-variance row has 4 voxels (a group
    of 32 values: N - 1 vs N is a 3 % change); the patch-merge edge row is odd on every axis; the pooled row has two samples."""
    attn = K.ROWS["attn_s7_c768_mixed_shift_bf16"]
    padded = [-(-e // 4) * 4 for e in attn.dims]
    assert [0 if 4 >= p else attn.shift for p in padded] == [2, 2, 0] and attn.heads == 24
    assert padded[:2] != list(attn.dims[:2])
    assert math.prod(K.ROWS["gn_4_voxels"].levels[0]) == 4
    assert all(e % 2 for e in K.ROWS["merge_c96_odd_all_bf16"].dims)
    assert K.ROWS["gn_small_bf16"].n == 2
