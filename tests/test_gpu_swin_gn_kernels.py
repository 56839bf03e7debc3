"""The Swin-3D kernels (csrc/swin.cu: window attention, LayerNorm, patch merging, patch embedding) and the FCOS GroupNorm + ReLU
(csrc/groupnorm.cu) against the float64 references of tests/emulate.py, in both 16-bit activation formats (bf16, and fp16 as
the default precision fp16_w2 runs them).

One table of named rows.  Every row draws its operands from a generator seeded by the row itself and checks:
  - nothing unwritten, nothing over-written: outputs are NaN-filled inside NaN guard bands (GUARD elements before and after);
    afterwards every element the kernel must write is finite and within bound, and every other element -- the guard bands and
    the pad channels [C, ld) of the output rows -- is still the same NaN, bit for bit;
  - nothing read that is not an operand: input pad channels (and the columns of qkv past 3C) are NaN, so reading one would
    put a NaN into the output;
  - a per-element bound, u = half an ulp of the output format (2^-8 bf16, 2^-11 fp16) and scale from the reference:

  window attention     |got - ref| <= u |ref| + 2u scale + [fp16 only] 2^-19 vmax + 2^-24,   scale = sum_j p_j |v_j|
      The kernel stores the un-normalised probabilities e_j = exp(s_j - max) <= 1 as 16-bit values and divides the fp32 P.V by
      the fp32 sum of the unrounded e_j, which is >= 1.  Rounding e_j costs at most u e_j, so u scale over the row.  In fp16
      an e_j below 2^-14 is subnormal and its absolute error is up to 2^-25 instead: at most 2^-25 * 64 vmax = 2^-19 vmax over
      a window's 64 keys, vmax the largest |v| the launch reads.  The rest is fp32: the 32-term q.k, the scale and bias adds,
      __expf (about 2^-21 + |s - max| 2^-24 relative) and the 64-term P.V and sum; with scores spanning +-30 that stays below
      2^-16 scale, so the second u of 2u covers it 32 times over in fp16.  Last the output is rounded to 16 bits: u |ref|.
  LayerNorm, patch merge   |got - ref| <= u |ref| + (K/32 + 32) 2^-24 scale + 2^-24,   K the normalised row length (C or 8C),
      scale = |gamma| (|x_hat| + mean|x| / sigma) + |beta|.  One warp per token: a lane sums K/32 values serially and five
      shuffle levels combine the lanes, so the fp32 mean is off by at most (K/32 + 5) 2^-24 mean|x|, an error the normalisation
      divides by sigma; the two-pass variance and rsqrtf move x_hat by a relative (K/32 + 5) 2^-25 + 2^-22, and the affine
      multiply-adds by a few 2^-24 of |x_hat gamma| + |beta|.  At K = 3072 the factor is 2^-17.
  GroupNorm    |got - ref| <= u |ref| + (2k + 32) 2^-24 scale + 2^-24,   k = 8 ceil(V / (8 nb)), nb = min(ceil(V / 64), 512),
      scale = |gamma| (|x_hat| E[x^2] / (var + eps) + mean|x| / sigma) + |beta|.  A thread sums the k values of its voxels of a
      group in fp32 before fp64 takes over, so E[x] and E[x^2] are off by at most k 2^-24 of mean|x| and of E[x^2]; the
      variance E[x^2] - mean^2 then carries a relative error up to 3k 2^-24 E[x^2] / var -- the statistics term, which grows
      with mean^2 / var -- and rstd half of it.  k <= 160 at config 3's largest level: at unit scale the factor is 2^-16.4.
The fp32 factors stay at or below 2^-16 at unit scale, 32 times below u in fp16.  A dropped or misplaced mask, a transposed
relative-position index, zero padding tokens, a missing 1/sqrt(32), a wrong parity, edge or group map and an unbiased or pooled
variance all land far outside these bounds: tests/test_norm_attention_reference_cpu.py checks that on the references.

Launch identities checked bit for bit: GroupNorm twice gives the same result, a 4-level launch equals its levels launched one
at a time, an n = 2 launch equals each sample launched alone (statistics are reduced in a fixed order).
Run with -s to see the worst err / bound of every row."""
import dataclasses
import math
import zlib
from typing import Optional, Tuple

import pytest
import torch

from tests.emulate import (reference_groupnorm64, reference_layernorm64, reference_patch_embed, reference_patch_merge64,
                           reference_window_attention64)

pytestmark = pytest.mark.gpu

DTYPE = {"bf16": torch.bfloat16, "fp16": torch.float16}
HALF_ULP = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
GUARD = 64                                   # NaN elements before and after every output tensor (keeps its 16-byte alignment)
EPS = 1e-5


@dataclasses.dataclass(frozen=True)
class Attn:
    dims: Tuple[int, int, int]               # token grid (H, W, D)
    heads: int                               # C = 32 heads
    shift: int
    dtype: str = "fp16"
    n: int = 1
    ld_out: Optional[int] = None             # output row pitch, C if None; channels [C, ld_out) must stay NaN
    qkv_pad: int = 0                         # NaN columns past 3C in every qkv row
    qk_std: float = 1.0                      # std of q and k (2.5: scores span about +-30)


@dataclasses.dataclass(frozen=True)
class LayerNorm:
    c: int
    tokens: Tuple[int, ...]                  # leading shape of the token rows
    dtype: str = "fp16"
    mean: float = 0.3
    std: float = 2.0


@dataclasses.dataclass(frozen=True)
class Merge:
    c: int
    dims: Tuple[int, int, int]
    n: int = 1
    dtype: str = "fp16"


@dataclasses.dataclass(frozen=True)
class Embed:
    dims: Tuple[int, int, int]               # grid extent (X, Y, Z)
    n: int = 1
    dtype: str = "fp16"


@dataclasses.dataclass(frozen=True)
class GroupNorm:
    levels: Tuple[Tuple[int, ...], ...]      # (X, Y, Z) of each level
    n: int = 1
    dtype: str = "fp16"
    relu: bool = True
    mean: float = 0.7
    std: float = 3.0


CONFIG3 = ((50, 50, 32), (25, 25, 16), (13, 13, 8), (7, 7, 4))          # the Swin-S token grids / FCOS levels of 200 x 200 x 130

ROWS = {
    # ---- window attention on config 3's token grids, Swin-S widths
    "attn_s50_c96_shift0_ld128_bf16": Attn((50, 50, 32), 3, 0, dtype="bf16", ld_out=128),
    "attn_s50_c96_shift2_ld128": Attn((50, 50, 32), 3, 2, ld_out=128),
    "attn_s25_c192_shift2": Attn((25, 25, 16), 6, 2),
    "attn_s13_c384_shift2_n2": Attn((13, 13, 8), 12, 2, n=2),                 # padding on the two shifted axes H, W
    "attn_s7_c768_mixed_shift": Attn((7, 7, 4), 24, 2),                       # D one window deep: shifted on H, W only
    "attn_s7_c768_mixed_shift_bf16": Attn((7, 7, 4), 24, 2, dtype="bf16"),
    "attn_5x8x8_c768_bf16": Attn((5, 8, 8), 24, 2, dtype="bf16", n=2),
    # ---- edges
    "attn_3x4x2_shift_dropped": Attn((3, 4, 2), 12, 2, n=2),                  # shift requested, dropped on every axis
    "attn_3x4x2_shift_dropped_bf16": Attn((3, 4, 2), 12, 2, dtype="bf16", n=2),
    "attn_9x3x4_only_h_shifted": Attn((9, 3, 4), 6, 2, n=2),
    "attn_9x9x9_odd_windows": Attn((9, 9, 9), 3, 2),                          # 27 windows: the second warpgroup sits out
    "attn_10x13x8_qkv_pad_bf16": Attn((10, 13, 8), 6, 2, dtype="bf16", n=2, qkv_pad=64),
    "attn_8x12x8_scores30": Attn((8, 12, 8), 3, 2, n=2, qk_std=2.5),          # masked pairs would dominate without the mask
    "attn_8x12x8_bf16": Attn((8, 12, 8), 3, 2, dtype="bf16", n=2),
    "attn_8x8x8_shift0_bf16": Attn((8, 8, 8), 3, 0, dtype="bf16", n=2),
    "attn_5x7x4_shift0_bf16": Attn((5, 7, 4), 6, 0, dtype="bf16", n=2),
    # ---- LayerNorm: ld = C rounded up to 64, input and output pad channels NaN
    "ln_c96_bf16": LayerNorm(96, (2, 5, 7, 3), dtype="bf16"),
    "ln_c96": LayerNorm(96, (2, 5, 7, 3)),
    "ln_c96_80k_tokens": LayerNorm(96, (1, 50, 50, 32)),
    "ln_c192_bf16": LayerNorm(192, (2, 5, 7, 3), dtype="bf16"),
    "ln_c384": LayerNorm(384, (1, 13, 13, 8)),
    "ln_c768_bf16": LayerNorm(768, (2, 5, 7, 3), dtype="bf16"),
    "ln_c768_mean50": LayerNorm(768, (1, 7, 7, 4), mean=50.0, std=0.5),
    "ln_c192_mean50_bf16": LayerNorm(192, (1, 9, 9, 5), dtype="bf16", mean=50.0, std=0.5),
    # ---- patch merging: ld_in = C + 64 with NaN pad channels; odd extents zero-filled
    "merge_c96_s50": Merge(96, (50, 50, 32)),
    "merge_c96_odd_all_bf16": Merge(96, (5, 7, 3), n=2, dtype="bf16"),
    "merge_c192_odd_h": Merge(192, (25, 24, 16), n=2),
    "merge_c192_odd_w": Merge(192, (12, 25, 16), n=2),
    "merge_c192_odd_all_bf16": Merge(192, (5, 7, 3), n=2, dtype="bf16"),
    "merge_c384_s13": Merge(384, (13, 13, 8)),                                # 8C = 3072, odd H and W
    "merge_c384_odd_d": Merge(384, (6, 8, 7), n=2),
    "merge_c384_odd_all_bf16": Merge(384, (13, 13, 7), n=2, dtype="bf16"),
    "merge_c768_odd_all_bf16": Merge(768, (5, 7, 3), n=2, dtype="bf16"),
    # ---- patch embedding: bit-exact
    "embed_21x18x14_n2": Embed((21, 18, 14), n=2),
    "embed_21x18x14_n2_bf16": Embed((21, 18, 14), n=2, dtype="bf16"),
    "embed_200x200x130": Embed((200, 200, 130)),
    "embed_200x200x130_bf16": Embed((200, 200, 130), dtype="bf16"),
    # ---- GroupNorm(32, 256) + ReLU
    "gn_config3": GroupNorm(CONFIG3),                                         # level 0: 80 000 voxels, CTAs clamped to 512
    "gn_config3_n2_bf16": GroupNorm(CONFIG3, n=2, dtype="bf16"),
    "gn_4_voxels": GroupNorm(((1, 2, 2),), n=2),                              # fewer voxels than the 8 rows of a CTA step
    "gn_unroll_minus1": GroupNorm(((49151, 1, 1), (1023, 1, 1))),             # 3 * 16384 - 1 (clamped), 2 * 512 - 1
    "gn_unroll_plus1_bf16": GroupNorm(((49153, 1, 1), (1025, 1, 1)), dtype="bf16"),
    "gn_mean_8sigma": GroupNorm(((9, 12, 10), (5, 6, 5)), n=2, mean=4.0, std=0.5),
    "gn_no_relu": GroupNorm(((9, 12, 10), (5, 6, 5), (2, 3, 3)), n=2, relu=False),
    "gn_small_bf16": GroupNorm(((9, 12, 10), (5, 6, 5), (2, 3, 3)), n=2, dtype="bf16"),
}


# ------------------------------------------------------------------------------------------------ bounds (shared with the CPU controls)
def attention_bound(ref, scale, dtype, vmax):
    u = HALF_ULP[dtype]
    sub = 2.0 ** -19 * vmax if dtype == torch.float16 else 0.0
    return u * ref.abs() + 2 * u * scale + sub + 2.0 ** -24


def norm_bound(ref, scale, dtype, terms):
    return HALF_ULP[dtype] * ref.abs() + terms * 2.0 ** -24 * scale + 2.0 ** -24


def layernorm_terms(k):
    return k / 32 + 32


def groupnorm_terms(voxels):
    nb = min(math.ceil(voxels / 64), 512)
    return 2 * 8 * math.ceil(voxels / (8 * nb)) + 32


# ------------------------------------------------------------------------------------------------ operands (CPU or GPU)
def _gen(row, device):
    return torch.Generator(device=device).manual_seed(zlib.crc32(repr(row).encode()) % 100000)


def attention_operands(row, device):
    """qkv (n, H, W, D, 3C + qkv_pad) with NaN past 3C, qkv_bias (3C) fp32, table (343, heads) fp32."""
    g, dt, C = _gen(row, device), DTYPE[row.dtype], row.heads * 32
    std = torch.tensor([row.qk_std] * (2 * C) + [1.0] * C, device=device)
    qkv = torch.full((row.n, *row.dims, 3 * C + row.qkv_pad), float("nan"), dtype=dt, device=device)
    qkv[..., :3 * C] = (torch.randn((row.n, *row.dims, 3 * C), device=device, generator=g) * std).to(dt)
    bias = torch.randn(3 * C, device=device, generator=g) * 0.3 * std
    table = torch.randn((343, row.heads), device=device, generator=g) * 0.5
    return qkv, bias, table


def attention_vmax(qkv, bias, C, dtype):
    return max(float(qkv[..., 2 * C:3 * C].float().abs().max()), float(bias[2 * C:].to(dtype).float().abs().max()))


def _ld64(c):
    return -(-c // 64) * 64


def layernorm_operands(row, device):
    """x (tokens..., ld) with NaN channels [C, ld), gamma, beta (C) fp32."""
    g, dt, ld = _gen(row, device), DTYPE[row.dtype], _ld64(row.c)
    x = torch.full((*row.tokens, ld), float("nan"), dtype=dt, device=device)
    x[..., :row.c] = (torch.randn((*row.tokens, row.c), device=device, generator=g) * row.std + row.mean).to(dt)
    return x, torch.rand(row.c, device=device, generator=g) + 0.5, torch.randn(row.c, device=device, generator=g)


def merge_operands(row, device):
    """x (n, H, W, D, C + 64) with NaN channels [C, C + 64), gamma, beta (8C) fp32."""
    g, dt = _gen(row, device), DTYPE[row.dtype]
    x = torch.full((row.n, *row.dims, row.c + 64), float("nan"), dtype=dt, device=device)
    x[..., :row.c] = (torch.randn((row.n, *row.dims, row.c), device=device, generator=g) * 2 + 0.3).to(dt)
    return x, torch.rand(8 * row.c, device=device, generator=g) + 0.5, torch.randn(8 * row.c, device=device, generator=g)


def groupnorm_operands(row, device):
    """levels [(n, X, Y, Z, 256)], gamma, beta (256) fp32."""
    g, dt = _gen(row, device), DTYPE[row.dtype]
    levels = [(torch.randn((row.n, *d, 256), device=device, generator=g) * row.std + row.mean).to(dt) for d in row.levels]
    return levels, torch.rand(256, device=device, generator=g) + 0.5, torch.randn(256, device=device, generator=g)


# ------------------------------------------------------------------------------------------------ checks
def _nan_buffer(shape, dtype):
    numel = math.prod(shape)
    buf = torch.full((numel + 2 * GUARD,), float("nan"), dtype=dtype, device="cuda")
    return buf, buf[GUARD: GUARD + numel].view(shape)


def _nan_bits(dtype):
    return torch.full((1,), float("nan"), dtype=dtype, device="cuda").view(torch.int16)


def _written(buf, shape, c, tag):
    """The first c channels of the (shape) tensor inside buf; asserts they are finite and that everything else in buf -- the
    channels [c, shape[-1]) and the guard bands -- is still the NaN it was."""
    numel = math.prod(shape)
    got = buf[GUARD: GUARD + numel].view(shape)[..., :c]
    assert torch.isfinite(got).all(), f"{tag}: {int((~torch.isfinite(got)).sum())} outputs unwritten or not finite"
    bits, nan = buf.view(torch.int16), _nan_bits(buf.dtype)
    assert bool((bits[GUARD: GUARD + numel].view(shape)[..., c:] == nan).all()), f"{tag}: pad channels written"
    assert bool((bits[:GUARD] == nan).all()) and bool((bits[GUARD + numel:] == nan).all()), f"{tag}: written outside the output"
    return got


def _within(got, ref, bound, tag, scale):
    err = (got.double() - ref).abs()
    ratio = err / bound
    at = int(ratio.argmax())
    worst = float(ratio.view(-1)[at])
    assert bool((err <= bound).all()), (
        f"{tag}: {int((err > bound).sum())} of {err.numel()} outputs out of bound; worst err/bound {worst:.3g} at "
        f"{tuple(int(v) for v in torch.unravel_index(torch.tensor(at), err.shape))}: got {float(got.reshape(-1)[at]):.8g} "
        f"ref {float(ref.reshape(-1)[at]):.8g} scale {float(scale.reshape(-1)[at]):.4g}")
    return worst


def _bits(t):
    return t.view(torch.int16)


def _run_attention(ops, row, tag):
    dt, C = DTYPE[row.dtype], row.heads * 32
    qkv, bias, table = attention_operands(row, "cuda")
    buf, out = _nan_buffer((row.n, *row.dims, row.ld_out or C), dt)
    ops.window_attention(qkv, out, bias, table, C, row.heads, row.shift)
    torch.cuda.synchronize()
    got = _written(buf, out.shape, C, tag)
    ref, scale = reference_window_attention64(qkv, bias, table, row.heads, row.shift, dt)
    return _within(got, ref, attention_bound(ref, scale, dt, attention_vmax(qkv, bias, C, dt)), tag, scale)


def _run_layernorm(ops, row, tag):
    dt = DTYPE[row.dtype]
    x, gamma, beta = layernorm_operands(row, "cuda")
    buf, out = _nan_buffer(x.shape, dt)
    ops.layernorm(x, out, row.c, gamma, beta, EPS)
    torch.cuda.synchronize()
    got = _written(buf, out.shape, row.c, tag)
    ref, scale = reference_layernorm64(x, row.c, gamma, beta, EPS)
    return _within(got, ref, norm_bound(ref, scale, dt, layernorm_terms(row.c)), tag, scale)


def _run_merge(ops, row, tag):
    dt = DTYPE[row.dtype]
    x, gamma, beta = merge_operands(row, "cuda")
    buf, out = _nan_buffer((row.n, *((e + 1) // 2 for e in row.dims), 8 * row.c), dt)
    ops.patch_merge_ln(x, out, row.c, gamma, beta, EPS)
    torch.cuda.synchronize()
    got = _written(buf, out.shape, 8 * row.c, tag)
    ref, scale = reference_patch_merge64(x, row.c, gamma, beta, EPS)
    return _within(got, ref, norm_bound(ref, scale, dt, layernorm_terms(8 * row.c)), tag, scale)


def _run_embed(ops, row, tag):
    dt = DTYPE[row.dtype]
    grid = (torch.rand((row.n, 4, *row.dims), device="cuda", generator=_gen(row, "cuda")) * 8 - 4).contiguous()
    buf, out = _nan_buffer((row.n, *(e // 4 for e in row.dims), 256), dt)
    ops.patch_embed_pack(grid, out)
    torch.cuda.synchronize()
    got = _written(buf, out.shape, 256, tag)
    want = reference_patch_embed(grid).to(dt)
    assert torch.equal(_bits(got), _bits(want)), f"{tag}: {int((_bits(got) != _bits(want)).sum())} elements differ"
    return 0.0


def _groupnorm(ops, row, levels, gamma, beta, tag):
    """Copies of `levels` in NaN-guarded buffers, normalised in one launch; returns the buffers."""
    bufs = []
    for x in levels:
        buf, view = _nan_buffer(x.shape, x.dtype)
        view.copy_(x)
        bufs.append((buf, view))
    ops.groupnorm_relu_([v for _, v in bufs], gamma, beta, EPS, row.relu)
    torch.cuda.synchronize()
    return [_written(buf, v.shape, 256, tag) for buf, v in bufs]


def _run_groupnorm(ops, row, tag):
    dt = DTYPE[row.dtype]
    levels, gamma, beta = groupnorm_operands(row, "cuda")
    got = _groupnorm(ops, row, levels, gamma, beta, tag)
    refs, scales = reference_groupnorm64(levels, gamma, beta, EPS, row.relu)
    worst = 0.0
    for l, (y, ref, scale) in enumerate(zip(got, refs, scales)):
        bound = norm_bound(ref, scale, dt, groupnorm_terms(math.prod(row.levels[l])))
        worst = max(worst, _within(y, ref, bound, f"{tag} level {l}", scale))
    # statistics are reduced in a fixed order: every launch of the same data gives the same bits
    again = _groupnorm(ops, row, levels, gamma, beta, tag)
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(got, again)), f"{tag}: a second call differs"
    if len(levels) > 1:
        for l, x in enumerate(levels):
            alone = _groupnorm(ops, row, [x], gamma, beta, tag)[0]
            assert torch.equal(_bits(alone), _bits(got[l])), f"{tag}: level {l} launched alone differs"
    if row.n > 1:
        for s in range(row.n):
            alone = _groupnorm(ops, row, [x[s:s + 1].clone() for x in levels], gamma, beta, tag)
            assert all(torch.equal(_bits(a), _bits(y[s:s + 1])) for a, y in zip(alone, got)), f"{tag}: sample {s} alone differs"
    return worst


RUN = {Attn: _run_attention, LayerNorm: _run_layernorm, Merge: _run_merge, Embed: _run_embed, GroupNorm: _run_groupnorm}


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available()
    from nerf_rpn_b200 import ops as _ops
    return _ops


@pytest.mark.parametrize("name", list(ROWS))
def test_kernel_row(ops, name):
    row = ROWS[name]
    worst = RUN[type(row)](ops, row, name)
    print(f"\n[swin/gn kernel] {name:34s} worst err/bound {worst:.3g}" + ("  (bit-exact)" if isinstance(row, Embed) else ""))


# ------------------------------------------------------------------------------------------------ refusals: nothing is launched
def test_window_attention_refusals(ops):
    heads, C = 3, 96
    qkv = torch.zeros((1, 4, 4, 4, 3 * C), device="cuda", dtype=torch.float16)
    bias, table = torch.zeros(3 * C, device="cuda"), torch.zeros((343, heads), device="cuda")
    out = torch.full((1, 4, 4, 4, C), float("nan"), device="cuda", dtype=torch.float16)
    for c, h, shift in ((C, heads + 1, 0), (C - 32, heads, 0), (C, heads, 1), (C, heads, 4)):
        with pytest.raises(RuntimeError, match="invalid argument"):
            ops.window_attention(qkv, out, bias, table, c, h, shift)
    torch.cuda.synchronize()
    assert torch.isnan(out).all()


def test_norm_refusals(ops):
    x = torch.zeros((2, 3, 4, 5, 64), device="cuda", dtype=torch.float16)
    out = torch.full((2, 3, 4, 5, 128), float("nan"), device="cuda", dtype=torch.float16)
    g, b = torch.ones(96 * 8, device="cuda"), torch.zeros(96 * 8, device="cuda")
    with pytest.raises(RuntimeError, match="invalid argument"):
        ops.layernorm(x, out, 96, g, b)                                      # ld_in 64 < c 96
    merged = torch.full((2, 2, 2, 3, 8 * 96), float("nan"), device="cuda", dtype=torch.float16)
    with pytest.raises(RuntimeError, match="invalid argument"):
        ops.patch_merge_ln(x, merged, 96, g, b)
    torch.cuda.synchronize()
    assert torch.isnan(out).all() and torch.isnan(merged).all()


def test_groupnorm_refusals(ops):
    from nerf_rpn_b200._lib import lib
    g, b = torch.ones(256, device="cuda"), torch.zeros(256, device="cuda")
    narrow = [torch.full((1, 4, 4, 4, 128), float("nan"), device="cuda", dtype=torch.float16)]
    with pytest.raises(RuntimeError, match="unsupported shape"):
        ops.groupnorm_relu_(narrow, g[:128], b[:128])
    levels = [torch.full((2, 4, 4, 4, 256), float("nan"), device="cuda", dtype=torch.float16) for _ in range(3)]
    need = lib().nrpn_groupnorm_workspace_bytes(3, 2)
    assert need > 0
    ws = torch.empty(need - 1, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError, match="workspace too small"):
        ops.groupnorm_relu_(levels, g, b, workspace=ws)
    torch.cuda.synchronize()
    assert torch.isnan(narrow[0]).all() and all(torch.isnan(t).all() for t in levels)
