"""Every kernel instance and plan nrpn_conv3d_wgrad can run, against the float64 reference (tests/emulate.py:reference_wgrad64).

One table: each row names the variant nrpn_conv3d_wgrad_variant must report for it -- instance <NT,NACC>, Cout slices per work item
(m), taps per work item (t) -- so that a change of wgrad_plan cannot move a row to another path unnoticed.  Rows marked `split` must
run with two or more K-splits, the others with one.  Every row checks the same things:
  - nothing unwritten, nothing over-written: dW is NaN-filled with GUARD NaN elements on each side, the workspace is NaN-filled (a
    partial tile that is never stored reaches dW as a NaN), and the row-pitch padding of dY (columns cout..ld_dy) and X (cin..ld_x)
    is NaN.  Afterwards every element of dW is finite and every guard element is still the NaN it was, bit for bit;
  - a per-element bound  |got - ref| <= 2^-24 |ref| + GAMMA mag,  mag = the same sum over |dY| |X|.
    GAMMA = 2^-17.  Each dW element is a chain of fp32 additions: the products of the voxels of one K-split (accumulated by wgmma,
    16 voxels per instruction), then the `splits` partial tiles added in a fixed order -- at most V + splits terms, V = the real
    voxels over all levels and samples (zero-filled voxel slots add exact zeros).  The worst-case bound of such a chain, (V + s) 2^-24
    mag, is 2^-12 mag at the table's sizes and would hide a dropped brick.  Rounding errors of sums of random-sign terms grow like
    sqrt(V + s) 2^-24 mag instead (each partial sum is O(sqrt(k)) of its k terms, whether the additions round to nearest or
    truncate), so every row asserts V + s <= 2^12 and GAMMA = 2 sqrt(2^12) 2^-24 = 2^-17 leaves a factor 2 over that -- the
    forward table's constant (tests/test_gpu_conv_variants.py).  Measured on an H100 80GB HBM3 (132 SMs, 700 W power limit), the
    worst err / bound over the table is 0.085 (k1_128_cin96), so 2^-17 needs no widening.  tests/test_wgrad_reference_cpu.py
    shows that a dropped 64-voxel brick, a tap shifted by one voxel, two swapped input channels, a missing level or a dropped last
    tap group exceed this bound by 10^3 or more;
  - rows marked `exact` draw dY and X from k/8, |k| <= 8: every product is a multiple of 2^-6 with |product| <= 1, and with fewer
    than 2^18 voxels summed into one element every partial sum -- in any order, the split reduction included -- is a multiple of
    2^-6 below 2^18, exact in fp32.  Their dW must equal the float64 reference bit for bit;
  - the bit identities the code claims: two launches give the same bits (fixed-order reduction), and dw_layout 1 (nn.Conv3d's
    (Cout, Cin, taps) order) is exactly the permutation of dw_layout 0 ((taps, Cout, Cin)).
Levels are consecutive rows of one dY buffer and one X buffer, as the training step stores them.  Run with -s to see each row's
variant, its splits and its worst err / bound."""
import ctypes
import dataclasses
import math
import re
import zlib
from typing import Optional, Tuple

import pytest
import torch

from tests.emulate import reference_wgrad64

pytestmark = pytest.mark.gpu

DTYPE = {"bf16": torch.bfloat16, "fp16": torch.float16}
GUARD = 64                                   # NaN elements before and after dW
GAMMA = 2.0 ** -17                           # see the module docstring
CHAIN_MAX = 2 ** 12                          # longest accumulation chain (voxels + splits) GAMMA is derived for
EXACT_MAX = 2 ** 18                          # exact rows: voxels summed into one element stay below this
TWO_TAPS = ((0, 0, -1), (1, -1, 1))
CORNER_TAPS = tuple((a, b, c) for a in (-1, 1) for b in (-1, 1) for c in (-1, 1))


@dataclasses.dataclass(frozen=True)
class Row:
    variant: str                             # "wgrad<NT,NACC>/m<M>/t<T>": the query's name without the split count
    cout: int
    cin: int
    taps: object                             # 1 or 3 ('same' taps of a k^3 filter), "stem" (its 32 taps) or a tuple of offsets
    levels: Tuple[Tuple[int, int, int], ...]  # dY extent (X, Y, Z) of each level
    n: int = 2
    dtype: str = "bf16"
    x_ext: Optional[Tuple[int, int, int]] = None   # X extent of a one-level row when it differs from dY's
    ld_pad: int = 0                          # ld_dy = cout + ld_pad, ld_x = cin + ld_pad (NaN columns)
    split: bool = False                      # runs with >= 2 K-splits
    exact: bool = False                      # operands on the k/8 grid: dW bit-exact


ROWS = {
    # ---- <64,NACC>: Cin <= 64
    "stem_like": Row("wgrad<64,4>/m1/t4", 64, 64, "stem", ((5, 6, 4),), x_ext=(5, 6, 5), exact=True),   # taps -2..1, 8 full groups
    "c2_64_fp16": Row("wgrad<64,4>/m1/t4", 64, 64, 3, ((6, 10, 9),), dtype="fp16", split=True),       # last group of 3
    "k3_64_128": Row("wgrad<64,4>/m1/t4", 128, 64, 3, ((8, 8, 16),), split=True),
    "cin32_cout40": Row("wgrad<64,4>/m1/t4", 40, 32, 3, ((3, 5, 7),), ld_pad=8, split=True),         # Cin, Cout < 64: zero fill
    "m2_t2_fp16": Row("wgrad<64,4>/m2/t2", 256, 64, 3, ((5, 6, 7),), dtype="fp16", split=True),       # the only m2 x t2 path
    "k1_64_x1": Row("wgrad<64,1>/m1/t1", 64, 64, 1, ((9, 1, 1),)),                                    # box 1 x 1 x 64
    "k1_64_256": Row("wgrad<64,2>/m2/t1", 256, 64, 1, ((6, 10, 9),), split=True),                     # stage-1 c3 / downsample
    "two_taps_c8": Row("wgrad<64,2>/m1/t2", 8, 64, TWO_TAPS, ((7, 3, 5),), dtype="fp16", ld_pad=8),   # Cout 8
    # ---- <128,NACC>: 64 < Cin <= 128
    "k1_128_cin96": Row("wgrad<128,1>/m1/t1", 64, 96, 1, ((3, 7, 5),), dtype="fp16", ld_pad=8),     # n_t 96 inside NT 128
    "c2_128": Row("wgrad<128,2>/m1/t2", 128, 128, 3, ((7, 5, 9),), split=True, exact=True),          # last group of 1
    "odd_mtiles": Row("wgrad<128,2>/m2/t1", 384, 128, 1, ((4, 4, 4),), exact=True),                   # 2nd slice of the last item > Cout
    "cin96_cout200": Row("wgrad<128,2>/m2/t1", 200, 96, 3, ((4, 6, 5),), dtype="fp16", split=True),
    "two_levels": Row("wgrad<128,2>/m2/t1", 256, 128, 3, ((9, 12, 10), (5, 6, 5)), split=True),
    "ld_padded": Row("wgrad<128,2>/m2/t1", 256, 128, 1, ((5, 3, 7),), ld_pad=8),
    # ---- <192,1>: reachable through the ABI, not used by the training step
    "nt192_cin160": Row("wgrad<192,1>/m1/t1", 64, 160, 3, ((4, 5, 6),), split=True),
    "nt192_cin192": Row("wgrad<192,1>/m1/t1", 128, 192, CORNER_TAPS, ((5, 4, 3),), dtype="fp16"),
    # ---- <256,1>: Cin >= 256
    "k1_256_64": Row("wgrad<256,1>/m1/t1", 64, 256, 1, ((6, 10, 9),), n=1),
    "c2_512": Row("wgrad<256,1>/m1/t1", 512, 512, 3, ((6, 6, 6),)),                               # n_tiles 2, m_tiles 4
    "wide_k_cin2048": Row("wgrad<256,1>/m1/t1", 512, 2048, 1, ((6, 10, 9),), n=1, split=True),     # n_tiles 8
    "wide_k_cout2048": Row("wgrad<256,1>/m1/t1", 2048, 512, 1, ((6, 10, 9),), n=1, split=True),    # m_tiles 16
    "head_4_levels": Row("wgrad<256,1>/m1/t1", 256, 256, 3, ((6, 8, 7), (3, 4, 4), (2, 2, 2), (1, 2, 2)), split=True,
                         exact=True),
    "predictor_fp16": Row("wgrad<256,1>/m1/t1", 128, 256, 1, ((6, 7, 9), (3, 4, 5), (2, 2, 3), (1, 2, 2)), dtype="fp16",
                          split=True),
}


def row_taps(row):
    if row.taps == "stem":
        from nerf_rpn_b200 import packing
        return packing.pack_stem_weight(torch.zeros(64, 4, 7, 7, 7), dtype=torch.float32)[1]
    if isinstance(row.taps, int):
        k = row.taps
        return [(a - k // 2, b - k // 2, c - k // 2) for a in range(k) for b in range(k) for c in range(k)]
    return [tuple(t) for t in row.taps]


def x_extents(row):
    if row.x_ext is not None:
        assert len(row.levels) == 1
        return [row.x_ext]
    return list(row.levels)


def real_voxels(row):
    return sum(row.n * math.prod(d) for d in row.levels)


def operands(row, device):
    """(dys, xs): per level, (N, X, Y, Z, ld) 16-bit views of one dY buffer and one X buffer (levels in consecutive rows); the pad
    columns are NaN.  exact rows draw from k/8, |k| <= 8, the others from N(0, 1) rounded to the 16-bit format."""
    dt = DTYPE[row.dtype]
    g = torch.Generator(device=device).manual_seed(zlib.crc32(repr(row).encode()) % 100000)

    def draw(shape):
        if row.exact:
            return (torch.randint(-8, 9, shape, device=device, generator=g).float() / 8).to(dt)
        return torch.randn(shape, device=device, generator=g).to(dt)

    def buffers(dims_list, c, ld):
        rows = [row.n * math.prod(d) for d in dims_list]
        buf = torch.full((sum(rows), ld), float("nan"), dtype=dt, device=device)
        buf[:, :c] = draw((sum(rows), c))
        out, o = [], 0
        for d, r in zip(dims_list, rows):
            out.append(buf[o:o + r].view(row.n, *d, ld))
            o += r
        return out
    return buffers(row.levels, row.cout, row.cout + row.ld_pad), buffers(x_extents(row), row.cin, row.cin + row.ld_pad)


def reference(row, dys, xs, taps):
    return reference_wgrad64([d[..., :row.cout] for d in dys], [x[..., :row.cin] for x in xs], taps,
                             None if row.x_ext is None else x_extents(row))


def bound(ref, mag):
    return 2.0 ** -24 * ref.abs() + GAMMA * mag


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available()
    from nerf_rpn_b200 import ops as _ops
    return _ops


def _launch(ops, row, dys, xs, taps, layout):
    """One nrpn_conv3d_wgrad call into a NaN-guarded dW with a NaN-filled workspace; returns the whole dW buffer."""
    from nerf_rpn_b200._lib import check, lib
    d = ops.wgrad_desc(dys, xs, taps, row.cout, row.cin, 1 if row.dtype == "fp16" else 0)
    d.dw_layout = layout
    need = lib().nrpn_conv3d_wgrad_workspace_bytes(ctypes.byref(d))
    assert need > 0
    ws = torch.full((need // 4 + 1,), float("nan"), dtype=torch.float32, device="cuda")
    buf = torch.full((len(taps) * row.cout * row.cin + 2 * GUARD,), float("nan"), dtype=torch.float32, device="cuda")
    d.dw, d.workspace, d.workspace_bytes = buf[GUARD:].data_ptr(), ws.data_ptr(), need
    check(lib().nrpn_conv3d_wgrad(ctypes.byref(d), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "conv3d_wgrad")
    torch.cuda.synchronize()
    return buf


def _check(row, buf, ref, mag, tag):
    """Every element of dW finite, the guards untouched, the per-element bound (bit-exact on exact rows).  Returns the worst
    err / bound."""
    numel = ref.numel()
    dw = buf[GUARD:GUARD + numel]
    assert torch.isfinite(dw).all(), f"{tag}: {int((~torch.isfinite(dw)).sum())} of {numel} elements unwritten or NaN"
    bits, nan = buf.view(torch.int32), torch.full((1,), float("nan"), device=buf.device).view(torch.int32)
    assert bool((bits[:GUARD] == nan).all()) and bool((bits[GUARD + numel:] == nan).all()), f"{tag}: written outside dW"
    got = dw.view(ref.shape).double()
    err = (got - ref).abs()
    if row.exact:
        assert torch.equal(ref.float().double(), ref), f"{tag}: the reference is not exact in fp32"
        assert torch.equal(got, ref), f"{tag}: {int((err > 0).sum())} elements differ, max |err| {float(err.max()):.3g}"
    b = bound(ref, mag)
    ratio = err / b
    at = int(ratio.argmax())
    assert bool((err <= b).all()), (
        f"{tag}: {int((err > b).sum())} of {numel} elements out of bound; worst err/bound {float(ratio.max()):.3g} at (tap, co, ci) "
        f"{tuple(int(v) for v in torch.unravel_index(torch.tensor(at), ref.shape))}: got {float(got.reshape(-1)[at]):.8g} "
        f"ref {float(ref.reshape(-1)[at]):.8g} mag {float(mag.reshape(-1)[at]):.4g}")
    return float(ratio.reshape(-1)[at])


@pytest.mark.parametrize("name", list(ROWS))
def test_wgrad_variant_row(ops, name):
    row = ROWS[name]
    taps = row_taps(row)
    dys, xs = operands(row, "cuda")
    variant = ops.conv3d_wgrad_variant(dys, xs, taps, row.cout, row.cin, 1 if row.dtype == "fp16" else 0)
    m = re.fullmatch(r"(wgrad<\d+,\d+>/m\d+/t\d+)/s(\d+)", variant)
    assert m and m.group(1) == row.variant, f"{name}: the plan now picks {variant}"
    splits = int(m.group(2))
    assert splits >= 2 if row.split else splits == 1, f"{name}: {splits} K-splits"
    V = real_voxels(row)
    assert V + splits <= CHAIN_MAX, f"{name}: chains of {V + splits} terms are longer than GAMMA is derived for"
    if row.exact:
        assert V < EXACT_MAX
    tag = f"{name} [{variant}]"
    first = _launch(ops, row, dys, xs, taps, 0)
    ref, mag = reference(row, dys, xs, taps)
    worst = _check(row, first, ref, mag, tag)
    again = _launch(ops, row, dys, xs, taps, 0)
    assert torch.equal(first.view(torch.int32), again.view(torch.int32)), f"{tag}: two launches differ"
    t, n_el = len(taps), ref.numel()
    conv_order = _launch(ops, row, dys, xs, taps, 1)
    assert torch.equal(conv_order[GUARD:GUARD + n_el].view(torch.int32).view(row.cout, row.cin, t).permute(2, 0, 1),
                       first[GUARD:GUARD + n_el].view(torch.int32).view(t, row.cout, row.cin)), f"{tag}: layout 1 differs from layout 0"
    _check(row, conv_order, ref.permute(1, 2, 0), mag.permute(1, 2, 0), tag + " layout 1")
    print(f"\n[wgrad variant] {name:18s} {variant:26s} splits {splits:2d}  {'exact' if row.exact else 'worst err/bound':15s} "
          f"{'' if row.exact else f'{worst:.3g}'}")


def test_table_covers_every_path():
    """Each instance <NT,NACC>, each (m_pair, t_group) pair wgrad_plan can produce, a partial last tap group, n_tiles > 1, odd
    m_tiles with m2, multiple splits, 4 levels, a different X extent and padded row pitches appear in a named row."""
    variants = {r.variant for r in ROWS.values()}
    instances = {v.split("/")[0] for v in variants}
    assert instances == {"wgrad<64,1>", "wgrad<64,2>", "wgrad<64,4>", "wgrad<128,1>", "wgrad<128,2>", "wgrad<192,1>", "wgrad<256,1>"}
    assert {v.split("/", 1)[1] for v in variants if v.startswith("wgrad<64,")} == {"m1/t1", "m1/t2", "m1/t4", "m2/t1", "m2/t2"}
    assert {v.split("/", 1)[1] for v in variants if v.startswith("wgrad<128,")} == {"m1/t1", "m1/t2", "m2/t1"}

    def ntaps(r):
        return len(CORNER_TAPS) if r.taps == CORNER_TAPS else (2 if r.taps == TWO_TAPS else (32 if r.taps == "stem" else r.taps ** 3))
    tg = {r: int(re.search(r"/t(\d)", r.variant).group(1)) for r in ROWS.values()}
    assert any(ntaps(r) % tg[r] for r in ROWS.values())
    assert any(r.cin > 256 for r in ROWS.values()) and any(-(-r.cout // 128) % 2 and "/m2" in r.variant and r.cout > 256 for r in ROWS.values())
    assert any(r.split for r in ROWS.values()) and any(len(r.levels) == 4 for r in ROWS.values())
    assert any(r.x_ext for r in ROWS.values()) and any(r.ld_pad for r in ROWS.values())
    assert {r.dtype for r in ROWS.values()} == {"bf16", "fp16"}
