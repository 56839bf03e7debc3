"""Every kernel instance nrpn_conv3d_fprop can launch, against the float64 reference (tests/emulate.py:reference_conv64).

One table: each row names the exact instance it expects, so that a change of the tile or epilogue rule cannot move a row to
another kernel unnoticed, and every launchable instance has a row (test_rows_cover_every_instance).  Every row checks the same
things:
  - nothing unwritten, nothing over-written: y is NaN-filled with ldy = cout + 8 and guard elements before and after it; the
    weight rows and shift entries cout..CoutPad are NaN (and so are residual columns cout..ldr).  Afterwards every column below
    cout is finite and every other element is still the NaN it was, bit for bit;
  - a per-element bound  |got - ref| <= r |ref| + 2^-17 mag + 2^-24,  r = half an ulp of the output format and mag the sum of
    the absolute values of every term: 2^-17 mag is far above the error of an fp32 accumulation of 16-bit products, and far
    below the effect of a dropped k-block, a wrong tap or a wrong shift / residual channel;
    Rows marked `exact` draw every operand from a coarse grid, so that every product and partial sum is exact in fp32 and the
    only error left is the epilogue's: their bound is  r |ref| + 2^-21 |pre-activation| + 2^-24, the fp32 GELU's error with
    room to spare, which a wrong GELU constant or any other epilogue slip exceeds;
  - the bit-identities the code claims: TMA versus register epilogue (NRPN_CONV_TMA_EPI=0 turns a `,tma-epilogue` instance
    into its register-epilogue twin and leaves every other row on its instance), narrow versus wide long-K tiles
    (NRPN_CONV_NARROW=0), and a 4-level launch versus its levels launched one at a time.
The TMA-store epilogue stages 128 x 64 sub-tiles in shared memory and stores them with cp.async.bulk.tensor, which clips partial
bricks and the channels past Cout; the `fallback` rows are cases it does not take (fp32 output, y not 16-byte aligned, a
nearest-upsampled residual).
Run with -s to see the worst err / bound of every row."""
import dataclasses
import math
import re
import zlib
from typing import Optional, Tuple

import pytest
import torch

from tests.emulate import reference_conv64

pytestmark = pytest.mark.gpu

HALF_ULP = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 2.0 ** -23}
INT_VIEW = {2: torch.int16, 4: torch.int32}
GUARD = 64                                   # NaN elements before and after every output tensor (keeps its 16-byte alignment)


@dataclasses.dataclass(frozen=True)
class Row:
    variant: str
    dims: Tuple[int, int, int]               # input extent (X, Y, Z)
    cin: int
    cout: int
    k: int = 3                               # 'same' taps of a k^3 filter (1 or 3)
    dtype: str = "bf16"                      # 16-bit format of x / w / res (and of y unless out_fp32)
    out_fp32: bool = False
    relu: int = 0                            # 0 none, 1 ReLU, 2 GELU
    res: Optional[object] = None             # None, "same" or the (Xr, Yr, Zr) of a nearest-upsampled residual
    n: int = 2
    stride: int = 1
    wsplit: bool = False                     # weights as hi + lo planes
    wrap: bool = False                       # more work items than resident CTAs: the stage / residual rings wrap
    levels: Optional[tuple] = None           # multi-level launch: the (X, Y, Z) of each level (dims unused)
    narrow: bool = False                     # long-K layer narrowed to 64-wide tiles: bit-identical to the wide tiles
    exact: bool = False                      # operands on a coarse grid: the fp32 accumulation is exact (see Case)
    # elements in front of y, moving its base address; not part of the seed, so a shifted row draws the same operands
    y_offset: int = dataclasses.field(default=0, repr=False)


LEVELS = ((16, 16, 32), (8, 8, 16), (5, 6, 7), (3, 2, 2))

ROWS = {
    # ---- short reductions (1^3), TMA epilogue: 16-bit output, cout % 64 == 0, same-extent or no residual
    "tma_bf16_relu_res_cpad": Row("igemm<64,2,2,tma-epilogue>", (9, 5, 7), 128, 192, k=1, relu=1, res="same"),   # CoutPad 256
    "tma_fp16_gelu_x1": Row("igemm<64,2,2,tma-epilogue>", (1, 12, 20), 64, 128, k=1, dtype="fp16", relu=2),
    "tma_bf16_res_wrap": Row("igemm<64,2,2,tma-epilogue>", (16, 24, 32), 64, 256, k=1, res="same", n=1, wrap=True),
    "tma_fp16_4_levels": Row("igemm<64,2,2,tma-epilogue>", None, 128, 64, k=1, dtype="fp16", relu=1, res="same", n=1,
                             levels=((8, 8, 16), (5, 6, 7), (1, 4, 30), (3, 2, 2))),
    # ---- short reductions, register epilogue: fp32 output, cout % 64 != 0, or an up-sampled residual
    "reg_bf16_f32_gelu_s2": Row("igemm<64,2,3>", (9, 7, 5), 256, 120, k=1, out_fp32=True, relu=2, stride=2),
    "reg_fp16_up_13_9": Row("igemm<64,2,3>", (13, 9, 4), 256, 256, k=1, dtype="fp16", res=(7, 5, 2)),
    "reg_bf16_relu_res_wrap": Row("igemm<64,2,3>", (16, 24, 40), 64, 120, k=1, relu=1, res="same", wrap=True),
    # ---- long reductions (3^3 taps)
    "long64_bf16_relu_wrap": Row("igemm<64,8,1,tma-epilogue>", (12, 16, 48), 128, 40, relu=1, wrap=True),
    "long64_narrow_fp16_gelu_k13824": Row("igemm<64,8,1,tma-epilogue>", (5, 8, 8), 512, 200, dtype="fp16", relu=2, n=1,
                                          narrow=True),
    "long64_narrow_bf16_res_c200": Row("igemm<64,8,1,tma-epilogue>", (5, 8, 8), 512, 200, relu=1, res="same", n=1, narrow=True),
    "long128_bf16_f32_res_wrap": Row("igemm<128,6,1>", (10, 16, 60), 64, 120, out_fp32=True, res="same", wrap=True),
    "long128_fp16_relu_res_c120_wrap": Row("igemm<128,6,1,tma-epilogue>", (10, 16, 60), 64, 120, dtype="fp16", relu=1,
                                           res="same", wrap=True),
    "long128_bf16_4_levels": Row("igemm<128,6,1,tma-epilogue>", None, 64, 128, relu=1, n=1, levels=LEVELS),
    "long256_fp16_relu_up_wrap": Row("igemm<256,4,1>", (12, 16, 96), 64, 200, dtype="fp16", relu=1, res=(7, 9, 55), n=1,
                                     wrap=True),
    # 128 x 256 tiles: Cout 200 leaves the last 64-channel sub-tile 8 channels wide; z = 95 leaves partial bricks
    "long256_bf16_relu_c200_wrap": Row("igemm<256,4,1,tma-epilogue>", (12, 16, 95), 64, 200, relu=1, n=1, wrap=True),
    "long256_fp16_gelu_4_levels": Row("igemm<256,4,1,tma-epilogue>", None, 64, 136, dtype="fp16", relu=2, n=1, levels=LEVELS),
    "long256_bf16_res_wrap": Row("igemm<256,4,1,tma-epilogue>", (12, 16, 96), 64, 256, res="same", n=1, wrap=True),
    # ---- long reductions the TMA store does not take: the register epilogue
    "fallback_long256_f32_out": Row("igemm<256,4,1>", (12, 16, 40), 64, 200, out_fp32=True, relu=1, n=1),
    "fallback_long256_y_not_16B_aligned": Row("igemm<256,4,1>", (12, 16, 40), 64, 200, relu=1, n=1, y_offset=2),
    "fallback_long128_upsampled_res": Row("igemm<128,6,1>", (12, 16, 48), 64, 128, dtype="fp16", relu=1, res=(6, 9, 21), n=1),
    # ---- weight split (hi + lo planes)
    "ws_tma_fp16_res_wrap": Row("igemm<64,2,2,tma-epilogue,wsplit>", (16, 24, 32), 64, 256, k=1, dtype="fp16", relu=1,
                                res="same", n=1, wsplit=True, wrap=True),             # the fp16_w2 bottleneck c3 convolution
    "ws_tma_fp16_4_levels": Row("igemm<64,2,2,tma-epilogue,wsplit>", None, 128, 64, k=1, dtype="fp16", relu=1, res="same", n=1,
                                wsplit=True, levels=((8, 8, 16), (5, 6, 7), (1, 4, 30), (3, 2, 2))),   # one-slot residual ring
    "ws_reg_fp16_gelu_up": Row("igemm<64,2,3,wsplit>", (13, 9, 2), 256, 120, k=1, dtype="fp16", relu=2, res=(7, 5, 1),
                               wsplit=True),
    "ws_long64_narrow_fp16": Row("igemm<64,6,1,tma-epilogue,wsplit>", (5, 8, 8), 256, 256, dtype="fp16", relu=1, n=1,
                                 wsplit=True, narrow=True),
    "ws_long64_fp16_c40_wrap": Row("igemm<64,6,1,tma-epilogue,wsplit>", (12, 16, 48), 128, 40, dtype="fp16", relu=1,
                                   wsplit=True, wrap=True),                          # Cout <= 64: 64-wide without narrowing
    "ws_long64_narrow_fp16_f32": Row("igemm<64,6,1,wsplit>", (5, 8, 8), 256, 256, dtype="fp16", out_fp32=True, relu=1, n=1,
                                     wsplit=True, narrow=True),
    "ws_long128_f32_wrap": Row("igemm<128,4,1,wsplit>", (16, 24, 48), 128, 128, dtype="fp16", out_fp32=True, n=1,
                               wsplit=True, wrap=True),
    "ws_long128_fp16_4_levels": Row("igemm<128,4,1,tma-epilogue,wsplit>", None, 64, 96, dtype="fp16", relu=2, n=1, wsplit=True,
                                    levels=LEVELS),
    "ws_long256_bf16_gelu_wrap": Row("igemm<256,2,1,tma-epilogue,wsplit>", (12, 16, 96), 64, 256, relu=2, n=1, wsplit=True,
                                     wrap=True),
    "ws_long256_fp16_relu_c248_wrap": Row("igemm<256,2,1,tma-epilogue,wsplit>", (12, 16, 95), 64, 248, dtype="fp16", relu=1,
                                          n=1, wsplit=True, wrap=True),
    "ws_long256_fp16_relu_up_wrap": Row("igemm<256,2,1,wsplit>", (12, 16, 96), 64, 256, dtype="fp16", relu=1, res=(7, 9, 55),
                                        n=1, wsplit=True, wrap=True),
    # ---- halo-slab kernel: 64 -> (<= 64) channels, stride 1, full box of taps, 16-bit output, no residual
    "slab_fp16_gelu_c24_wrap": Row("slab<4x16x8,N64>", (40, 33, 17), 64, 24, dtype="fp16", relu=2, wrap=True),
    "slab_bf16_relu_y1": Row("slab<4x16x8,N64>", (5, 1, 9), 64, 48, relu=1),
    # ---- exact accumulation: the fp32 epilogues checked to a few ulps
    "exact_reg_bf16_f32_gelu_up": Row("igemm<64,2,3>", (9, 7, 13), 128, 120, k=1, out_fp32=True, relu=2, res=(5, 4, 7),
                                      exact=True),
    "exact_long64_fp16_f32_gelu_res": Row("igemm<64,8,1>", (6, 9, 10), 128, 64, dtype="fp16", out_fp32=True, relu=2, res="same",
                                          exact=True),
}

# Every instance nrpn_conv3d_fprop can launch (conv3d_igemm.cu:kConvInstances and the halo-slab kernel), written out so that
# an instance without a row in ROWS fails test_rows_cover_every_instance.
LAUNCHABLE = {
    "slab<4x16x8,N64>",
    "igemm<64,2,3>", "igemm<64,2,2,tma-epilogue>",
    "igemm<64,8,1>", "igemm<64,8,1,tma-epilogue>",
    "igemm<128,6,1>", "igemm<128,6,1,tma-epilogue>",
    "igemm<256,4,1>", "igemm<256,4,1,tma-epilogue>",
    "igemm<64,2,3,wsplit>", "igemm<64,2,2,tma-epilogue,wsplit>",
    "igemm<64,6,1,wsplit>", "igemm<64,6,1,tma-epilogue,wsplit>",
    "igemm<128,4,1,wsplit>", "igemm<128,4,1,tma-epilogue,wsplit>",
    "igemm<256,2,1,wsplit>", "igemm<256,2,1,tma-epilogue,wsplit>",
}


def _dtype(row):
    return torch.float16 if row.dtype == "fp16" else torch.bfloat16


def _out_dims(dims, stride):
    return tuple((d - 1) // stride + 1 for d in dims)


def _nan_buffer(shape, dtype, device, offset=0):
    """NaN-filled tensor of `shape` inside a NaN-filled buffer with GUARD elements on each side; `offset` more elements in front
    move its base address.  Returns (buffer, view)."""
    numel = math.prod(shape)
    buf = torch.full((numel + 2 * GUARD + offset,), float("nan"), dtype=dtype, device=device)
    return buf, buf[GUARD + offset: GUARD + offset + numel].view(shape)


def _nan_bits(dtype, device):
    return torch.full((1,), float("nan"), dtype=dtype, device=device).view(INT_VIEW[torch.finfo(dtype).bits // 8])


class Case:
    """The operands of one row: NaN weight / shift padding, residuals with NaN columns cout..ldr, NaN-filled outputs."""

    def __init__(self, ops, row, device="cuda"):
        from nerf_rpn_b200 import packing
        self.ops, self.row = ops, row
        dt = _dtype(row)
        g = torch.Generator(device=device).manual_seed(zlib.crc32(repr(row).encode()) % 100000)
        k, cin, cout = row.k, row.cin, row.cout

        def draw(shape, scale):
            # exact rows: x, res in k/8 and w in k/64 (|k| <= 8), shift in k/512 (|k| <= 512) -- every product is a multiple of
            # 2^-9 and every partial sum stays far below 2^24 * 2^-9, so fp32 sums them exactly in any order
            if row.exact:
                return torch.randint(-8, 9, shape, device=device, generator=g).float() * (scale / 8)
            return torch.randn(shape, device=device, generator=g) * scale

        w = draw((cout, cin, k, k, k), 1 / 8 if row.exact else 1 / math.sqrt(cin * k ** 3))
        self.wp, self.taps = packing.pack_conv_weight(w, dtype=dt, split=row.wsplit)
        self.cpad = self.wp.shape[-2]
        self.wp.narrow(-2, cout, self.cpad - cout).fill_(float("nan"))
        shift = (torch.randint(-512, 513, (cout,), device=device, generator=g).float() / 512 if row.exact
                 else torch.randn((cout,), device=device, generator=g))
        self.shift = packing.pad_shift(shift, self.cpad)
        self.shift[cout:] = float("nan")
        self.ldy = cout + 8
        self.out_dtype = torch.float32 if row.out_fp32 else dt
        self.levels = []
        for dims in (row.levels or (row.dims,)):
            x = draw((row.n, *dims, cin), 1.0).to(dt)
            od = _out_dims(dims, row.stride)
            res, rdims = None, None
            if row.res is not None:
                rdims = od if row.res == "same" else tuple(row.res)
                res = draw((row.n, *rdims, cout + 8), 1.0).to(dt)                                    # ldr = cout + 8
                res[..., cout:] = float("nan")
            self.levels.append(dict(x=x, dims=dims, od=od, res=res, rdims=rdims))
        self.y_offset = row.y_offset

    def args(self, ys):
        row = self.row
        return [self.ops.ConvLevelArgs(L["x"], y, row.n, L["dims"], L["od"], self.ldy, res=L["res"], res_dims=L["rdims"],
                                       ldr=0 if L["res"] is None else L["res"].shape[-1]) for L, y in zip(self.levels, ys)]

    def call(self, fn, ys, **kw):
        row = self.row
        return fn(self.args(ys), self.wp, self.shift, row.cin, row.cout, self.taps, stride=row.stride, relu=row.relu,
                  out_fp32=row.out_fp32, **kw)

    def outputs(self):
        return [_nan_buffer((self.row.n, *L["od"], self.ldy), self.out_dtype, self.levels[0]["x"].device, self.y_offset)
                for L in self.levels]

    def variant(self, ys):
        return self.call(self.ops.conv3d_variant, ys)

    def run(self, levels=None):
        """Launch over all levels (or the given level indices); returns the NaN-guarded output buffers."""
        keep = range(len(self.levels)) if levels is None else levels
        outs = self.outputs()
        bufs, ys = [outs[i][0] for i in keep], [outs[i][1] for i in keep]
        saved = self.levels
        self.levels = [saved[i] for i in keep]
        try:
            self.call(self.ops.conv3d_fprop, ys)
        finally:
            self.levels = saved
        torch.cuda.synchronize()
        return bufs

    def check(self, bufs, tag):
        """Per-element bound on columns < cout; every other element of each buffer still the NaN it was.  Returns the worst
        err / bound."""
        row, cout = self.row, self.row.cout
        r = HALF_ULP[self.out_dtype]
        worst = 0.0
        for L, buf in zip(self.levels, bufs):
            shape = (row.n, *L["od"], self.ldy)
            numel = math.prod(shape)
            y = buf[GUARD + self.y_offset: GUARD + self.y_offset + numel].view(shape)
            got = y[..., :cout]
            assert torch.isfinite(got).all(), f"{tag}: {int((~torch.isfinite(got)).sum())} outputs unwritten or NaN"
            bits = buf.view(INT_VIEW[buf.element_size()])
            ncol = bits[GUARD + self.y_offset: GUARD + self.y_offset + numel].view(shape)[..., cout:]
            nan = _nan_bits(buf.dtype, buf.device)
            assert bool((ncol == nan).all()), f"{tag}: columns cout..ldy written"
            assert bool((bits[:GUARD + self.y_offset] == nan).all()) and bool((bits[GUARD + self.y_offset + numel:] == nan).all()), \
                f"{tag}: written outside the output tensor"
            res = None if L["res"] is None else L["res"][..., :cout]
            operands = (L["x"], self.wp.narrow(-2, 0, cout), self.taps, self.shift[:cout], L["od"])
            ref, mag = reference_conv64(*operands, stride=row.stride, act=row.relu, res=res)
            err = (got.double() - ref).abs()
            if row.exact:                        # the kernel accumulates the pre-activation exactly: only the epilogue rounds
                pre, _ = reference_conv64(*operands, stride=row.stride, act=0, res=res)
                bound = r * ref.abs() + 2.0 ** -21 * pre.abs() + 2.0 ** -24
            else:
                bound = r * ref.abs() + 2.0 ** -17 * mag + 2.0 ** -24
            ratio = err / bound
            at = int(ratio.argmax())
            worst = max(worst, float(ratio.view(-1)[at]))
            assert bool((err <= bound).all()), (
                f"{tag}: {int((err > bound).sum())} of {err.numel()} outputs out of bound; worst err/bound {float(ratio.max()):.3g} at "
                f"{tuple(int(v) for v in torch.unravel_index(torch.tensor(at), err.shape))}: got {float(got.reshape(-1)[at]):.8g} "
                f"ref {float(ref.reshape(-1)[at]):.8g} mag {float(mag.reshape(-1)[at]):.4g}")
        return worst


def _items_and_slots(case, variant):
    """Lower bound of the work items of the launch (every brick holds 128 voxels) and the CTAs the GPU keeps resident."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if variant.startswith("slab"):
        items = sum(case.row.n * math.ceil(L["od"][0] / 4) * math.ceil(L["od"][1] / 16) * math.ceil(L["od"][2] / 8)
                    for L in case.levels)
        return items, sms
    block_n, _, min_blocks = (int(v) for v in re.match(r"igemm<(\d+),(\d+),(\d+)", variant).groups())
    voxels = sum(case.row.n * math.prod(L["od"]) for L in case.levels)
    return math.ceil(voxels / 128) * (case.cpad // block_n), sms * min_blocks


def _same_bits(a, b):
    return all(torch.equal(x.view(INT_VIEW[x.element_size()]), y.view(INT_VIEW[y.element_size()])) for x, y in zip(a, b))


def _report(name, variant, worst, extra=""):
    print(f"\n[conv variant] {name:34s} {variant:36s} worst err/bound {worst:.3g}{extra}")


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available()
    from nerf_rpn_b200 import ops as _ops
    return _ops


def test_rows_cover_every_instance():
    assert {row.variant for row in ROWS.values()} == LAUNCHABLE


@pytest.mark.parametrize("name", list(ROWS))
def test_conv_variant_row(ops, monkeypatch, name):
    row = ROWS[name]
    case = Case(ops, row)
    probe = [y for _, y in case.outputs()]
    if row.y_offset:
        assert probe[0].data_ptr() % 16 != 0
    variant = case.variant(probe)
    assert variant == row.variant, f"{name}: the tile rule now picks {variant}"
    items, slots = _items_and_slots(case, variant)
    if row.wrap:
        assert items > slots, f"{name}: {items} work items do not wrap {slots} resident CTAs"
    bufs = case.run()
    worst = case.check(bufs, f"{name} [{variant}]")
    _report(name, variant, worst, f"  ({items}+ work items, {slots} resident CTAs)" if row.wrap else "")

    # the register epilogue performs the same fp32 operations in the same order as the TMA store; a row that does not take the
    # TMA store keeps its instance
    monkeypatch.setenv("NRPN_CONV_TMA_EPI", "0")
    reg = variant.replace(",2,2,tma-epilogue", ",2,3").replace(",tma-epilogue", "")
    assert case.variant(probe) == reg
    assert _same_bits(bufs, case.run()), f"{name}: {reg} differs from {variant}"
    monkeypatch.delenv("NRPN_CONV_TMA_EPI")
    if row.narrow:                               # 64-wide tiles keep the reduction order of every output element
        monkeypatch.setenv("NRPN_CONV_NARROW", "0")
        wide = case.variant(probe)
        assert wide != variant and "igemm<64," not in wide, wide
        assert _same_bits(bufs, case.run()), f"{name}: {wide} differs from {variant}"
        monkeypatch.delenv("NRPN_CONV_NARROW")
    if row.levels:                               # one launch over 4 levels == the 4 levels launched one at a time
        for i in range(len(row.levels)):
            assert _same_bits(case.run(levels=[i]), [bufs[i]]), f"{name}: level {i} launched alone differs"


def test_conv_rejects_misaligned_pointers(ops):
    """y must be aligned to one output pair (4 bytes for 16-bit output), shift to 8 bytes: otherwise the launch is refused before
    it starts and the variant query says so."""
    row = Row("igemm<64,2,2,tma-epilogue>", (4, 5, 6), 64, 64, k=1)
    case = Case(ops, dataclasses.replace(row, y_offset=1))                 # a 16-bit y at a 2-byte offset
    _, y = case.outputs()[0]
    assert y.data_ptr() % 4 == 2
    assert case.variant([y]) == "invalid"
    with pytest.raises(RuntimeError, match="invalid argument"):
        case.call(ops.conv3d_fprop, [y])
    aligned = Case(ops, row)
    _, y = aligned.outputs()[0]
    shift = torch.full((aligned.cpad + 2,), float("nan"), device="cuda")
    shift[1:aligned.cpad + 1] = aligned.shift
    aligned.shift = shift[1:aligned.cpad + 1]                               # fp32 shift at a 4-byte offset
    with pytest.raises(RuntimeError, match="invalid argument"):
        aligned.call(ops.conv3d_fprop, [y])
    torch.cuda.synchronize()
    assert torch.isnan(y).all()


def test_conv_fp32_output_needs_only_pair_alignment(ops):
    """An fp32 y that is 8- but not 16-byte aligned (one output pair) is accepted, matches the reference and equals the launch
    on an aligned y bit for bit."""
    row = Row("igemm<64,8,1>", (5, 8, 8), 512, 256, out_fp32=True, relu=1, res="same", n=1)
    aligned = Case(ops, row)
    shifted = Case(ops, dataclasses.replace(row, y_offset=2))                # fp32 y at an 8-byte offset
    _, y = shifted.outputs()[0]
    assert y.data_ptr() % 16 == 8
    assert shifted.variant([y]) == row.variant
    got = shifted.run()
    worst = shifted.check(got, "fp32 y at an 8-byte offset")
    ref = aligned.run()
    n = math.prod((row.n, *_out_dims(row.dims, 1), aligned.ldy))
    assert torch.equal(got[0][GUARD + 2: GUARD + 2 + n].view(torch.int32), ref[0][GUARD: GUARD + n].view(torch.int32))
    _report("pair_aligned_f32", row.variant, worst)
