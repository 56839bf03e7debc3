"""The shared-memory (TMA-store) epilogue of the long-reduction convolutions (conv3d_igemm.cu, TMA_EPI with one CTA per SM).

The tile is staged as 128 x 64 sub-tiles in two alternating shared-memory buffers and stored with cp.async.bulk.tensor, which
clips partial bricks and the channels past Cout.  Every row is checked like a row of tests/test_gpu_conv_variants.py (the float64
reference, nothing written outside columns < cout of the NaN-filled output with ldy = cout + 8) and must equal the register
epilogue (NRPN_CONV_TMA_EPI=0) bit for bit.  The `fallback` rows are the cases the TMA store does not take (fp32 output, y not
16-byte aligned, a nearest-upsampled residual): they must give the same bits whatever NRPN_CONV_TMA_EPI says."""
import pytest
import torch

from tests.test_gpu_conv_variants import INT_VIEW, Case, Row, _items_and_slots, _report

pytestmark = pytest.mark.gpu

LEVELS = ((16, 16, 32), (8, 8, 16), (5, 6, 7), (3, 2, 2))

ROWS = {
    # 128 x 256 tiles: Cout 200 leaves the last 64-channel sub-tile 8 channels wide; z = 95 leaves partial bricks
    "long256_bf16_relu_c200_wrap": (Row("igemm<256,4,1>", (12, 16, 95), 64, 200, relu=1, n=1, wrap=True), 0),
    "long256_fp16_gelu_4_levels": (Row("igemm<256,4,1>", None, 64, 136, dtype="fp16", relu=2, n=1, levels=LEVELS), 0),
    "long256_bf16_res_wrap": (Row("igemm<256,4,1>", (12, 16, 96), 64, 256, res="same", n=1, wrap=True), 0),
    # 128 x 128 tiles
    "long128_fp16_relu_res_c120_wrap": (Row("igemm<128,6,1>", (10, 16, 60), 64, 120, dtype="fp16", relu=1, res="same",
                                            wrap=True), 0),
    "long128_bf16_4_levels": (Row("igemm<128,6,1>", None, 64, 128, relu=1, n=1, levels=LEVELS), 0),
    # 128 x 64 tiles (a layer with few tiles, narrowed from 256 wide), and the split-weight variants
    "long64_narrow_bf16_res_c200": (Row("igemm<64,8,1>", (5, 8, 8), 512, 200, relu=1, res="same", n=1, narrow=True), 0),
    "ws_long256_fp16_relu_c248_wrap": (Row("igemm<256,2,1,wsplit>", (12, 16, 95), 64, 248, dtype="fp16", relu=1, n=1,
                                           wsplit=True, wrap=True), 0),
    "ws_long128_fp16_4_levels": (Row("igemm<128,4,1,wsplit>", None, 64, 96, dtype="fp16", relu=2, n=1, wsplit=True,
                                     levels=LEVELS), 0),
    # register-epilogue fallbacks
    "fallback_long256_f32_out": (Row("igemm<256,4,1>", (12, 16, 40), 64, 200, out_fp32=True, relu=1, n=1), 0),
    "fallback_long256_y_not_16B_aligned": (Row("igemm<256,4,1>", (12, 16, 40), 64, 200, relu=1, n=1), 2),
    "fallback_long128_upsampled_res": (Row("igemm<128,6,1>", (12, 16, 48), 64, 128, dtype="fp16", relu=1, res=(6, 9, 21),
                                           n=1), 0),
}


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available()
    from nerf_rpn_b200 import ops as _ops
    return _ops


def _same_bits(a, b):
    return all(torch.equal(x.view(INT_VIEW[x.element_size()]), y.view(INT_VIEW[y.element_size()])) for x, y in zip(a, b))


@pytest.mark.parametrize("name", list(ROWS))
def test_long_reduction_epilogue(ops, monkeypatch, name):
    row, y_offset = ROWS[name]
    case = Case(ops, row, y_offset=y_offset)
    probe = [y for _, y in case.outputs()]
    if y_offset:
        assert probe[0].data_ptr() % 16 != 0
    variant = case.variant(probe)
    assert variant == row.variant, f"{name}: the tile rule now picks {variant}"
    items, slots = _items_and_slots(case, variant)
    if row.wrap:
        assert items > slots, f"{name}: {items} work items do not wrap {slots} resident CTAs"
    bufs = case.run()
    worst = case.check(bufs, f"{name} [{variant}]")
    _report(name, variant, worst)

    monkeypatch.setenv("NRPN_CONV_TMA_EPI", "0")
    assert case.variant(probe) == variant
    assert _same_bits(bufs, case.run()), f"{name}: the register epilogue differs"
    monkeypatch.delenv("NRPN_CONV_TMA_EPI")
    if row.levels:                               # one launch over 4 levels == the 4 levels launched one at a time
        for i in range(len(row.levels)):
            assert _same_bits(case.run(levels=[i]), [bufs[i]]), f"{name}: level {i} launched alone differs"
