"""The training plan's gradient helpers (nerf_rpn_b200/train.py: _TConv.repack, _TrainPlan._wgrad_stem / _param_grad / _dgrad) on
every convolution shape of ResNet50-FPN + the anchor RPN head, against float64 torch.autograd of the same nn.Conv3d.

Each test goes through the code the training step runs -- the operands packed on the device by nrpn_pack_weights / nrpn_gather_pack,
the weight gradient written in nn.Conv3d's own layout, the bias gradient, the data gradient with its 16-bit residual -- on small
extents.  Outputs land in NaN-guarded buffers: every element must be written and nothing around it.  Bounds:
  - dW and db (fp32):  |got - ref| <= 2^-24 |ref| + GAMMA mag,  mag = the same sum over absolute values, GAMMA = 2^-17 as derived
    in tests/test_gpu_wgrad_variants.py; the stem's dW on the k/8 grid must equal the reference bit for bit;
  - dX (16-bit):  |got - ref| <= r |ref| + 2^-17 mag + 2^-24, r = half an ulp of the format, as for the forward kernels
    (tests/test_gpu_conv_variants.py); a stride-2 layer's dX is rounded twice (the strided data gradient plus the residual, then
    that plus the lateral part), so its bound adds r |first sum|.
Run with -s to see the worst err / bound of each layer."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_wgrad_variants import GAMMA

pytestmark = pytest.mark.gpu

HALF_ULP = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
INT_VIEW = {2: torch.int16, 4: torch.int32}
GUARD = 64

# (cout, cin, k, stride) of every distinct convolution of ResNet50-FPN (Bottleneck stages of 3, 4, 6, 3 blocks; the stride-2 1^3
# conv1 / downsample of stages 2-4), its laterals and smoothing, the RPN head's 3^3 conv and its fused 1^3 cls | bbox predictor
LAYERS = [
    (64, 64, 1, 1), (64, 64, 3, 1), (256, 64, 1, 1), (64, 256, 1, 1),
    (128, 256, 1, 2), (128, 128, 3, 1), (512, 128, 1, 1), (512, 256, 1, 2), (128, 512, 1, 1),
    (256, 512, 1, 2), (256, 256, 3, 1), (1024, 256, 1, 1), (1024, 512, 1, 2), (256, 1024, 1, 1),
    (512, 1024, 1, 2), (512, 512, 3, 1), (2048, 512, 1, 1), (2048, 1024, 1, 2), (512, 2048, 1, 1),
    (256, 2048, 1, 1), (256, 512, 1, 1), (256, 256, 1, 1),                     # laterals (256 <- 1024 is stage 3's conv1 above)
    (128, 256, 1, 1),                                                          # the fused predictor
]
MULTI_LEVEL = {(256, 256, 3, 1), (128, 256, 1, 1)}                            # the head's layers also run over P2..P5 in one launch
HEAD_LEVELS = ((4, 5, 3), (2, 3, 2), (1, 2, 1), (1, 1, 1))
DIMS_S1 = (3, 5, 4)
DIMS_S2 = (5, 7, 3)                                                            # odd: the stride-2 output is ceil(X / 2)


class _Engine:
    """What _TConv and _TrainPlan read from the engine: the 16-bit format, the device and the stem layer."""

    def __init__(self, dtype):
        self.act_dtype, self.device, self.stem = dtype, torch.device("cuda"), None

    def _drop_graphs(self):
        pass


def _plan(eng, n, packed=None):
    from nerf_rpn_b200 import train as T
    plan = T._TrainPlan.__new__(T._TrainPlan)
    plan.eng, plan._scratch, plan.n, plan.packed = eng, {}, n, packed
    plan.f16 = 1 if eng.act_dtype == torch.float16 else 0
    return plan


def _nan_guarded(numel, dtype):
    buf = torch.full((numel + 2 * GUARD,), float("nan"), dtype=dtype, device="cuda")
    return buf, buf[GUARD:GUARD + numel]


def _written(buf, tag):
    """Every element of the guarded tensor finite, every guard element still the NaN it was."""
    got = buf[GUARD:buf.numel() - GUARD]
    assert torch.isfinite(got).all(), f"{tag}: {int((~torch.isfinite(got)).sum())} of {got.numel()} elements unwritten or NaN"
    bits = buf.view(INT_VIEW[buf.element_size()])
    nan = torch.full((1,), float("nan"), dtype=buf.dtype, device=buf.device).view(bits.dtype)
    assert bool((bits[:GUARD] == nan).all()) and bool((bits[-GUARD:] == nan).all()), f"{tag}: written outside the tensor"
    return got


def _within(got, ref, bound, tag):
    err = (got.double() - ref).abs()
    ratio = err / bound
    at = int(ratio.argmax())
    assert bool((err <= bound).all()), (
        f"{tag}: {int((err > bound).sum())} of {err.numel()} out of bound; worst err/bound {float(ratio.max()):.3g}: "
        f"got {float(got.reshape(-1)[at]):.8g} ref {float(ref.reshape(-1)[at]):.8g}")
    return float(ratio.reshape(-1)[at])


def _draw(shape, dtype, g, exact=False):
    if exact:
        return (torch.randint(-8, 9, shape, device="cuda", generator=g).float() / 8).to(dtype)
    return torch.randn(shape, device="cuda", generator=g).to(dtype)


def _ncdhw(t):
    return t.double().permute(0, 4, 1, 2, 3)


# ------------------------------------------------------------------------------------------------ stem
@pytest.mark.parametrize("dims,dtype,exact", [((9, 8, 11), torch.bfloat16, False), ((7, 10, 5), torch.float16, False),
                                              ((8, 5, 6), torch.bfloat16, True), ((5, 7, 9), torch.float16, True)])
def test_stem_weight_gradient_and_repack(dims, dtype, exact):
    """_TrainPlan._wgrad_stem (wgrad of the 4 x 4 x 2-tap stride-1 conv on the packed space-to-depth input, then nrpn_gather_pack
    into nn.Conv3d(4, 64, 7, stride 2, padding 3).weight's layout) against float64 autograd of that convolution on the grid rounded
    as nrpn_pack_stem_input rounds it; and _TConv.repack of the stem (nrpn_gather_pack, 16-bit) against packing.pack_stem_weight."""
    from nerf_rpn_b200 import ops, packing
    from nerf_rpn_b200.train import _TConv
    g = torch.Generator(device="cuda").manual_seed(sum(dims) * 3 + int(exact))
    n = 2
    eng = _Engine(dtype)
    weight = torch.randn((64, 4, 7, 7, 7), device="cuda", generator=g) * 0.05
    dw_buf, dw = _nan_guarded(weight.numel(), torch.float32)
    st = _TConv(eng, weight, None, stride=2, need_dgrad=False, stem=True, dw=dw)
    eng.stem = st

    st.fwd.fill_(float("nan"))
    st.repack()
    want, _ = packing.pack_stem_weight(weight, dtype=dtype)
    assert torch.equal(st.fwd.view(torch.int16), want.view(torch.int16)), "stem repack differs from packing.pack_stem_weight"
    assert int((want == 0).sum()) > 0                               # the structural zeros are written, not left as they were

    if exact:
        grid = torch.randint(-8, 9, (n, 4, *dims), device="cuda", generator=g).float() / 8
    else:
        grid = torch.rand((n, 4, *dims), device="cuda", generator=g) * 4 - 1
    packed = ops.pack_stem_input(grid, dtype=dtype)
    od = tuple((d + 1) // 2 for d in dims)
    assert tuple(packed.shape) == (n, od[0], od[1], od[2] + 1, 64)
    dy = _draw((n, *od, 64), dtype, g, exact)
    _plan(eng, n, packed)._wgrad_stem(dy)
    torch.cuda.synchronize()
    got = _written(dw_buf, "stem dW").view(weight.shape)

    def autograd(grid16, dy64):
        w = torch.zeros(weight.shape, dtype=torch.float64, device="cuda", requires_grad=True)
        F.conv3d(grid16, w, stride=2, padding=3).backward(dy64)
        return w.grad
    grid16 = grid.to(dtype).double()
    ref = autograd(grid16, _ncdhw(dy))
    mag = autograd(grid16.abs(), _ncdhw(dy).abs())
    if exact:
        assert torch.equal(ref.float().double(), ref)
        assert torch.equal(got.double(), ref), f"stem dW differs from the exact reference in {int((got.double() != ref).sum())} elements"
        print(f"\n[stem] {str(dims):12s} {str(dtype):15s} exact")
        return
    worst = _within(got, ref, 2.0 ** -24 * ref.abs() + GAMMA * mag, "stem dW")
    print(f"\n[stem] {str(dims):12s} {str(dtype):15s} worst err/bound {worst:.3g}")


# ------------------------------------------------------------------------------------------------ every other layer shape
def _reference(x, w16, dy, stride, k):
    """float64 autograd of F.conv3d(x, w16, stride, padding k // 2) given dY: (dW, dX) and their magnitudes (the same on |x|, |w|,
    |dY|).  x, dy channels-last 16-bit."""
    def run(x64, w64, g64):
        x64, w64 = x64.clone().requires_grad_(True), w64.clone().requires_grad_(True)
        F.conv3d(x64, w64, stride=stride, padding=k // 2).backward(g64)
        return w64.grad, x64.grad.permute(0, 2, 3, 4, 1)
    x64, w64, g64 = _ncdhw(x), w16.double(), _ncdhw(dy)
    dw, dx = run(x64, w64, g64)
    mag_w, mag_x = run(x64.abs(), w64.abs(), g64.abs())
    return dw, dx, mag_w, mag_x


def _levels_of_one_buffer(level_dims, n, c, dtype, g):
    rows = [n * math.prod(d) for d in level_dims]
    buf = _draw((sum(rows), c), dtype, g)
    out, o = [], 0
    for d, r in zip(level_dims, rows):
        out.append(buf[o:o + r].view(n, *d, c))
        o += r
    return out


@pytest.mark.parametrize("cout,cin,k,stride", LAYERS)
def test_layer_parameter_and_data_gradients(cout, cin, k, stride):
    from nerf_rpn_b200._lib import check, lib
    from nerf_rpn_b200.train import _TConv, _stream, _p
    i = LAYERS.index((cout, cin, k, stride))
    dtype = torch.float16 if i % 2 else torch.bfloat16
    tag = f"{cout}<-{cin} k{k} s{stride} {str(dtype)[6:]}"
    g = torch.Generator(device="cuda").manual_seed(1000 + i)
    torch.manual_seed(1000 + i)
    conv = torch.nn.Conv3d(cin, cout, k, stride=stride, padding=k // 2, bias=True).cuda()
    with torch.no_grad():
        conv.bias.normal_(0, 0.5)
    n, eng = 2, _Engine(dtype)
    dw_buf, dw = _nan_guarded(conv.weight.numel(), torch.float32)
    db_buf, db = _nan_guarded(cout, torch.float32)
    layer = _TConv(eng, conv.weight, conv.bias, stride=stride, dw=dw, db=db)
    layer.repack()
    plan = _plan(eng, n)
    assert layer.bwd_cols == cout                              # dY rows are read as the data gradient's input channels
    w16 = conv.weight.detach().to(dtype)

    if stride == 1:
        level_dims = HEAD_LEVELS if (cout, cin, k, stride) in MULTI_LEVEL else (DIMS_S1,)
        dys = _levels_of_one_buffer(level_dims, n, cout, dtype, g)
        xs = _levels_of_one_buffer(level_dims, n, cin, dtype, g)
        res = None if len(level_dims) > 1 else _draw((n, *DIMS_S1, cin), dtype, g)
        dx_bufs = [_nan_guarded(n * math.prod(d) * cin, dtype) for d in level_dims]
        dxs = [v.view(n, *d, cin) for (_, v), d in zip(dx_bufs, level_dims)]
        plan._param_grad(layer, dys, xs)
        plan._dgrad(layer, dys, dxs, list(level_dims), res=res)
    else:
        # the stride-2 sequence of _make_block_bwd: gather the even voxels, wgrad on them; dgrad (+ residual) on the output grid,
        # zero-stuff it back to the input grid and add it to the lateral part already in dX
        xd = DIMS_S2
        od = tuple((d + 1) // 2 for d in xd)
        level_dims = (xd,)
        x = _draw((n, *xd, cin), dtype, g)
        xs_even = torch.full((n, *od, cin), float("nan"), dtype=dtype, device="cuda")
        check(lib().nrpn_stride2(_p(x), _p(xs_even), n, *xd, cin, 0, _stream()), "stride2 gather")
        dys = [_draw((n, *od, cout), dtype, g)]
        xs = [x]
        res = _draw((n, *od, cin), dtype, g)
        lateral = _draw((n, *xd, cin), dtype, g)
        plan._param_grad(layer, dys, [xs_even])
        t = torch.full((n, *od, cin), float("nan"), dtype=dtype, device="cuda")
        plan._dgrad(layer, dys, [t], [od], res=res)
        full = torch.full((n, *xd, cin), float("nan"), dtype=dtype, device="cuda")
        check(lib().nrpn_stride2(_p(t), _p(full), n, *xd, cin, 1, _stream()), "stride2 scatter")
        dx_bufs = [_nan_guarded(lateral.numel(), dtype)]
        dx_bufs[0][1].copy_(lateral.reshape(-1))
        check(lib().nrpn_add_inplace(_p(dx_bufs[0][1]), _p(full), lateral.numel(), plan.f16, _stream()), "add_inplace")
    torch.cuda.synchronize()

    ref_w = torch.zeros(conv.weight.shape, dtype=torch.float64, device="cuda")
    mag_w = torch.zeros_like(ref_w)
    ref_b, mag_b = torch.zeros(cout, dtype=torch.float64, device="cuda"), torch.zeros(cout, dtype=torch.float64, device="cuda")
    r = HALF_ULP[dtype]
    worst_x = 0.0
    for lv, (dy, x, (dxb, _)) in enumerate(zip(dys, xs, dx_bufs)):
        w_l, dx_l, mw_l, mx_l = _reference(x, w16, dy, stride, k)
        ref_w += w_l
        mag_w += mw_l
        ref_b += dy.double().sum((0, 1, 2, 3))
        mag_b += dy.double().abs().sum((0, 1, 2, 3))
        got_x = _written(dxb, f"{tag} dX level {lv}").view(dx_l.shape)
        if stride == 1:
            if res is not None:
                dx_l, mx_l = dx_l + res.double(), mx_l + res.double().abs()
            bound = r * dx_l.abs() + 2.0 ** -17 * mx_l + 2.0 ** -24
        else:
            first = dx_l.clone()                                # the strided data gradient + residual, before the lateral add
            first[:, ::2, ::2, ::2] += res.double()
            mx_l = mx_l.clone()
            mx_l[:, ::2, ::2, ::2] += res.double().abs()
            dx_l, mx_l = first + lateral.double(), mx_l + lateral.double().abs()
            bound = r * (dx_l.abs() + first.abs()) + 2.0 ** -17 * mx_l + 2.0 ** -24
        worst_x = max(worst_x, _within(got_x, dx_l, bound, f"{tag} dX level {lv}"))
    got_w = _written(dw_buf, f"{tag} dW").view(conv.weight.shape)
    worst_w = _within(got_w, ref_w, 2.0 ** -24 * ref_w.abs() + GAMMA * mag_w, f"{tag} dW")
    got_b = _written(db_buf, f"{tag} db")
    worst_b = _within(got_b, ref_b, 2.0 ** -24 * ref_b.abs() + GAMMA * mag_b, f"{tag} db")
    print(f"\n[layer grads] {tag:26s} levels {len(level_dims)}  worst err/bound  dW {worst_w:.3g}  db {worst_b:.3g}  dX {worst_x:.3g}")


def test_layer_list_is_the_models():
    """LAYERS holds exactly the distinct (cout, cin, k, stride) of ResNet_FPN_256 (layers 3, 4, 6, 3) and RPNHead, the fused
    predictor standing in for the cls / bbox pair it replaces."""
    from nerf_rpn_b200.model.anchor import RPNHead
    from nerf_rpn_b200.model.feature_extractor import Bottleneck, ResNet_FPN_256
    with torch.device("meta"):
        bb = ResNet_FPN_256(Bottleneck, [3, 4, 6, 3], input_dim=4, is_max_pool=True)
        head = RPNHead(256, 13, 4, rotate=True)
    shapes = {(m.out_channels, m.in_channels, m.kernel_size[0], m.stride[0]) for mod in (bb, head) for m in mod.modules()
              if isinstance(m, torch.nn.Conv3d) and m is not bb.conv1 and m not in (head.cls_logits, head.bbox_pred)}
    assert shapes | {(128, 256, 1, 1)} == set(LAYERS) and len(LAYERS) == len(set(LAYERS))
