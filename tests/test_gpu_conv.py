"""GPU numerics tests for the wgmma implicit-GEMM convolution and the bandwidth kernels, through the C ABI.
Reference = plain PyTorch fp32 conv3d on the same bf16-rounded operands (tests/emulate.py).  Tolerance: the
kernel accumulates in fp32, so with fp32 output the error is accumulation-order only (2e-3 of the output scale
for K up to 13 824); with bf16 output one extra rounding (2^-8 relative)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.emulate import emulate_conv, emulate_pack_stem

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available()
    from nerf_rpn_b200 import ops as _ops
    return _ops


def _diagnose(got, ref, tag):
    err = (got - ref).abs()
    scale = ref.abs().max().item() + 1e-12
    msg = [f"[{tag}] max abs err {err.max().item():.4g} (scale {scale:.4g}), mean abs err {err.mean().item():.4g}"]
    bad = err > 0.02 * scale
    msg.append(f"  bad fraction {bad.float().mean().item():.4f}")
    if bad.any():
        idx = bad.nonzero()[:8].tolist()
        msg.append(f"  first bad idx {idx}")
        for d in range(got.dim()):
            other = [i for i in range(got.dim()) if i != d]
            per = bad.float().mean(dim=other)
            msg.append(f"  bad fraction along dim {d}: {[round(v, 3) for v in per.tolist()[:40]]}")
    return "\n".join(msg)


def run_conv(ops, x, w, bias=None, stride=1, relu=False, res=None, out_fp32=False, levels=None):
    from nerf_rpn_b200 import packing
    cout = w.shape[0]
    wp, taps = packing.pack_conv_weight(w)
    cpad = wp.shape[1]
    shift = packing.pad_shift(bias if bias is not None else torch.zeros(cout, device=w.device), cpad)
    wp = wp.cuda(); shift = shift.cuda()
    xs = [x] if levels is None else levels
    ress = [res] if levels is None else [None] * len(levels)
    args, outs = [], []
    ldy = ((cout + 7) // 8) * 8
    for xi, ri in zip(xs, ress):
        n, X, Y, Z, cin = xi.shape
        od = tuple((d - 1) // stride + 1 for d in (X, Y, Z))
        y = torch.full((n, *od, ldy), float("nan"), dtype=torch.float32 if out_fp32 else torch.bfloat16, device="cuda")
        outs.append(y)
        a = ops.ConvLevelArgs(xi, y, n, (X, Y, Z), od, ldy, res=ri, res_dims=None if ri is None else ri.shape[1:4],
                              ldr=0 if ri is None else ri.shape[-1])
        args.append(a)
    ops.conv3d_fprop(args, wp, shift, xs[0].shape[-1], ldy, taps, stride=stride, relu=relu, out_fp32=out_fp32)
    torch.cuda.synchronize()
    refs = []
    for xi, ri in zip(xs, ress):
        n, X, Y, Z, cin = xi.shape
        od = tuple((d - 1) // stride + 1 for d in (X, Y, Z))
        refs.append(emulate_conv(xi.float(), wp.float(), taps, shift, od, stride=stride, relu=relu, res=ri)[..., :ldy])
    return outs, refs


CASES = [
    # name, dims, cin, cout, k, stride, relu, res mode, out_fp32
    ("1x1_64_64", (8, 8, 16), 64, 64, 1, 1, False, None, True),
    ("3x3_64_64", (8, 8, 16), 64, 64, 3, 1, False, None, True),
    ("3x3_odd_relu", (10, 13, 9), 64, 64, 3, 1, True, None, False),
    ("3x3_256_256", (9, 12, 17), 256, 256, 3, 1, True, None, False),
    ("1x1_256_1024_res", (6, 9, 10), 256, 1024, 1, 1, True, "same", False),
    ("1x1_s2_512_128", (9, 12, 11), 512, 128, 1, 2, False, None, True),
    ("1x1_upsample_add", (13, 9, 7), 512, 256, 1, 1, False, "up", False),
    ("pred_1x1_256_120", (7, 8, 9), 256, 120, 1, 1, False, None, True),
]


@pytest.mark.parametrize("name,dims,cin,cout,k,stride,relu,resmode,out_fp32", CASES)
def test_conv_cases(ops, name, dims, cin, cout, k, stride, relu, resmode, out_fp32):
    g = torch.Generator(device="cuda").manual_seed(hash(name) % 1000)
    x = torch.randn((2, *dims, cin), device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn((cout, cin, k, k, k), device="cuda", generator=g) / (cin * k ** 3) ** 0.5
    bias = torch.randn((cout,), device="cuda", generator=g)
    res = None
    od = tuple((d - 1) // stride + 1 for d in dims)
    if resmode == "same":
        res = torch.randn((2, *od, cout), device="cuda", generator=g).to(torch.bfloat16)
    elif resmode == "up":
        rd = tuple((d + 1) // 2 for d in od)                      # odd sizes: 13 -> 7 etc. (size-based nearest)
        res = torch.randn((2, *rd, cout), device="cuda", generator=g).to(torch.bfloat16)
    outs, refs = run_conv(ops, x, w, bias, stride, relu, res, out_fp32)
    got, ref = outs[0].float(), refs[0]
    assert not torch.isnan(got).any(), _diagnose(torch.nan_to_num(got, nan=1e9), ref, name + " (NaN = never written)")
    tol = 2e-3 if out_fp32 else 1e-2
    scale = ref.abs().max().item()
    assert (got - ref).abs().max().item() <= tol * scale, _diagnose(got, ref, name)


def test_conv_multi_level_shared_weights(ops):
    """The RPN head shape: one launch over 4 pyramid levels sharing 3^3 256->256 weights (anchor.py:206-213)."""
    g = torch.Generator(device="cuda").manual_seed(9)
    levels = [torch.randn((1, *d, 256), device="cuda", generator=g).to(torch.bfloat16)
              for d in [(10, 16, 16), (5, 8, 8), (3, 4, 4), (2, 2, 2)]]
    w = torch.randn((256, 256, 3, 3, 3), device="cuda", generator=g) / (256 * 27) ** 0.5
    bias = torch.randn((256,), device="cuda", generator=g)
    outs, refs = run_conv(ops, None, w, bias, 1, True, None, False, levels=levels)
    for i, (o, r) in enumerate(zip(outs, refs)):
        got = o.float()
        assert not torch.isnan(got).any(), f"level {i}: unwritten outputs"
        assert (got - r).abs().max().item() <= 1e-2 * r.abs().max().item(), _diagnose(got, r, f"level{i}")


def test_conv_split_k_small_grids(ops, monkeypatch):
    """Late ResNet stages: few output tiles, long reductions -> split-K through the fp32 scratch (atomics + last-CTA
    fix-up). Run twice on the same zero-initialised scratch: every launch must leave it zero-filled."""
    import os
    if os.environ.get("NRPN_SPLITK") != "1":
        # split-K is opt-in and NRPN_SPLITK is read when the library initialises: run this test again in a second process that sets it
        import subprocess, sys
        root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
        r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-rs",
                            os.path.abspath(__file__) + "::test_conv_split_k_small_grids"],
                           cwd=root, capture_output=True, text=True, timeout=900, env={**os.environ, "NRPN_SPLITK": "1"})
        assert r.returncode == 0 and "1 passed" in r.stdout, (r.stdout + r.stderr)[-3000:]
        return
    from nerf_rpn_b200 import packing
    g = torch.Generator(device="cuda").manual_seed(21)
    ws = torch.zeros(64 << 20, dtype=torch.uint8, device="cuda")
    for dims, cin, cout, k, relu, with_res in [((5, 8, 8), 512, 512, 3, True, False), ((10, 16, 16), 1024, 256, 1, False, True),
                                                ((5, 8, 8), 2048, 512, 1, True, True), ((10, 16, 16), 256, 256, 3, False, False)]:
        x = torch.randn((1, *dims, cin), device="cuda", generator=g).to(torch.bfloat16)
        w = torch.randn((cout, cin, k, k, k), device="cuda", generator=g) / (cin * k ** 3) ** 0.5
        bias = torch.randn((cout,), device="cuda", generator=g)
        res = torch.randn((1, *dims, cout), device="cuda", generator=g).to(torch.bfloat16) if with_res else None
        wp, taps = packing.pack_conv_weight(w.cpu()); wp = wp.cuda()
        shift = packing.pad_shift(bias, wp.shape[1])
        ref = emulate_conv(x.float(), wp.float(), taps, shift, dims, relu=relu, res=res)[..., :cout]
        args_probe = [ops.ConvLevelArgs(x, x, 1, dims, dims, cout)]
        need = ops.conv3d_workspace_bytes(args_probe, wp, shift, cin, cout, taps)
        assert need > 0, "this shape is expected to be split along K"
        for rep in range(2):
            y = torch.full((1, *dims, cout), float("nan"), dtype=torch.bfloat16, device="cuda")
            a = ops.ConvLevelArgs(x, y, 1, dims, dims, cout, res=res, res_dims=dims if with_res else None, ldr=cout if with_res else 0)
            ops.conv3d_fprop([a], wp, shift, cin, cout, taps, relu=relu, workspace=ws)
            torch.cuda.synchronize()
            got = y.float()
            assert not torch.isnan(got).any()
            assert (got - ref).abs().max().item() <= 1e-2 * ref.abs().max().item(), _diagnose(got, ref, f"splitk {dims} {cin}->{cout} rep{rep}")
            if rep == 1:
                assert torch.equal(y, first), "split-K must be bit-reproducible"
            first = y
        assert int(ws[:16].count_nonzero().item()) == 0, "split-K arrival counters not restored to zero"


def test_conv_large_p2_tile_count(ops):
    """More tiles than SMs (persistent loop, stage ring wrap-around)."""
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.randn((1, 24, 32, 40, 128), device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn((256, 128, 3, 3, 3), device="cuda", generator=g) / (128 * 27) ** 0.5
    outs, refs = run_conv(ops, x, w, None, 1, False, None, True)
    got, ref = outs[0], refs[0]
    assert (got - ref).abs().max().item() <= 2e-3 * ref.abs().max().item(), _diagnose(got, ref, "p2like")


def test_stem_pack_and_conv(ops):
    from nerf_rpn_b200 import packing
    g = torch.Generator(device="cuda").manual_seed(12)
    for dims in [(24, 20, 28), (21, 19, 27)]:
        x = torch.rand((1, 4, *dims), device="cuda", generator=g)
        packed = ops.pack_stem_input(x)
        torch.testing.assert_close(packed.float(), emulate_pack_stem(x).to(torch.bfloat16).float(), rtol=0, atol=0)
        w = torch.randn((64, 4, 7, 7, 7), device="cuda", generator=g) * 0.05
        wp, taps = packing.pack_stem_weight(w)
        od = tuple((d + 1) // 2 for d in dims)
        y = torch.empty((1, *od, 64), dtype=torch.float32, device="cuda")
        shift = torch.zeros(64, device="cuda")
        a = ops.ConvLevelArgs(packed, y, 1, packed.shape[1:4], od, 64)
        ops.conv3d_fprop([a], wp.cuda(), shift, 64, 64, taps, out_fp32=True)
        ref = F.conv3d(x.to(torch.bfloat16).float(), w.to(torch.bfloat16).float(), stride=2, padding=3).permute(0, 2, 3, 4, 1)
        assert (y - ref).abs().max().item() <= 2e-3 * ref.abs().max().item(), _diagnose(y, ref, "stem")


def test_maxpool(ops):
    g = torch.Generator(device="cuda").manual_seed(13)
    for dims in [(12, 10, 14), (11, 9, 13)]:
        x = torch.randn((2, *dims, 64), device="cuda", generator=g).to(torch.bfloat16)
        got = ops.maxpool3d_k3s2(x)
        ref = F.max_pool3d(x.float().permute(0, 4, 1, 2, 3), kernel_size=3, stride=2, padding=1).permute(0, 2, 3, 4, 1)
        torch.testing.assert_close(got.float(), ref, rtol=0, atol=0)


def _stem_case(ops, dims, n, seed):
    from nerf_rpn_b200 import packing
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand((n, 4, *dims), device="cuda", generator=g)
    packed = ops.pack_stem_input(x)
    w = torch.randn((64, 4, 7, 7, 7), device="cuda", generator=g) * 0.05
    bias = torch.randn((64,), device="cuda", generator=g) * 0.1
    wp, taps = packing.pack_stem_weight(w)
    od = tuple((d + 1) // 2 for d in dims)
    ref = F.relu(F.conv3d(x.to(torch.bfloat16).float(), w.to(torch.bfloat16).float(), bias, stride=2, padding=3)).permute(0, 2, 3, 4, 1)
    return packed, wp.cuda(), taps, bias, od, ref


@pytest.mark.parametrize("dims,n", [((48, 64, 40), 1), ((42, 38, 54), 2), ((80, 96, 64), 2)])
def test_slab_kernel_stem(ops, monkeypatch, dims, n):
    """csrc/conv3d_slab.cu on the packed stem (4 x 4 x 2 taps, z offsets {-1, +1}): bf16 output routes to the halo-slab
    kernel; it must agree with fp32 PyTorch on the bf16-rounded operands and with the brick kernel (NRPN_CONV_SLAB=0)."""
    packed, wp, taps, bias, od, ref = _stem_case(ops, dims, n, 31)
    outs = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("NRPN_CONV_SLAB", mode)
        y = torch.full((n, *od, 64), float("nan"), dtype=torch.bfloat16, device="cuda")
        a = ops.ConvLevelArgs(packed, y, n, packed.shape[1:4], od, 64)
        ops.conv3d_fprop([a], wp, bias, 64, 64, taps, relu=True)
        torch.cuda.synchronize()
        got = y.float()
        assert not torch.isnan(got).any(), _diagnose(torch.nan_to_num(got, nan=1e9), ref, f"stem slab={mode}: unwritten outputs")
        assert (got - ref).abs().max().item() <= 1e-2 * ref.abs().max().item(), _diagnose(got, ref, f"stem slab={mode}")
        outs[mode] = got
    # same products, different fp32 summation order, one bf16 rounding each
    assert (outs["1"] - outs["0"]).abs().max().item() <= 2 ** -7 * ref.abs().max().item()


@pytest.mark.parametrize("dims,n", [((40, 64, 64), 1), ((13, 21, 11), 2), ((4, 16, 8), 1)])
def test_slab_kernel_3x3x3(ops, monkeypatch, dims, n):
    """ResNet layer1 conv2 shape (64 -> 64, 3^3, BN shift + ReLU): three z phases, ring wrap-around over > 132 tiles."""
    g = torch.Generator(device="cuda").manual_seed(32)
    x = torch.randn((n, *dims, 64), device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn((64, 64, 3, 3, 3), device="cuda", generator=g) / (64 * 27) ** 0.5
    bias = torch.randn((64,), device="cuda", generator=g)
    got = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("NRPN_CONV_SLAB", mode)
        outs, refs = run_conv(ops, x, w, bias, 1, True, None, False)
        got[mode] = outs[0].float()
        assert not torch.isnan(got[mode]).any(), f"slab={mode}: unwritten outputs"
        assert (got[mode] - refs[0]).abs().max().item() <= 1e-2 * refs[0].abs().max().item(), _diagnose(got[mode], refs[0], f"3x3x3 slab={mode}")
    assert (got["1"] - got["0"]).abs().max().item() <= 2 ** -7 * refs[0].abs().max().item()


def test_slab_kernel_is_faster_than_brick(ops, monkeypatch):
    """Not a timing gate (no thresholds on a shared box) -- prints both timings so the run log records the A/B."""
    packed, wp, taps, bias, od, ref = _stem_case(ops, (160, 256, 256), 1, 33)
    y = torch.empty((1, *od, 64), dtype=torch.bfloat16, device="cuda")
    a = ops.ConvLevelArgs(packed, y, 1, packed.shape[1:4], od, 64)
    ms = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("NRPN_CONV_SLAB", mode)
        for _ in range(3):
            ops.conv3d_fprop([a], wp, bias, 64, 64, taps, relu=True)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            ops.conv3d_fprop([a], wp, bias, 64, 64, taps, relu=True)
        e1.record(); torch.cuda.synchronize()
        ms[mode] = e0.elapsed_time(e1) / 10
        got = y.float()
        assert (got - ref).abs().max().item() <= 1e-2 * ref.abs().max().item(), _diagnose(got, ref, f"full-size stem slab={mode}")
    print(f"\n[stem 160x256x256] slab {ms['1']:.3f} ms, brick {ms['0']:.3f} ms")


@pytest.mark.parametrize("dims,cin,cout,stride,resmode,relu", [
    ((13, 9, 7), 64, 256, 1, "same", True),        # ResNet c3 + residual, ragged bricks (TMA store clips)
    ((40, 32, 24), 256, 64, 1, None, True),        # c1, > 132 tiles
    ((9, 12, 11), 512, 128, 2, None, False),       # stride-2 1^3 through the sub-sampled tensor map
    ((13, 9, 7), 512, 256, 1, "up", False),        # FPN lateral + nearest-upsampled coarser level: stays on the register epilogue
])
def test_tma_epilogue_matches_register_epilogue(ops, monkeypatch, dims, cin, cout, stride, resmode, relu):
    """The shared-memory / cp.async.bulk.tensor epilogue of the 1^3 layers performs the same fp32 operations in the same order
    as the register epilogue: outputs must be bit-identical, and both within tolerance of fp32 PyTorch."""
    g = torch.Generator(device="cuda").manual_seed(41)
    x = torch.randn((2, *dims, cin), device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn((cout, cin, 1, 1, 1), device="cuda", generator=g) / cin ** 0.5
    bias = torch.randn((cout,), device="cuda", generator=g)
    od = tuple((d - 1) // stride + 1 for d in dims)
    res = None
    if resmode == "same":
        res = torch.randn((2, *od, cout), device="cuda", generator=g).to(torch.bfloat16)
    elif resmode == "up":
        res = torch.randn((2, *tuple((d + 1) // 2 for d in od), cout), device="cuda", generator=g).to(torch.bfloat16)
    got = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("NRPN_CONV_TMA_EPI", mode)
        outs, refs = run_conv(ops, x, w, bias, stride, relu, res, False)
        assert not torch.isnan(outs[0].float()).any(), f"tma_epi={mode}: unwritten outputs"
        assert (outs[0].float() - refs[0]).abs().max().item() <= 1e-2 * refs[0].abs().max().item(), _diagnose(outs[0].float(), refs[0], f"tma_epi={mode}")
        got[mode] = outs[0]
    assert torch.equal(got["1"], got["0"])


@pytest.mark.parametrize("dims,cin,cout,k", [((9, 12, 10), 64, 128, 3), ((8, 8, 16), 256, 64, 1), ((10, 13, 9), 128, 128, 3)])
def test_conv_data_gradient_runs_on_the_forward_kernel(ops, dims, cin, cout, k):
    """dL/dx of a stride-1 'same' Conv3d = the same implicit GEMM with mirrored taps and transposed matrices
    (packing.pack_conv_weight_dgrad); checked against torch.autograd on the bf16-rounded operands."""
    from nerf_rpn_b200 import packing
    g = torch.Generator(device="cuda").manual_seed(51)
    w = (torch.randn((cout, cin, k, k, k), device="cuda", generator=g) / (cout * k ** 3) ** 0.5).to(torch.bfloat16).float()
    dy = torch.randn((2, *dims, cout), device="cuda", generator=g).to(torch.bfloat16)
    x = torch.zeros((2, cin, *dims), device="cuda", requires_grad=True)
    y = F.conv3d(x, w, padding=k // 2)
    (ref,) = torch.autograd.grad(y, x, dy.float().permute(0, 4, 1, 2, 3))
    ref = ref.permute(0, 2, 3, 4, 1)
    wp, taps = packing.pack_conv_weight_dgrad(w.cpu())
    shift = torch.zeros(wp.shape[1], device="cuda")
    dx = torch.full((2, *dims, cin), float("nan"), dtype=torch.float32, device="cuda")
    a = ops.ConvLevelArgs(dy, dx, 2, dims, dims, cin)
    ops.conv3d_fprop([a], wp.cuda(), shift, cout, cin, taps, out_fp32=True)
    torch.cuda.synchronize()
    assert not torch.isnan(dx).any()
    assert (dx - ref).abs().max().item() <= 2e-3 * ref.abs().max().item(), _diagnose(dx, ref, "dgrad")


@pytest.mark.parametrize("level_dims,cin,cout,k,dtype", [
    ([(8, 8, 16)], 64, 128, 3, torch.bfloat16),
    ([(9, 12, 10), (5, 6, 5)], 128, 256, 3, torch.bfloat16),        # two levels sharing the weights, ragged bricks
    ([(6, 7, 9)], 256, 128, 1, torch.float16),
])
@pytest.mark.parametrize("operands", ["channels_last", "planar"])
def test_conv_weight_gradient_vs_autograd(ops, level_dims, cin, cout, k, dtype, operands):
    """dW of a stride-1 'same' Conv3d on wgmma (K = voxels; channels-last tensors as MN-major operands, or the earlier planar staging copies)
    against torch.autograd on the rounded operands."""
    g = torch.Generator(device="cuda").manual_seed(61)
    w = torch.zeros((cout, cin, k, k, k), device="cuda", requires_grad=True)
    dys, xs, ref = [], [], torch.zeros_like(w)
    for dims in level_dims:
        x = torch.randn((2, *dims, cin), device="cuda", generator=g).to(dtype)
        dy = torch.randn((2, *dims, cout), device="cuda", generator=g).to(dtype)
        y = F.conv3d(x.float().permute(0, 4, 1, 2, 3), w, padding=k // 2)
        (gw,) = torch.autograd.grad(y, w, dy.float().permute(0, 4, 1, 2, 3))
        ref += gw
        assert torch.equal(ops.to_planar(x), x.permute(0, 4, 1, 2, 3))
        sh = ops.to_planar(x, 1)                                        # out[z'] = x[z' + 1]
        assert torch.equal(sh[..., :-1], x.permute(0, 4, 1, 2, 3)[..., 1:]) and sh[..., -1].abs().max().item() == 0
        xs.append(x); dys.append(dy)
    taps = [(a - k // 2, b - k // 2, c - k // 2) for a in range(k) for b in range(k) for c in range(k)]
    dw = ops.conv3d_wgrad(dys, xs, taps, operands=operands)
    torch.cuda.synchronize()
    refp = ref.permute(2, 3, 4, 0, 1).reshape(len(taps), cout, cin)
    assert not torch.isnan(dw).any()
    assert (dw - refp).abs().max().item() <= 2e-3 * refp.abs().max().item(), _diagnose(dw, refp, "wgrad")
    assert torch.equal(dw, ops.conv3d_wgrad(dys, xs, taps, operands=operands)), "weight gradients must be bit-reproducible"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_bias_grad_and_relu_backward(ops, dtype):
    g = torch.Generator(device="cuda").manual_seed(71)
    dy = torch.randn((2, 9, 11, 10, 256), device="cuda", generator=g).to(dtype)
    act = torch.randn((2, 9, 11, 10, 256), device="cuda", generator=g).to(dtype)
    act[0, 0, 0, 0, :8] = 0                                                   # exactly zero activations: gradient must be cut
    db = ops.bias_grad(dy)
    ref = dy.float().sum(dim=(0, 1, 2, 3))
    assert (db - ref).abs().max().item() <= 1e-4 * max(1.0, ref.abs().max().item())
    assert torch.equal(db, ops.bias_grad(dy))
    want = torch.where(act.float() > 0, dy, torch.zeros_like(dy))
    got = ops.relu_backward_(dy.clone(), act)
    assert torch.equal(got, want)


WSPLIT_CASES = [
    # name, dims, cin, cout, k, stride, relu, res mode  -> kernel variant exercised
    ("ws_1x1_256_64_res", (8, 12, 16), 256, 64, 1, 1, True, "same"),       # igemm<64,2,2,tma-epilogue,wsplit>
    ("ws_1x1_s2_256_128", (9, 12, 11), 256, 128, 1, 2, True, None),        # igemm<64,2,3,wsplit> path (stride-2 1^3)
    ("ws_1x1_up_512_256", (13, 9, 7), 512, 256, 1, 1, False, "up"),        # igemm<64,2,3,wsplit> with up-sampled residual
    ("ws_3x3_128_128", (20, 32, 32), 128, 128, 3, 1, True, None),          # igemm<128,4,1,wsplit>
    ("ws_3x3_256_256", (10, 16, 16), 256, 256, 3, 1, True, None),          # igemm<256,2,1,wsplit> or <64,6,1,wsplit> (narrow)
    ("ws_3x3_512_512_narrow", (5, 8, 8), 512, 512, 3, 1, True, None),      # igemm<64,6,1,wsplit>
]


@pytest.mark.parametrize("name,dims,cin,cout,k,stride,relu,resmode", WSPLIT_CASES)
def test_conv_weight_split_cases(ops, name, dims, cin, cout, k, stride, relu, resmode):
    """nrpn_conv_desc.wsplit: weights as hi + lo fp16 planes.  Against an fp32 conv on the UNROUNDED weights (fp16 activations)
    the error must be accumulation-order only -- an order of magnitude below what single-fp16 weights give -- and the launch
    must hit the wsplit variant of every igemm template."""
    from nerf_rpn_b200 import packing
    g = torch.Generator(device="cuda").manual_seed(hash(name) % 1000)
    x = torch.randn((2, *dims, cin), device="cuda", generator=g).to(torch.float16)
    w = torch.randn((cout, cin, k, k, k), device="cuda", generator=g) / (cin * k ** 3) ** 0.5
    bias = torch.randn((cout,), device="cuda", generator=g)
    od = tuple((d - 1) // stride + 1 for d in dims)
    res = None
    if resmode == "same":
        res = torch.randn((2, *od, cout), device="cuda", generator=g).to(torch.float16)
    elif resmode == "up":
        res = torch.randn((2, *tuple((d + 1) // 2 for d in od), cout), device="cuda", generator=g).to(torch.float16)
    errs = {}
    for split in (False, True):
        wp, taps = packing.pack_conv_weight(w, dtype=torch.float16, split=split)
        shift = packing.pad_shift(bias, wp.shape[-2]).cuda()
        y = torch.full((2, *od, cout), float("nan"), dtype=torch.float32, device="cuda")
        a = [ops.ConvLevelArgs(x, y, 2, dims, od, cout, res=res, res_dims=None if res is None else res.shape[1:4],
                               ldr=0 if res is None else res.shape[-1])]
        variant = ops.conv3d_variant(a, wp, shift, cin, cout, taps, stride=stride, relu=relu, out_fp32=True)
        assert ("wsplit" in variant) == split, variant
        ops.conv3d_fprop(a, wp, shift, cin, cout, taps, stride=stride, relu=relu, out_fp32=True)
        torch.cuda.synchronize()
        w_exact, _ = packing.pack_conv_weight(w, dtype=torch.float32)
        ref = emulate_conv(x.float(), w_exact.cuda(), taps, shift, od, stride=stride, relu=relu, res=res)[..., :cout]
        assert not torch.isnan(y).any(), f"{name} [{variant}]: unwritten outputs"
        errs[split] = ((y - ref).norm() / ref.norm()).item()
        print(f"{name} [{variant}]: norm-wise rel err vs exact-weight fp32 conv {errs[split]:.3e}")
    assert errs[True] < 5e-5, errs          # fp32 accumulation order + the lo plane's fp16-subnormal step only (measured 1.8e-5 at K = 13 824)
    assert errs[False] > 5 * errs[True]     # single fp16 weights: ~1.4e-4 rounding error per weight


@pytest.mark.parametrize("layout", ["dataset", "ncdhw"])
def test_pack_stem_density_to_alpha_fused(ops, layout, tmp_path):
    """SURVEY.md 8(f) rank 2: datasets.py:50-52,165-167 (--normalize_density: alpha = clip(1 - exp(-exp(sigma)/100), 0, 1)) applied by the stem
    packing kernel on a RAW-density grid == packing the grid numpy already converted on the host; the scene comes from an .npz through
    nerf_rpn_b200.io.read_rgbsigma (pinned, on-disk order)."""
    from nerf_rpn_b200 import io
    rng = np.random.default_rng(3)
    raw = rng.random((10, 12, 9, 4)).astype(np.float32)
    raw[..., 3] = rng.normal(2.0, 3.0, raw.shape[:3]).astype(np.float32)                 # densities: any real number
    np.savez(str(tmp_path / "s.npz"), rgbsigma=raw)
    host = io.read_rgbsigma(str(tmp_path / "s.npz"))
    assert host.is_pinned() and host.shape == (4, 10, 12, 9) and not host.is_contiguous()
    ref = raw.copy()
    ref[..., 3] = np.clip(1.0 - np.exp(-np.exp(ref[..., 3]) / 100.0), 0.0, 1.0)        # BaseDataset.density_to_alpha, verbatim
    g_raw = host.cuda()[None] if layout == "dataset" else host.cuda().contiguous()[None]
    g_ref = torch.from_numpy(ref).permute(3, 0, 1, 2).contiguous().cuda()[None]
    got = ops.pack_stem_input(g_raw, dtype=torch.float16, density_to_alpha=True)
    want = ops.pack_stem_input(g_ref, dtype=torch.float16)
    torch.cuda.synchronize()
    assert (got.float() - want.float()).abs().max().item() <= 2.0 ** -10                  # expf vs numpy's exp: <= 1 fp16 ulp of values in [0, 1]
