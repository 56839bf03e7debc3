"""GPU: the VGG19-FPN backbones (VGG_FPN cfg AF / EF, strided stem) in the training step (nerf_rpn_b200/train.py).

1. The ceil-mode 2/2 max-pool with argmax and its backward against float64 statements of them (below, next to tests/emulate.py's
   reference_maxpool2_ceil), exact, in NaN guard bands.
2. The gradient helpers on the VGG convolution shapes tests/test_gpu_train_layer_grads.py does not cover, with that file's bounds.
3. One whole step against the unmodified reference's VGG_FPN in fp32 and under its own autocast, with the criteria of
   tests/test_gpu_train.py.  The conv biases in front of a BatchNorm have an analytically zero gradient: both sides produce rounding
   noise there, which AdamW turns into steps of up to ~lr, so those parameters are compared after the update with an absolute bound.
4. Frozen backbone, ragged batch and the all-reduce schedule of a VGG plan.
5. The drop-in autograd node and inference on the trained weights."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import emulate
from tests.test_gpu_train import _grad_metrics, _planted, _reference_step
from tests.test_gpu_train_layer_grads import (DIMS_S1, GUARD, HALF_ULP, _Engine, _draw, _levels_of_one_buffer, _nan_guarded, _plan,
                                              _reference, _within, _written)
from tests.test_gpu_train_ragged import _batch, _need_ref, _reference_batch_step
from tests.test_gpu_wgrad_variants import GAMMA

pytestmark = pytest.mark.gpu

DTYPES = (torch.bfloat16, torch.float16)
LR = 1e-4


def _p(t):
    import ctypes
    return ctypes.c_void_p(t.data_ptr())


def _s():
    import ctypes
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ------------------------------------------------------------------------------------------------ 1. the 2/2 ceil-mode pool
MAXPOOL2_TAPS = [(dx, dy, dz) for dx in (0, 1) for dy in (0, 1) for dz in (0, 1)]        # window position dx*4 + dy*2 + dz: x outer, z inner


def reference_maxpool2_ceil_argmax(x):
    """nrpn_maxpool3d_k2s2_ceil_argmax: the window position of the FIRST maximum of each nn.MaxPool3d(2, 2, ceil_mode=True) window in
    scan order (x outer, z inner; positions outside an odd extent never win), a NaN counting as a maximum.  x (N,X,Y,Z,C) 16-bit.
    Exact: returns (out in x's dtype, code uint8)."""
    n, X, Y, Z, C = x.shape
    xp = F.pad(x.float(), (0, 0, 0, Z % 2, 0, Y % 2, 0, X % 2), value=-math.inf)
    best = xp[:, 0::2, 0::2, 0::2].clone()                     # position 0 lies inside the map in every window
    code = torch.zeros(best.shape, dtype=torch.uint8, device=x.device)
    for p, (dx, dy, dz) in enumerate(MAXPOOL2_TAPS[1:], start=1):
        v = xp[:, dx::2, dy::2, dz::2]
        take = (v > best) | (v.isnan() & ~best.isnan())
        best = torch.where(take, v, best)
        code[take] = p
    return best.to(x.dtype), code


def reference_maxpool2_ceil_backward(dy, code, in_dims):
    """nrpn_maxpool3d_k2s2_ceil_backward: input voxel 2 o + (dx, dy, dz) of output o receives dy[o] when code[o] names its position, else
    0.  Exact (it only moves values): returns dy's dtype, (N,X,Y,Z,C)."""
    n, Xo, Yo, Zo, C = dy.shape
    X, Y, Z = in_dims
    out = torch.zeros((n, 2 * Xo, 2 * Yo, 2 * Zo, C), dtype=dy.dtype, device=dy.device)
    for p, (dx, dy_, dz) in enumerate(MAXPOOL2_TAPS):
        out[:, dx::2, dy_::2, dz::2] = torch.where(code == p, dy, torch.zeros_like(dy))
    return out[:, :X, :Y, :Z].contiguous()


# (n, extent, channels, content): "relu" = post-ReLU values with many all-zero windows (ties), "nan" = one NaN planted in a window
POOL_ROWS = [(2, (8, 6, 4), 128, "relu"), (2, (7, 5, 3), 256, "randn"), (1, (5, 8, 9), 512, "nan"), (2, (9, 7, 6), 128, "relu+nan"),
             (2, (4, 3, 10), 512, "relu")]


def _pool_input(n, d, c, content, dtype, g):
    x = torch.randn((n, *d, c), device="cuda", generator=g)
    if "relu" in content:
        x = x.clamp_min(0)
        x[:, ::2, ::2] = 0.0                                        # whole windows of zeros: the first position must win
    x = x.to(dtype)
    if "nan" in content:
        x[0, d[0] - 1, d[1] - 1, d[2] - 1, 3] = float("nan")        # in the last (partial along odd extents) window
        x[-1, 1, 0, 1, c - 1] = float("nan")
    return x


def _guarded(shape, dtype, fill):
    numel = math.prod(shape)
    buf = torch.full((numel + 2 * GUARD,), fill, dtype=dtype, device="cuda")
    return buf, buf[GUARD:GUARD + numel].view(shape)


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t


def _guards_kept(buf, fill, tag):
    ref = torch.full((GUARD,), fill, dtype=buf.dtype, device="cuda")
    assert torch.equal(_bits(buf[:GUARD]), _bits(ref)) and torch.equal(_bits(buf[-GUARD:]), _bits(ref)), f"{tag}: written outside the tensor"


def _same_values(a, b):
    """Equal as numbers, a NaN equal to a NaN (bf16 / fp16 NaN payloads are not part of the contract)."""
    return bool(((a == b) | (a.isnan() & b.isnan())).all())


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("n,d,c,content", POOL_ROWS)
def test_maxpool_k2s2_ceil_argmax_and_backward(n, d, c, content, dtype):
    from nerf_rpn_b200._lib import check, lib
    L, f16 = lib(), int(dtype == torch.float16)
    g = torch.Generator(device="cuda").manual_seed(sum(d) * 7 + c + n)
    x = _pool_input(n, d, c, content, dtype, g)
    od = tuple((v + 1) // 2 for v in d)
    nan = float("nan")
    out_buf, out = _guarded((n, *od, c), dtype, nan)
    idx_buf, idx = _guarded((n, *od, c), torch.uint8, 0xFF)
    check(L.nrpn_maxpool3d_k2s2_ceil_argmax(_p(x), n, *d, c, _p(out), _p(idx), f16, _s()), "maxpool_k2s2_ceil_argmax")
    inf_buf, inf = _guarded((n, *od, c), dtype, nan)
    check(L.nrpn_maxpool3d_k2s2_ceil(_p(x), n, *d, c, _p(inf), f16, _s()), "maxpool_k2s2_ceil")
    torch.cuda.synchronize()
    want = emulate.reference_maxpool2_ceil(x)
    want_out, want_idx = reference_maxpool2_ceil_argmax(x)
    tag = f"{n}x{d}x{c} {content} {str(dtype)[6:]}"
    _guards_kept(out_buf, nan, tag + " out"); _guards_kept(idx_buf, 0xFF, tag + " idx"); _guards_kept(inf_buf, nan, tag + " inference out")
    assert _same_values(out, want), f"{tag}: pooled map differs from nn.MaxPool3d(2, 2, ceil_mode=True)"
    assert _same_values(want_out, want)
    assert torch.equal(_bits(out), _bits(inf)), f"{tag}: the training pool's map differs from the inference pool's"
    assert torch.equal(idx, want_idx), f"{tag}: {int((idx != want_idx).sum())} argmax bytes differ"
    if "nan" in content:
        assert out.isnan().sum() >= 2
    if "relu" in content:
        assert int((want_idx == 0).sum()) > 0 and bool((out[:, 0, 0] == 0).any())

    dy = torch.randn((n, *od, c), device="cuda", generator=g).to(dtype)
    dx_buf, dx = _guarded((n, *d, c), dtype, nan)
    check(L.nrpn_maxpool3d_k2s2_ceil_backward(_p(dy), _p(idx), n, *d, c, _p(dx), f16, _s()), "maxpool_k2s2_ceil_backward")
    torch.cuda.synchronize()
    _guards_kept(dx_buf, nan, tag + " dx")
    want_dx = reference_maxpool2_ceil_backward(dy, want_idx, d)
    assert torch.equal(_bits(dx), _bits(want_dx)), f"{tag}: backward differs in {int((_bits(dx) != _bits(want_dx)).sum())} elements"


# ------------------------------------------------------------------------------------------------ 2. per-layer gradients
# (cout, cin, k): the VGG body's 3^3 convs whose shapes ResNet50-FPN lacks, and the 128-channel stage's lateral
VGG_LAYERS = [(128, 64, 3), (256, 128, 3), (512, 256, 3), (256, 128, 1)]


@pytest.mark.parametrize("cout,cin,k", VGG_LAYERS)
def test_vgg_layer_parameter_and_data_gradients(cout, cin, k):
    """_param_grad (weight + bias) and _dgrad (+ the residual the step adds through nrpn_add_inplace's operand) of one stride-1 VGG
    layer against float64 autograd, with the bounds of tests/test_gpu_train_layer_grads.py."""
    from nerf_rpn_b200.train import _TConv
    i = VGG_LAYERS.index((cout, cin, k))
    dtype = DTYPES[i % 2]
    tag = f"{cout}<-{cin} k{k} {str(dtype)[6:]}"
    g = torch.Generator(device="cuda").manual_seed(2000 + i)
    torch.manual_seed(2000 + i)
    conv = torch.nn.Conv3d(cin, cout, k, padding=k // 2, bias=True).cuda()
    with torch.no_grad():
        conv.bias.normal_(0, 0.5)
    n, eng = 2, _Engine(dtype)
    dw_buf, dw = _nan_guarded(conv.weight.numel(), torch.float32)
    db_buf, db = _nan_guarded(cout, torch.float32)
    layer = _TConv(eng, conv.weight, conv.bias, dw=dw, db=db)
    layer.repack()
    plan = _plan(eng, n)
    (dy,) = _levels_of_one_buffer((DIMS_S1,), n, cout, dtype, g)
    (x,) = _levels_of_one_buffer((DIMS_S1,), n, cin, dtype, g)
    res = _draw((n, *DIMS_S1, cin), dtype, g)
    dx_buf, dx = _nan_guarded(n * math.prod(DIMS_S1) * cin, dtype)
    plan._param_grad(layer, [dy], [x])
    plan._dgrad(layer, [dy], [dx.view(n, *DIMS_S1, cin)], [DIMS_S1], res=res)
    torch.cuda.synchronize()
    ref_w, ref_x, mag_w, mag_x = _reference(x, conv.weight.detach().to(dtype), dy, 1, k)
    ref_x, mag_x = ref_x + res.double(), mag_x + res.double().abs()
    got_x = _written(dx_buf, f"{tag} dX").view(ref_x.shape)
    wx = _within(got_x, ref_x, HALF_ULP[dtype] * ref_x.abs() + 2.0 ** -17 * mag_x + 2.0 ** -24, f"{tag} dX")
    got_w = _written(dw_buf, f"{tag} dW").view(conv.weight.shape)
    ww = _within(got_w, ref_w, 2.0 ** -24 * ref_w.abs() + GAMMA * mag_w, f"{tag} dW")
    ref_b, mag_b = dy.double().sum((0, 1, 2, 3)), dy.double().abs().sum((0, 1, 2, 3))
    wb = _within(_written(db_buf, f"{tag} db"), ref_b, 2.0 ** -24 * ref_b.abs() + GAMMA * mag_b, f"{tag} db")
    print(f"\n[vgg layer grads] {tag:22s} worst err/bound  dW {ww:.3g}  db {wb:.3g}  dX {wx:.3g}")


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_vgg_stem_bias_gradient(dtype):
    """The VGG stem conv's bias (ResNet's stem has none): _TrainPlan._bias_grad on the stem's dY0, as the stem's backward launches it."""
    from nerf_rpn_b200.train import _TConv
    g = torch.Generator(device="cuda").manual_seed(31)
    eng = _Engine(dtype)
    weight = torch.randn((64, 4, 7, 7, 7), device="cuda", generator=g) * 0.05
    bias = torch.randn(64, device="cuda", generator=g)
    db_buf, db = _nan_guarded(64, torch.float32)
    st = _TConv(eng, weight, bias, stride=2, need_dgrad=False, stem=True, dw=torch.empty_like(weight).reshape(-1), db=db)
    eng.stem = st
    plan = _plan(eng, 2)
    dy = _draw((2, 9, 6, 7, 64), dtype, g)
    plan._bias_grad(st, [dy])
    torch.cuda.synchronize()
    ref, mag = dy.double().sum((0, 1, 2, 3)), dy.double().abs().sum((0, 1, 2, 3))
    _within(_written(db_buf, "stem db"), ref, 2.0 ** -24 * ref.abs() + GAMMA * mag, "stem db")


# ------------------------------------------------------------------------------------------------ models
def _vgg_reference_model(rotated=False, seed=0, layers="AF", **rpn_kw):
    """The reference's own VGG_FPN(cfg, 4, True, 160) + anchor head + wrapper under torch.manual_seed(seed), in place of
    oracle.ref_gpu.build_reference_model's ResNet (`layers` carries the cfg)."""
    from oracle import ref_gpu
    ref = ref_gpu.load()
    torch.manual_seed(seed)
    bb = ref.feature_extractor.VGG_FPN(layers, 4, True, 160)
    ag = ref.anchor.AnchorGenerator3D(ref_gpu.ANCHOR_SIZES, ref_gpu.ASPECT)
    head = ref.anchor.RPNHead(256, ag.num_anchors_per_location()[0], 4, rotate=rotated)
    kw = dict(rpn_pre_nms_top_n_test=2500, rpn_post_nms_top_n_test=2500, rpn_nms_thresh=0.3, rpn_score_thresh=0.0, rotated_bbox=rotated)
    kw.update(rpn_kw)
    return ref.nerf_rpn.NeRFRegionProposalNetwork(bb, ag, head, **kw)


@pytest.fixture
def vgg_reference(monkeypatch):
    ref_gpu = _need_ref()
    monkeypatch.setattr(ref_gpu, "build_reference_model", _vgg_reference_model)
    return ref_gpu


def _vgg_model(cfg, rotated, state=None):
    from oracle import ref_gpu
    from nerf_rpn_b200.model.anchor import AnchorGenerator3D, RPNHead
    from nerf_rpn_b200.model.feature_extractor import VGG_FPN
    from nerf_rpn_b200.model.nerf_rpn import NeRFRegionProposalNetwork
    torch.manual_seed(0)
    backbone = VGG_FPN(cfg, 4, True, 160)
    head = RPNHead(256, 13, 4, rotate=rotated)
    if state is not None:
        backbone.load_state_dict(state["bsd"]); head.load_state_dict(state["hsd"])
    return NeRFRegionProposalNetwork(backbone, AnchorGenerator3D(ref_gpu.ANCHOR_SIZES, ref_gpu.ASPECT), head, rpn_fg_iou_thresh=0.35,
                                     rpn_bg_iou_thresh=0.2, rotated_bbox=rotated).cuda().train()


def _pre_bn_biases(model):
    return {id(m.bias) for m in model.backbone.layers.modules() if isinstance(m, torch.nn.Conv3d)}


def _no_tf32(fn):
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False; torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return fn()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _parity_checks(tag, cfg, precision, same, got_l, grads, r32, rac):
    cos_o, rel_o, per_o = _grad_metrics(grads, r32)
    cos_a, rel_a, per_a = _grad_metrics(rac["grads"], r32)
    print(f"{tag} sampler reproduces the reference's draws: {same}")
    print(f"{tag} losses: ours {got_l}  reference fp32 {r32['losses']}  reference autocast {rac['losses']}")
    print(f"{tag} gradient vs reference fp32: ours cosine {cos_o:.4f} rel {rel_o:.3f} | reference autocast cosine {cos_a:.4f} rel {rel_a:.3f}")
    worst = sorted(per_o.items(), key=lambda kv: -kv[1])[:4]
    print(f"{tag} worst large tensors ours {[(n, round(v, 3), 'autocast', round(per_a[n], 3)) for n, v in worst]}")
    checks = [(same, "the sampler did not reproduce the reference's draws")]
    for k in range(2):
        e_o, e_a = abs(got_l[k] - r32["losses"][k]), abs(rac["losses"][k] - r32["losses"][k])
        slack = (1e-2 if precision == "bf16" else 3e-3) * abs(r32["losses"][k])
        checks.append((e_o <= 3.0 * e_a + slack, f"loss {k}: ours off by {e_o}, autocast by {e_a}"))
    checks.append((cos_o >= cos_a - 0.08, f"gradient cosine {cos_o} vs autocast {cos_a}"))
    checks.append((rel_o <= 1.15 * rel_a + 0.02, f"gradient rel err {rel_o} vs autocast {rel_a}"))
    bad = [(n, v, per_a[n]) for n, v in per_o.items() if v > 1.25 * per_a[n] + 0.03]
    checks.append((not bad, f"tensors worse than the autocast reference: {bad[:5]}"))
    if cfg == "AF":                                                 # 9 normalisations: absolute bounds, as the shallow ResNet gets
        checks.append((cos_o >= (0.98 if precision == "fp16" else 0.80), f"AF: gradient cosine {cos_o}"))
    return checks


# ------------------------------------------------------------------------------------------------ 3. whole step vs the reference
@pytest.mark.parametrize("cfg,rotated,precision,dims", [
    ("AF", True, "fp16", (64, 96, 80)), ("AF", False, "bf16", (64, 96, 80)), ("EF", True, "bf16", (64, 96, 80)), ("EF", False, "fp16", (64, 96, 80)),
    ("AF", True, "bf16", (72, 90, 66)), ("EF", False, "fp16", (72, 90, 66)), ("EF", True, "bf16", (160, 256, 256))])
def test_vgg_training_step_vs_reference_autograd(vgg_reference, cfg, rotated, precision, dims):
    """One step against the unmodified reference's VGG_FPN in fp32 (+ clip + AdamW) and under its own autocast, same seed-0 weights, same
    planted boxes, same sampler draws; 72x90x66 has odd extents at every pool (ceil windows) and non-2x up-sampling in the FPN."""
    from nerf_rpn_b200.train import RPNTrainEngine
    grid, gt = _planted(dims, 16 if dims[0] >= 160 else 12, 11, rotated)
    grid, gt = grid.cuda(), gt.cuda()
    r32 = _no_tf32(lambda: _reference_step(rotated, cfg, grid, gt, None, optimise=True))
    rac = _no_tf32(lambda: _reference_step(rotated, cfg, grid, gt, torch.bfloat16 if precision == "bf16" else torch.float16))
    model = _vgg_model(cfg, rotated, r32)
    eng = RPNTrainEngine(model, precision=precision, lr=LR, weight_decay=0.01, clip_grad_norm=0.1, reg_loss_weight=5.0)
    plan = eng.plan(1, dims)
    torch.manual_seed(123)
    out = eng.forward_backward(grid[None], [gt])
    torch.cuda.synchronize()
    pos_o, neg_o, _ = plan.last_samples[0]
    same = set(pos_o.tolist()) == set(r32["samples"][0].tolist()) and set(neg_o.tolist()) == set(r32["samples"][1].tolist())
    params = list(model.backbone.parameters()) + list(model.rpn.head.parameters())
    grads = [eng.grad_of(p).view(p.shape).clone() / eng.loss_scale for p in params]
    tag = f"[VGG {cfg} {'OBB' if rotated else 'AABB'} {precision} {dims[0]}x{dims[1]}x{dims[2]}]"
    checks = _parity_checks(tag, cfg, precision, same, out.tolist(), grads, r32, rac)
    eng.optimizer_step()
    torch.cuda.synchronize()
    pre_bn = _pre_bn_biases(model)
    old_w = [v.float() for k, v in list(r32["bsd"].items()) + list(r32["hsd"].items()) if "running" not in k and "num_batches" not in k]
    rest = [(p.data.reshape(-1) - o.reshape(-1), r.reshape(-1) - o.reshape(-1)) for p, o, r in zip(params, old_w, r32["new"]) if id(p) not in pre_bn]
    d_ours, d_ref = torch.cat([a for a, _ in rest]), torch.cat([b for _, b in rest])
    bias_err = max((p.data - r).abs().max().item() for p, r in zip(params, r32["new"]) if id(p) in pre_bn)
    print(f"{tag} AdamW update: cosine {torch.nn.functional.cosine_similarity(d_ours, d_ref, dim=0).item():.4f}, |dw| ours {d_ours.norm().item():.4e} "
          f"reference {d_ref.norm().item():.4e}; pre-BN conv biases max |ours - reference| {bias_err:.3e} (lr {LR})")
    checks.append((abs(d_ours.norm().item() - d_ref.norm().item()) <= 0.02 * d_ref.norm().item(), "size of the first AdamW update"))
    checks.append((bias_err <= 2 * LR, f"pre-BN conv biases after the update differ by {bias_err}"))
    failed = [msg for ok, msg in checks if not ok]
    assert not failed, failed


# ------------------------------------------------------------------------------------------------ 4. modes
DIMS = (64, 96, 80)


@pytest.mark.parametrize("cfg,rotated,precision", [("AF", True, "bf16"), ("EF", False, "fp16")])
def test_vgg_frozen_step_bit_identical_to_full_step_head(cfg, rotated, precision):
    """As tests/test_gpu_train_frozen.py checks ResNet: losses and the head's range of flat_g of the frozen step equal the full step's bit for
    bit, eagerly and in graph replay; the backbone's gradients stay untouched; the frozen plan needs less pool memory."""
    from nerf_rpn_b200.train import RPNTrainEngine
    grid, gt = _planted(DIMS, 12, 11, rotated)
    grid, gt = grid.cuda()[None], [gt.cuda()]
    full = RPNTrainEngine(_vgg_model(cfg, rotated), precision=precision, seed=7)
    frozen = RPNTrainEngine(_vgg_model(cfg, rotated), precision=precision, seed=7, freeze_backbone=True)
    lo = full.head_lo
    assert lo == frozen.head_lo
    for it in range(4):                                          # eager, eager, capture + replay, replay
        lf = full.forward_backward(grid, gt).clone()
        lz = frozen.forward_backward(grid, gt).clone()
        torch.cuda.synchronize()
        assert torch.equal(lf, lz), (it, lf.tolist(), lz.tolist())
        assert torch.equal(full.flat_g[lo:], frozen.flat_g[lo:]), it
        assert not frozen.flat_g[:lo].any()
    assert len(frozen.plan(1, DIMS).bwd) == 1 and frozen.cache_stats()["graphs"] == 2
    zb, fb = frozen.cache_stats()["pool_bytes"], full.cache_stats()["pool_bytes"]
    print(f"[VGG {cfg}] pool bytes at {DIMS}: frozen {zb / 2**20:.1f} MiB, full {fb / 2**20:.1f} MiB")
    assert zb < fb


def test_vgg_ragged_training_step_vs_reference_autograd(vgg_reference):
    """Two differently sized scenes trained as the reference trains their padded batch, criteria of test 3."""
    from nerf_rpn_b200.train import RPNTrainEngine
    cfg, rotated, precision = "EF", True, "bf16"
    grids, gts = _batch([(64, 96, 80), (56, 80, 72)], 12, rotated)
    r32 = _no_tf32(lambda: _reference_batch_step(vgg_reference, rotated, cfg, grids, gts))
    rac = _no_tf32(lambda: _reference_batch_step(vgg_reference, rotated, cfg, grids, gts, torch.bfloat16))
    model = _vgg_model(cfg, rotated, r32)
    eng = RPNTrainEngine(model, precision=precision, lr=LR, weight_decay=0.01, clip_grad_norm=0.1, reg_loss_weight=5.0)
    torch.manual_seed(123)
    out = eng.forward_backward(grids, gts)
    torch.cuda.synchronize()
    plan = eng.plan_for(grids)
    assert plan.dims == (64, 96, 80) and plan.valid is not None
    same = all(set(p.tolist()) == set(rp.tolist()) and set(q.tolist()) == set(rq.tolist())
               for (p, q, _), (rp, rq) in zip(plan.last_samples, r32["samples"]))
    params = list(model.backbone.parameters()) + list(model.rpn.head.parameters())
    grads = [eng.grad_of(p).view(p.shape).clone() / eng.loss_scale for p in params]
    failed = [msg for ok, msg in _parity_checks(f"[VGG ragged {cfg}]", cfg, precision, same, out.tolist(), grads, r32, rac) if not ok]
    assert not failed, failed


@pytest.mark.parametrize("cfg", ["AF", "EF"])
def test_vgg_bucket_schedule_and_bwd_lo(cfg):
    """bucket_schedule over a VGG plan's bwd_lo covers [0, n_params) disjointly, and each backward stage's bwd_lo is the lowest flat offset it
    writes: with flat_g NaN-filled, the stages run one by one in execution order and the lowest written offset is checked after each."""
    from nerf_rpn_b200.train import RPNTrainEngine, bucket_schedule
    grid, gt = _planted(DIMS, 12, 11, True)
    eng = RPNTrainEngine(_vgg_model(cfg, True), precision="bf16", seed=7)
    plan = eng.plan(1, DIMS)
    assert len(plan.bwd) == 7 and len(plan.bwd_lo) == 7                 # stem, four stages, FPN, head
    for bucket in (1, 1 << 16, eng.n_params):
        sched = bucket_schedule(plan.bwd_lo, eng.n_params, bucket)
        cover = sorted((lo, hi) for _, lo, hi in sched)
        assert cover[0][0] == 0 and cover[-1][1] == eng.n_params and all(a[1] == b[0] for a, b in zip(cover, cover[1:]))
    torch.manual_seed(3)
    plan.forward_loss(grid.cuda()[None], [gt.cuda()])
    eng.flat_g.fill_(float("nan"))
    for i in range(len(plan.bwd) - 1, -1, -1):
        plan.bwd[i]()
        torch.cuda.synchronize()
        written = torch.nonzero(~eng.flat_g.isnan()).reshape(-1)
        assert int(written.min()) == plan.bwd_lo[i], (i, int(written.min()), plan.bwd_lo[i])
    assert not eng.flat_g.isnan().any()


# ------------------------------------------------------------------------------------------------ 5. drop-in
def test_vgg_dropin_gradients_then_eval_on_trained_weights():
    """model.train(): forward + loss.backward() through the autograd node gives the engine's own gradients (same samples); after torch AdamW
    steps, model.eval() runs inference on the trained weights: its features equal a fresh model's loaded from the trained state_dict."""
    cfg, rotated = "EF", True
    grid, gt = _planted(DIMS, 12, 5, rotated)
    grid, gt = grid.cuda(), gt.cuda()
    model = _vgg_model(cfg, rotated)
    opt = torch.optim.AdamW(model.parameters(), lr=LR, weight_decay=0.01)
    losses_seen = []
    for k in range(3):
        torch.manual_seed(10 + k)
        _, losses, _ = model([grid], [gt])
        assert all(v.grad_fn is not None for v in losses.values())
        loss = losses["loss_objectness"] + 5.0 * losses["loss_rpn_box_reg"]
        loss.backward()
        losses_seen.append(loss.item())
        if k == 0:
            params = list(model.backbone.parameters()) + list(model.rpn.head.parameters())
            got = [p.grad.clone() for p in params]
            eng = model.train_engine()
            plan = eng.plan_for(grid[None])
            plan.forced_samples = [(p, q) for p, q, _ in plan.last_samples]
            try:
                eng.forward_backward(grid[None], [gt])
            finally:
                del plan.forced_samples
            torch.cuda.synchronize()
            for p, g in zip(params, got):
                e = eng.grad_of(p).view(p.shape)
                assert torch.equal(g, e / eng.loss_scale if eng.loss_scale != 1.0 else e)
        torch.nn.utils.clip_grad_norm_(model.parameters(), 0.1)
        opt.step()
        opt.zero_grad()
    assert all(math.isfinite(v) for v in losses_seen)
    print(f"[VGG drop-in] losses over three steps on one planted scene: {losses_seen}")
    model.eval()
    fresh = _vgg_model(cfg, rotated)
    fresh.load_state_dict(model.state_dict())
    fresh.eval()
    with torch.no_grad():
        a = model.backbone(grid[None])
        b = fresh.backbone(grid[None])
    assert len(a) == 4 and all(torch.equal(x, y) for x, y in zip(a, b))
    changed = any(not torch.equal(p, q) for p, q in zip(model.backbone.parameters(), _vgg_model(cfg, rotated).backbone.parameters()))
    assert changed


def test_unsupported_backbones_still_raise():
    """A VGG_FPN with the stride-1 stem (input_size < 160) or without BatchNorm is refused with a message naming what the engine trains."""
    from nerf_rpn_b200.model.feature_extractor import VGG_FPN
    from nerf_rpn_b200.train import RPNTrainEngine
    for bb in (VGG_FPN("AF", 4, True, 128), VGG_FPN("AF", 4, False, 160)):
        model = _vgg_model("AF", True)
        model.backbone = bb.cuda()
        with pytest.raises(NotImplementedError, match="VGG_FPN"):
            RPNTrainEngine(model, precision="bf16")
