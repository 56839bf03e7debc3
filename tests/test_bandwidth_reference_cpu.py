"""The float64 references of the bandwidth-kernel tests (tests/emulate.py) against torch in float64, and negative controls: each bound
of tests/test_gpu_bandwidth_kernels.py, evaluated on the reference's own scale, must reject a reference with one deliberate mistake by
at least 4x on the row the mistake is aimed at."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import test_gpu_bandwidth_kernels as K
from tests.emulate import (MAXPOOL3_TAPS, encode_targets64, reference_adamw64, reference_bn_apply64, reference_bn_backward64,
                           reference_bn_stats64, reference_grad_norm64, reference_maxpool2_ceil, reference_maxpool3_argmax,
                           reference_maxpool3_backward64, reference_rpn_loss64, reference_upsample_backward64, rpn_anchors_f32)

EPS = K.EPS


def _close(a, b, tol=1e-10):
    torch.testing.assert_close(a, b, rtol=tol, atol=tol)


def _bn_case(name, rows=None):
    row = K.ROWS[name]
    if rows is not None:
        row = K.BN(row.c, rows, row.dtype, row.kind, row.mean, row.std, row.running)
    return row, K.bn_operands(row, name, "cpu")


@pytest.mark.parametrize("name", ["bn_c96_1000_fp16", "bn_c2048_333_bf16", "bn_small_s4_c2048_plain_bf16", "bn_mean30_c64_fp16"])
def test_bn_references_match_torch_autograd(name):
    row, (y, res, gamma, beta, dout, rm0, rv0) = _bn_case(name, rows=min(K.ROWS[name].rows, 2000))
    relu = row.kind != "plain"
    st = reference_bn_stats64(y, EPS, rm0, rv0, 0.1)
    rm, rv = rm0.double().clone(), rv0.double().clone()
    y64 = y.double().requires_grad_(True)
    g64, b64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    lin = F.batch_norm(y64, rm, rv, g64, b64, True, 0.1, EPS)
    _close(st["running_mean"], rm); _close(st["running_var"], rv)
    _close(st["mean"], y.double().mean(0)); _close(st["var"], y.double().var(0, unbiased=False))
    out_t = lin + (res.double() if res is not None else 0.0)
    out_t = out_t.clamp_min(0) if relu else out_t
    ref, scale = reference_bn_apply64(y, res, st["mean"], st["rstd"], gamma, beta, relu)
    _close(ref, out_t.detach())
    assert bool((ref.abs() <= scale + 1e-12).all())
    act = out_t.detach().to(y.dtype)                                     # the kernel's mask comes from its 16-bit output
    mask = (act > 0).double() if relu else torch.ones_like(lin)
    lin.backward(dout.double() * mask)
    rb = reference_bn_backward64(dout, act, y, st["mean"], st["rstd"], gamma, relu)
    _close(rb["dgamma"], g64.grad); _close(rb["dbeta"], b64.grad); _close(rb["dy"], y64.grad)
    _close(rb["dres"], dout.double() * mask, 0)
    assert bool((rb["dgamma"].abs() <= rb["mag_dgamma"] + 1e-12).all()) and bool((rb["dy"].abs() <= rb["mag_dy"] + 1e-12).all())


def test_bn_chain_length():
    assert K.bn_chain(1_310_720, 64) == 139 + 32                       # config 4's stem: 4429 rows per block, 32 lanes
    assert K.bn_chain(18, 2048) == 2 and K.bn_chain(333, 2048) == 3
    assert K.bn_chain(1000, 96) == 1 + 21                            # 4 rows per block, 21 lanes of 12 channel groups


@pytest.mark.parametrize("name", ["pool_small_stem_bf16", "pool_odd_c16_n2_randn_fp16", "pool_9x12x10_n2_randn_bf16"])
def test_maxpool_references_match_torch(name):
    row = K.ROWS[name]
    g = K._gen(name, "cpu")
    dims = row.dims if math.prod(row.dims) < 100_000 else (12, 10, 9)
    x = torch.randn(row.n, *dims, 8, generator=g)
    x = ((x - 2.0).clamp_min(0) if row.post_relu else x).to(K.DTYPE[row.dtype])
    out, code = reference_maxpool3_argmax(x)
    xc = x.double().permute(0, 4, 1, 2, 3).contiguous().requires_grad_(True)
    o, ind = F.max_pool3d(xc, 3, 2, 1, return_indices=True)
    assert torch.equal(out.double(), o.detach().permute(0, 2, 3, 4, 1))
    X, Y, Z = dims
    od = out.shape[1:4]
    i, j, k = torch.meshgrid(*(torch.arange(e) for e in od), indexing="ij")
    taps = torch.tensor(MAXPOOL3_TAPS)[code.long()]                     # (n, Xo, Yo, Zo, C, 3)
    flat = ((2 * i[None, ..., None] + taps[..., 0]) * Y + 2 * j[None, ..., None] + taps[..., 1]) * Z + 2 * k[None, ..., None] + taps[..., 2]
    assert torch.equal(flat, ind.permute(0, 2, 3, 4, 1)), "not torch's first maximum"
    if row.post_relu:
        assert float((out == 0).float().mean()) > 0.05
    dy = torch.randn(out.shape, generator=g).to(x.dtype)
    o.backward(dy.double().permute(0, 4, 1, 2, 3))
    ref, mag = reference_maxpool3_backward64(dy, code, dims)
    _close(ref, xc.grad.permute(0, 2, 3, 4, 1))
    assert bool((ref.abs() <= mag).all())
    y2 = reference_maxpool2_ceil(x)
    _close(y2.double(), F.max_pool3d(x.double().permute(0, 4, 1, 2, 3), 2, 2, ceil_mode=True).permute(0, 2, 3, 4, 1), 0)


@pytest.mark.parametrize("fine,coarse", [((46, 9, 7), (14, 5, 4)), ((12, 16, 33), (6, 8, 17)), ((25, 25, 17), (13, 13, 9))])
def test_upsample_reference_matches_interpolate_backward(fine, coarse):
    g = torch.Generator().manual_seed(sum(fine))
    df = torch.randn(2, *fine, 8, generator=g).to(torch.bfloat16)
    dc = torch.randn(2, *coarse, 8, generator=g).to(torch.bfloat16)
    ref, mag, terms = reference_upsample_backward64(df, dc)
    cz = torch.zeros(2, 8, *coarse, dtype=torch.float64, requires_grad=True)
    F.interpolate(cz, size=fine, mode="nearest").backward(df.double().permute(0, 4, 1, 2, 3))
    _close(ref, dc.double() + cz.grad.permute(0, 2, 3, 4, 1))
    assert bool((ref.abs() <= mag).all()) and terms >= 8


def test_anchor_indexing_matches_anchor_generator():
    from nerf_rpn_b200.model.anchor import AnchorGenerator3D
    from oracle import ref_gpu
    ag = AnchorGenerator3D(ref_gpu.ANCHOR_SIZES, ref_gpu.ASPECT)
    feats = [torch.empty(1, 1, *d) for d in K.LOSS_FD]
    anchors = ag(torch.empty(1, 4, *K.LOSS_DIMS), feats)[0][0]
    strides = [tuple(K.LOSS_DIMS[k] // d[k] for k in range(3)) for d in K.LOSS_FD]
    flat = torch.arange(anchors.shape[0])
    _, _, _, an = rpn_anchors_f32(flat, K.LOSS_FD, strides, ag.cell_anchors_np(), 13)
    assert torch.equal(an, anchors.float())


@pytest.mark.parametrize("name", ["loss_obb_fp16", "loss_aabb_bf16", "loss_obb_theta_edges_fp16", "loss_background_bf16"])
def test_rpn_loss_reference_matches_torch_on_oracle_targets(name):
    from oracle import loss_oracle as lo
    row = K.ROWS[name]
    calls, cells, strides, A, code = K.loss_setup(row, name, "cpu")
    preds, pos, neg, gt = calls[0]
    samp = torch.cat([pos, neg])
    lvl, vox, a, an = rpn_anchors_f32(samp, K.LOSS_FD, strides, cells, A)
    npos = pos.numel()
    logits = torch.stack([preds[l][v, aa] for l, v, aa in zip(lvl.tolist(), vox.tolist(), a.tolist())])
    prow = torch.stack([preds[l][v, A + aa * code: A + (aa + 1) * code] for l, v, aa in zip(lvl[:npos].tolist(), vox[:npos].tolist(), a[:npos].tolist())]) \
        if npos else torch.zeros(0, code)
    t, tmag = encode_targets64(an[:npos], gt, row.rotated)
    if npos:
        an_np, gt_np = an[:npos].numpy(), gt.numpy()
        enc = lo.encode_obb_midpoint(an_np, gt_np) if row.rotated else lo.encode_aabb(gt_np, an_np)
        assert bool(((t - torch.from_numpy(enc).double()).abs() <= K.target_bound(tmag) + 2.0 ** -24 * t.abs()).all())
        t = torch.from_numpy(enc).double()                              # torch on the oracle's targets
    norm = float(samp.numel())
    ref = reference_rpn_loss64(prow, logits, npos, t, norm, 1.0, 5.0, 256.0)
    x = logits.double().requires_grad_(True)
    d = prow.double().requires_grad_(True)
    lab = torch.cat([torch.ones(npos), torch.zeros(neg.numel())]).double()
    l_obj = F.binary_cross_entropy_with_logits(x, lab)
    l_reg = F.smooth_l1_loss(d, t, beta=1 / 9, reduction="sum") / norm
    (l_obj + 5.0 * l_reg).backward()
    assert abs(ref["l_obj"] - l_obj.item()) <= 1e-12 and abs(ref["l_reg"] - l_reg.item()) <= 1e-12
    _close(ref["dlogit"], x.grad * 256.0)
    if npos:
        _close(ref["ddelta"], d.grad * 256.0)


def test_frozen_head_range_matches_the_model():
    from nerf_rpn_b200.model.anchor import RPNHead
    from nerf_rpn_b200.model.feature_extractor import Bottleneck, ResNet_FPN_256
    backbone = ResNet_FPN_256(Bottleneck, [3, 4, 6, 3], input_dim=4, is_max_pool=True)
    assert sum(p.numel() for p in backbone.parameters()) == K.HEAD_LO and K.HEAD_LO % 4 == 0
    for rotated in (True, False):
        n = sum(p.numel() for p in RPNHead(256, 13, 4, rotate=rotated).parameters())
        assert n == K.HEAD_N[rotated] and n % 2 == 1


def _opt_case(name, step_i=0, n=None):
    row = K.ROWS[name]
    n = n or row.n
    g = torch.Generator().manual_seed(len(name))
    p = torch.randn(n, generator=g)
    m = torch.randn(n, generator=g) * 1e-3 if row.warm else torch.zeros(n)
    v = torch.rand(n, generator=g) * 1e-6 if row.warm else torch.zeros(n)
    grad = torch.randn(n, generator=g) * (row.grad_std[step_i] / row.inv_scale)
    return row, p, grad, m, v


def _hp(row):
    lr, b1, b2, eps, wd = (K.f32(v) for v in K.OPT_HP)
    return K.f32(row.max_norm), K.f32(row.inv_scale), lr, b1, b2, eps, wd


@pytest.mark.parametrize("name", ["opt_3steps_step2_clipped", "opt_frozen_head_obb_fp16", "opt_max_norm0"])
def test_norm_and_adamw_references_match_torch(name):
    row = K.ROWS[name]
    max_norm, inv, lr, b1, b2, eps, wd = _hp(row)
    _, p, _, m, v = _opt_case(name, n=10_007)
    q = torch.nn.Parameter(p.double().clone())
    opt = torch.optim.AdamW([q], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd)
    g = torch.Generator().manual_seed(3)
    p64, m64, v64 = p.double(), m.double(), v.double()
    for step, std in zip(row.steps, row.grad_std):
        grad = (torch.randn(10_007, generator=g) * (std / row.inv_scale)).float()
        q.grad = grad.double() * inv
        tn = torch.nn.utils.clip_grad_norm_([q], max_norm) if max_norm > 0 else None
        opt.step()
        norm = reference_grad_norm64(grad, inv)
        if tn is not None:
            assert abs(norm - tn.item()) <= 1e-12 * norm
        p64, m64, v64, _ = reference_adamw64(p64, grad, m64, v64, norm, max_norm, inv, lr, b1, b2, eps, wd, step)
        _close(p64, q.data, 1e-12)
        _close(m64, opt.state[q]["exp_avg"], 1e-12)


# ------------------------------------------------------------------------------------------------ negative controls
def _rejects(flawed, ref, bound, what):
    ratio = float(((flawed - ref).abs() / bound).max())
    assert ratio >= 4.0, f"{what}: the bound rejects the flawed reference only by {ratio:.3g}x"
    return ratio


def test_control_biased_running_variance():
    row, (y, res, gamma, beta, dout, rm0, rv0) = _bn_case("bn_c2048_333_bf16")
    ref = reference_bn_stats64(y, EPS, rm0, rv0, 0.1)
    bad = reference_bn_stats64(y, EPS, rm0, rv0, 0.1, flaw="biased_running_var")
    _rejects(bad["running_var"], ref["running_var"], K.bn_stats_bounds(ref, row.rows, row.c)["running_var"], "biased running variance")


@pytest.mark.parametrize("flaw,key", [("relu_mask_dropped", "dy"), ("dres_unmasked", "dres")])
def test_control_bn_backward(flaw, key):
    row, (y, res, gamma, beta, dout, rm0, rv0) = _bn_case("bn_c96_1000_fp16")
    st = reference_bn_stats64(y, EPS)
    mean, rstd = st["mean"].float(), st["rstd"].float()
    act, _ = reference_bn_apply64(y, res, mean, rstd, gamma, beta, True)
    act = act.to(y.dtype)
    ref = reference_bn_backward64(dout, act, y, mean, rstd, gamma, True)
    bad = reference_bn_backward64(dout, act, y, mean, rstd, gamma, True, flaw=flaw)
    dt = K.DTYPE[row.dtype]
    bound = K.act_bound(ref["dy"], ref["mag_dy"], dt, 10) if key == "dy" else K.HALF_ULP[dt] * ref["dres"].abs() + K.E
    _rejects(bad[key], ref[key], bound, flaw)
    if key == "dy":
        _rejects(bad["dgamma"], ref["dgamma"], K.bn_sum_bounds(ref, row.rows, row.c)[0], flaw + " (dgamma)")


def test_control_last_maximum():
    row = K.ROWS["pool_small_stem_bf16"]
    g = K._gen("pool_small_stem_bf16", "cpu")
    x = (torch.randn(row.n, *row.dims, row.c, generator=g) - 2.0).clamp_min(0).to(torch.bfloat16)
    _, code = reference_maxpool3_argmax(x)
    _, bad_code = reference_maxpool3_argmax(x, flaw="last_max")
    dy = torch.randn(code.shape, generator=g).to(torch.bfloat16)
    ref, mag = reference_maxpool3_backward64(dy, code, row.dims)
    bad, _ = reference_maxpool3_backward64(dy, bad_code, row.dims)
    _rejects(bad, ref, K.act_bound(ref, mag, torch.bfloat16, 8), "last maximum")


def test_control_float64_nearest_index():
    row = K.ROWS["up_46_from_14_bf16"]
    g = K._gen("up_46_from_14_bf16", "cpu")
    df = torch.randn(row.n, *row.fine, row.c, generator=g).to(torch.bfloat16)
    dc = torch.randn(row.n, *row.coarse, row.c, generator=g).to(torch.bfloat16)
    ref, mag, terms = reference_upsample_backward64(df, dc)
    bad, _, _ = reference_upsample_backward64(df, dc, flaw="float64_index")
    _rejects(bad, ref, K.act_bound(ref, mag, torch.bfloat16, terms + 1), "float64 nearest index")


@pytest.mark.parametrize("name,flaw,key", [("loss_aabb_fp16", "beta_1", "ddelta"), ("loss_obb_fp16", "bce_over_positives", "dlogit")])
def test_control_rpn_loss(name, flaw, key):
    row = K.ROWS[name]
    calls, cells, strides, A, code = K.loss_setup(row, name, "cpu")
    preds, pos, neg, gt = calls[0]
    samp = torch.cat([pos, neg])
    lvl, vox, a, an = rpn_anchors_f32(samp, K.LOSS_FD, strides, cells, A)
    npos = pos.numel()
    logits = torch.stack([preds[l][v, aa] for l, v, aa in zip(lvl.tolist(), vox.tolist(), a.tolist())])
    prow = torch.stack([preds[l][v, A + aa * code: A + (aa + 1) * code] for l, v, aa in zip(lvl[:npos].tolist(), vox[:npos].tolist(), a[:npos].tolist())])
    t, tmag = encode_targets64(an[:npos], gt, row.rotated)
    norm = float(samp.numel())
    ref = reference_rpn_loss64(prow, logits, npos, t, norm, 1.0, row.w_reg, 256.0)
    bad = reference_rpn_loss64(prow, logits, npos, t, norm, 1.0, row.w_reg, 256.0, flaw=flaw)
    bl, bd, bo, br = K.loss_bounds(ref, t, tmag, prow, K.DTYPE[row.dtype], norm, 1.0, row.w_reg, 256.0)
    _rejects(bad[key], ref[key], bd if key == "ddelta" else bl, flaw)
    _rejects(torch.tensor(bad["l_reg" if key == "ddelta" else "l_obj"]), torch.tensor(ref["l_reg" if key == "ddelta" else "l_obj"]),
             torch.tensor(br if key == "ddelta" else bo), flaw + " (loss)")


@pytest.mark.parametrize("name,step_i,flaw", [("opt_3steps_step2_clipped", 0, "no_bias_correction"), ("opt_late_step", 0, "l2_decay"),
                                              ("opt_not_clipped_warm", 0, "unclamped_clip")])
def test_control_adamw(name, step_i, flaw):
    row, p, grad, m, v = _opt_case(name, step_i, n=100_003)
    max_norm, inv, lr, b1, b2, eps, wd = _hp(row)
    step = row.steps[step_i]
    norm = K.f32(reference_grad_norm64(grad, inv))
    if flaw == "unclamped_clip":
        assert norm < max_norm                                           # the row is aimed at an unclipped step
    ref = reference_adamw64(p, grad, m, v, norm, max_norm, inv, lr, b1, b2, eps, wd, step)
    bad = reference_adamw64(p, grad, m, v, norm, max_norm, inv, lr, b1, b2, eps, wd, step, flaw=flaw)
    bp, bm, bv = K.adamw_bounds(p, grad, m, v, ref, norm, max_norm, inv, lr, b1, b2, eps, step)
    _rejects(bad[0], ref[0], bp, flaw)


def test_row_names_are_unique_and_seeds_differ():
    seeds = {K._gen(n, "cpu").initial_seed() for n in K.ROWS}
    assert len(seeds) >= 0.95 * len(K.ROWS)
