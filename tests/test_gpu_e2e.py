"""GPU end-to-end parity: NeRFRegionProposalNetwork (our module mirror -> fused engine -> CUDA kernels) against
(a) the reference's golden outputs on the same seeded weights/input and (b) the oracle.

Tolerances (stated per north_star, see DESIGN.md "precision"):
  - feature maps / logits: norm-wise relative error <= 2e-2.  The engine stores activations in bf16 (8-bit mantissa,
    BASELINE config 2 dtype), so the 1e-3 target of the fp32 reference is not reachable element-wise; measured
    values are printed.
  - post-processing: bit-identical to the oracle when fed the SAME head outputs (proposal sets, order, scores).
"""
import os

import numpy as np
import pytest
import torch

from oracle import box as obox
from oracle import rpn_post as rp
from tests import recipes

pytestmark = pytest.mark.gpu


class NS:
    pass


def _ns():
    from nerf_rpn_b200.model import anchor, feature_extractor
    NS.ResNet_FPN_256 = feature_extractor.ResNet_FPN_256
    NS.Bottleneck = feature_extractor.Bottleneck
    NS.AnchorGenerator3D = anchor.AnchorGenerator3D
    NS.RPNHead = anchor.RPNHead
    NS.VGG_FPN = feature_extractor.VGG_FPN
    return NS


def build(rot, g):
    from nerf_rpn_b200.model.nerf_rpn import NeRFRegionProposalNetwork
    backbone, ag, head = recipes.build_small_model(_ns(), rot, g)
    model = NeRFRegionProposalNetwork(backbone, ag, head, rpn_pre_nms_top_n_test=2500, rpn_post_nms_top_n_test=2500,
                                      rpn_nms_thresh=0.3, rpn_fg_iou_thresh=0.35, rpn_bg_iou_thresh=0.2,
                                      rpn_score_thresh=0.0, rotated_bbox=rot)
    return model.cuda().eval(), ag


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def oracle_post_from_engine(plan, eng, scene=0):
    code = eng.code
    logits = [p[scene].reshape(-1, 128)[:, :13].reshape(-1).cpu().numpy() for p in plan.pred]
    deltas = [p[scene].reshape(-1, 128)[:, 13:13 + 13 * code].reshape(-1, code).cpu().numpy() for p in plan.pred]
    return rp.rpn_proposals(logits, deltas, plan.feat_dims, plan.strides, eng.cells, plan.dims, eng.rotated,
                            eng.pre_n, eng.post_n, eng.nms_thresh, eng.score_thresh)


@pytest.mark.parametrize("name,rot", [("rpn_small_aabb", False), ("rpn_small_obb", True)])
def test_small_scene_vs_reference_golden(golden_dir, name, rot):
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    model, ag = build(rot, g)
    x = recipes.golden_input(g).cuda()
    with torch.no_grad():
        (features, proposals, level_index), losses, scores = model([x])
    assert losses == {} and len(proposals) == 1
    # (a) feature maps, norm-wise
    for i, f in enumerate(features):
        assert tuple(f.shape[1:]) == g[f"feat{i}"].shape and f.dtype == torch.float32
        ref = torch.from_numpy(g[f"feat{i}"].astype(np.float32)).cuda()
        rel = ((f[0] - ref).norm() / ref.norm()).item()
        print(f"{name}: feature P{i + 2} norm-wise rel err {rel:.3e}")
        assert rel < 2e-2
    plan = model.engine()._plans[next(iter(model.engine()._plans))]
    for i, p in enumerate(plan.pred):
        lg = p[0][..., :13].permute(3, 0, 1, 2).cpu()
        ref = torch.from_numpy(g[f"logits{i}"])
        rel = ((lg - ref).norm() / ref.norm()).item()
        print(f"{name}: logits level {i} norm-wise rel err {rel:.3e}")
        assert rel < 3e-2
    # (b) post-processing is bit-identical to the oracle on the engine's own head outputs
    ob, os_, ol = oracle_post_from_engine(plan, model.engine())
    assert proposals[0].shape[0] == ob.shape[0]
    np.testing.assert_array_equal(bits(proposals[0].cpu().numpy()), bits(ob))
    np.testing.assert_array_equal(bits(scores[0].cpu().numpy()), bits(os_))
    np.testing.assert_array_equal(level_index[0].cpu().numpy(), ol)
    # (c) proposals agree with the reference's (bf16 perturbs logits, so compare by overlap, not by index)
    refp, refs = g["proposals"], g["scores"]
    ours = proposals[0].cpu().numpy()
    top = np.argsort(-refs, kind="stable")[:100]
    iou = obox.iou_matrix(refp[top], ours) if ours.shape[0] else np.zeros((len(top), 0), np.float32)
    hit = (iou.max(axis=1) >= 0.7).mean() if ours.shape[0] else 0.0
    print(f"{name}: {ours.shape[0]} proposals (reference {refp.shape[0]}); top-100 reference proposals matched at IoU>=0.7: {hit:.2f}")
    assert hit >= 0.85
    assert abs(ours.shape[0] - refp.shape[0]) <= 0.15 * refp.shape[0] + 10


def test_batch_of_two_padded_scenes(golden_dir):
    """batch > 1 with different extents: zero padding to the batch max + -inf objectness in padded voxels
    (nerf_rpn.py:129-146, anchor.py:124-152, rpn.py:321-322); the post-processing must equal the oracle's."""
    g = np.load(os.path.join(golden_dir, "rpn_small_aabb.npz"))
    model, ag = build(False, g)
    x0 = recipes.golden_input(g).cuda()
    x1 = x0[:, :24, :40, :32].contiguous()
    with torch.no_grad():
        (features, proposals, level_index), _, scores = model([x0, x1])
    eng = model.engine()
    plan = [p for k, p in eng._plans.items() if k[0] == 2][0]
    code = eng.code
    for i, valid in enumerate([(32, 48, 40), (24, 40, 32)]):
        logits = [p[i].reshape(-1, 128)[:, :13].reshape(-1).cpu().numpy() for p in plan.pred]
        deltas = [p[i].reshape(-1, 128)[:, 13:13 + 13 * code].reshape(-1, code).cpu().numpy() for p in plan.pred]
        ob, os_, ol = rp.rpn_proposals(logits, deltas, plan.feat_dims, plan.strides, eng.cells, plan.dims, False,
                                       eng.pre_n, eng.post_n, eng.nms_thresh, eng.score_thresh, valid=valid)
        np.testing.assert_array_equal(bits(proposals[i].cpu().numpy()), bits(ob))
        np.testing.assert_array_equal(bits(scores[i].cpu().numpy()), bits(os_))


def test_full_size_scene_runs_and_matches_oracle_post():
    """BASELINE config 2 size: 160x256x256x4 grid, ResNet50-FPN + anchor head, random-init (seed 0) weights."""
    from nerf_rpn_b200.model.nerf_rpn import NeRFRegionProposalNetwork
    ns = _ns()
    torch.manual_seed(0)
    backbone = ns.ResNet_FPN_256(ns.Bottleneck, [3, 4, 6, 3], input_dim=4, is_max_pool=True)
    ag = ns.AnchorGenerator3D(recipes.ANCHOR_SIZES, recipes.ASPECT)
    head = ns.RPNHead(256, 13, 4, rotate=False)
    model = NeRFRegionProposalNetwork(backbone, ag, head, rpn_pre_nms_top_n_test=2500, rpn_post_nms_top_n_test=2500,
                                      rpn_nms_thresh=0.3, rpn_score_thresh=0.0).cuda().eval()
    gi = torch.Generator().manual_seed(1000)
    x = torch.rand(160, 256, 256, 4, generator=gi).permute(3, 0, 1, 2).contiguous().cuda()
    with torch.no_grad():
        (features, proposals, level_index), _, scores = model([x])
        (features2, proposals2, _), _, scores2 = model([x])            # graph replay is deterministic
    assert [tuple(f.shape) for f in features] == [(1, 256, 40, 64, 64), (1, 256, 20, 32, 32), (1, 256, 10, 16, 16), (1, 256, 5, 8, 8)]
    assert all(torch.isfinite(f).all() for f in features)
    assert torch.equal(proposals[0], proposals2[0]) and torch.equal(scores[0], scores2[0])
    eng = model.engine()
    plan = eng._plans[next(iter(eng._plans))]
    ob, os_, ol = oracle_post_from_engine(plan, eng)
    np.testing.assert_array_equal(bits(proposals[0].cpu().numpy()), bits(ob))
    np.testing.assert_array_equal(bits(scores[0].cpu().numpy()), bits(os_))
    s = scores[0].cpu().numpy()
    assert s.shape[0] > 0 and np.all(s[:-1] >= s[1:])
    print(f"full-size: {s.shape[0]} proposals, {plan.algorithmic_flops / 1e12:.3f} TFLOP/scene algorithmic")
    assert abs(plan.algorithmic_flops / 1e12 - 3.913) < 0.05           # SURVEY.md section 8(d)


@pytest.mark.parametrize("precision", ["bf16", "fp16", "fp16_w2"])
def test_config1_vgg19_fpn_small_grid(golden_dir, precision):
    """BASELINE config 1: single 32x32x32 grid, VGG19 ("EF") + FPN backbone, anchor head -- against the reference's golden
    outputs (the reference ran this exact configuration on CPU, tools/make_golden.py)."""
    from nerf_rpn_b200.model.nerf_rpn import NeRFRegionProposalNetwork
    g = np.load(os.path.join(golden_dir, "vgg_small_aabb.npz"))
    backbone, ag, head = recipes.build_vgg_small(_ns(), g)
    model = NeRFRegionProposalNetwork(backbone, ag, head, rpn_pre_nms_top_n_test=2500, rpn_post_nms_top_n_test=2500,
                                      rpn_nms_thresh=0.3, rpn_score_thresh=0.0).cuda().eval()
    model.precision = precision
    backbone.precision = precision
    x = recipes.golden_input(g).cuda()
    with torch.no_grad():
        (features, proposals, level_index), _, scores = model([x])
        standalone = backbone(x[None])                                   # the backbone module is also callable on its own
    assert [tuple(f.shape) for f in features] == [(1, 256, 32, 32, 32), (1, 256, 16, 16, 16), (1, 256, 8, 8, 8), (1, 256, 4, 4, 4)]
    for i, f in enumerate(features):
        st = int(g["fstride"][i])
        ref = torch.from_numpy(g[f"feat{i}"].astype(np.float32)).cuda()
        rel = ((f[0][:, ::st, ::st, ::st] - ref).norm() / ref.norm()).item()
        print(f"vgg config 1 [{precision}]: feature level {i} norm-wise rel err {rel:.3e}")
        assert rel < {"bf16": 2e-2, "fp16": 2e-3, "fp16_w2": 1e-3}[precision]
        assert torch.equal(standalone[i], f)
    eng = model.engine()
    plan = eng._plans[next(iter(eng._plans))]
    for i, p in enumerate(plan.pred):
        st = int(g["lstride"][i])
        lg = p[0][..., :13].permute(3, 0, 1, 2)[:, ::st, ::st, ::st].cpu()
        ref = torch.from_numpy(g[f"logits{i}"])
        rel = ((lg - ref).norm() / ref.norm()).item()
        print(f"vgg config 1: logits level {i} norm-wise rel err {rel:.3e}")
        assert rel < 3e-2
    ob, os_, ol = oracle_post_from_engine(plan, eng)
    np.testing.assert_array_equal(bits(proposals[0].cpu().numpy()), bits(ob))
    refp, refs = g["proposals"], g["scores"]
    ours = proposals[0].cpu().numpy()
    top = np.argsort(-refs, kind="stable")[:50]
    hit = (obox.iou_matrix(refp[top], ours).max(axis=1) >= 0.7).mean()
    print(f"vgg config 1: {ours.shape[0]} proposals (reference {refp.shape[0]}); top-50 matched at IoU>=0.7: {hit:.2f}")
    # The 32^3 random-init scene has near-tied objectness (top-10 reference scores are 1e-3 apart), so bf16 rounding flips which
    # box of an overlapping cluster wins NMS.  A displaced reference winner must still be covered by the box that suppressed it
    # (IoU > nms_thresh = 0.3); the IoU >= 0.7 rate is reported and loosely bounded.  Tight numerics live in the logits check above.
    cover = (obox.iou_matrix(refp[top], ours).max(axis=1) > 0.3).mean()
    print(f"vgg config 1: top-50 reference proposals covered at IoU>0.3 (NMS threshold): {cover:.2f}")
    assert cover >= 0.95 and hit >= 0.6


@pytest.mark.parametrize("name,rot", [("rpn_small_aabb", False), ("rpn_small_obb", True)])
def test_fp16_activation_mode_reaches_the_north_star_tolerance(golden_dir, name, rot):
    """precision='fp16' (IEEE half activations / weights, same tensor-core rate, fp32 accumulation): feature maps against the
    reference's fp32 golden. bf16 storage cannot get below ~7e-3 (8-bit significand); fp16 is expected around 1e-3."""
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    model, ag = build(rot, g)
    model.precision = "fp16"
    x = recipes.golden_input(g).cuda()
    with torch.no_grad():
        (features, proposals, level_index), losses, scores = model([x])
    rels = []
    for i, f in enumerate(features):
        ref = torch.from_numpy(g[f"feat{i}"].astype(np.float32)).cuda()      # golden features are stored as fp16 (5e-4 of their own)
        rels.append(((f[0] - ref).norm() / ref.norm()).item())
    plan = model.engine()._plans[next(iter(model.engine()._plans))]
    lrels = []
    for i, p in enumerate(plan.pred):
        lg = p[0][..., :13].permute(3, 0, 1, 2).cpu()
        ref = torch.from_numpy(g[f"logits{i}"])
        lrels.append(((lg - ref).norm() / ref.norm()).item())
    print(f"{name} fp16 mode: feature rel err {['%.2e' % r for r in rels]}, logits rel err {['%.2e' % r for r in lrels]}")
    assert max(rels) < 2e-3 and max(lrels) < 3e-3
    ob, os_, ol = oracle_post_from_engine(plan, model.engine())
    np.testing.assert_array_equal(bits(proposals[0].cpu().numpy()), bits(ob))
    refp, refs = g["proposals"], g["scores"]
    ours = proposals[0].cpu().numpy()
    top = np.argsort(-refs, kind="stable")[:100]
    hit = (obox.iou_matrix(refp[top], ours).max(axis=1) >= 0.7).mean()
    print(f"{name} fp16 mode: {ours.shape[0]} proposals (reference {refp.shape[0]}); top-100 matched at IoU>=0.7: {hit:.2f}")
    assert hit >= 0.9


def test_dataset_channels_last_view_is_consumed_in_place(golden_dir):
    """datasets.py:55-56 hands the model a (4,W,L,H) VIEW of the (W,L,H,4) array. The stem packing must read that memory order
    directly (bit-identical packed rows), and model / ScenePipeline results must not depend on the memory order."""
    from nerf_rpn_b200 import ops
    from nerf_rpn_b200.runtime import ScenePipeline
    g = np.load(os.path.join(golden_dir, "rpn_small_aabb.npz"))
    model, ag = build(False, g)
    wlhc = torch.from_numpy(g["grid"]).cuda()                              # (W,L,H,4) as on disk
    view = wlhc.permute(3, 0, 1, 2)                                        # what the dataset yields
    dense = view.contiguous()
    assert ops.is_channels_last_grid(view[None]) and not ops.is_channels_last_grid(dense[None])
    assert torch.equal(ops.pack_stem_input(view[None]), ops.pack_stem_input(dense[None]))
    odd = torch.rand((2, 21, 19, 27, 4), device="cuda").permute(0, 4, 1, 2, 3)          # odd extents, batch 2
    assert torch.equal(ops.pack_stem_input(odd), ops.pack_stem_input(odd.contiguous()))
    with torch.no_grad():
        (_, p_view, _), _, s_view = model([view])
        (_, p_dense, _), _, s_dense = model([dense])
    assert torch.equal(p_view[0], p_dense[0]) and torch.equal(s_view[0], s_dense[0])
    eng = model.engine()
    assert any(k[3] for k in eng._plans) and any(not k[3] for k in eng._plans)          # both plan kinds were built
    pipe = ScenePipeline(model, tuple(dense.shape[1:]), batch=1)
    host_view = wlhc.cpu().pin_memory().permute(3, 0, 1, 2)
    out = pipe.run([host_view, host_view])
    assert pipe.stage_channels_last
    for boxes, scores, levels in out:
        assert torch.equal(boxes, p_dense[0].cpu()) and torch.equal(scores, s_dense[0].cpu())


def test_raw_uint8_grid_is_normalised_on_the_device(golden_dir):
    """datasets.py:59-61: uint8 grids are normalised with .float() / 255.0 on the host. Handing the raw (4,W,L,H) uint8 view to the
    model must give exactly the result of the host-normalised fp32 grid (same correctly rounded x / 255), through model and pipeline."""
    from nerf_rpn_b200 import ops
    from nerf_rpn_b200.runtime import ScenePipeline
    g = np.load(os.path.join(golden_dir, "rpn_small_aabb.npz"))
    model, ag = build(False, g)
    gen = torch.Generator().manual_seed(77)
    raw = torch.randint(0, 256, (32, 48, 40, 4), generator=gen, dtype=torch.uint8)        # (W,L,H,4) as on disk
    view_u8 = raw.permute(3, 0, 1, 2)                                                       # what the dataset's transpose yields
    ref_f32 = view_u8.float() / 255.0                                                       # datasets.py:59-61
    assert torch.equal(ops.pack_stem_input(view_u8.cuda()[None]), ops.pack_stem_input(ref_f32.cuda()[None]))
    with torch.no_grad():
        (_, p_u8, _), _, s_u8 = model([view_u8.cuda()])
        (_, p_f, _), _, s_f = model([ref_f32.cuda()])
    assert torch.equal(p_u8[0], p_f[0]) and torch.equal(s_u8[0], s_f[0]) and p_u8[0].shape[0] > 0
    pipe = ScenePipeline(model, (32, 48, 40), batch=1)
    host = raw.pin_memory().permute(3, 0, 1, 2)
    out = pipe.run([host, host])
    assert pipe.stage_dtype == torch.uint8 and pipe.h2d_bytes_per_scene == 32 * 48 * 40 * 4
    for boxes, scores, levels in out:
        assert torch.equal(boxes, p_f[0].cpu()) and torch.equal(scores, s_f[0].cpu())
