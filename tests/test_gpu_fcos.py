"""GPU parity for the anchor-free (FCOS) path: device post-processing vs the oracle (bit-exact), FCOSOverNeRF end to end vs the
reference's golden outputs.  The GroupNorm kernel: tests/test_gpu_swin_gn_kernels.py."""
import os

import numpy as np
import pytest
import torch

from oracle import box as obox
from oracle import fcos_post as fp
from tests import recipes

pytestmark = pytest.mark.gpu

GRIDS = [(8, 12, 10), (4, 6, 5), (2, 3, 3), (1, 2, 2)]
STRIDES = [4, 8, 16, 32]


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


@pytest.mark.parametrize("obb,pre,post", [(False, 2500, 2500), (True, 2500, 2500), (False, 300, 150), (True, 300, 150)])
def test_fcos_postprocessing_bit_exact_vs_oracle(obb, pre, post):
    from nerf_rpn_b200 import ops
    code = 8 if obb else 6
    g = torch.Generator(device="cuda").manual_seed(5 + int(obb))
    grids = [(20, 24, 16), (10, 12, 8), (5, 6, 4), (3, 3, 2)]
    scales = [1.0, 1.1, 0.9, 1.3]
    cls, reg = [], []
    for gr in grids:
        v = gr[0] * gr[1] * gr[2]
        c = torch.zeros((v, 8), device="cuda"); c[:, 0] = torch.randn(v, device="cuda", generator=g) * 2 - 1
        r = torch.zeros((v, 16), device="cuda")
        r[:, :6] = torch.randn((v, 6), device="cuda", generator=g) * 1.5 + 1.0
        if obb:
            r[:, 6:8] = torch.randn((v, 2), device="cuda", generator=g) * 0.3
        r[:, code] = torch.randn(v, device="cuda", generator=g)
        c[::11, 0] = c[::7, 0][: c[::11, 0].numel()]                          # exact ties
        cls.append(c.contiguous()); reg.append(r.contiguous())
    mesh = (80, 96, 64)
    d = ops.make_fcos_desc(cls, reg, grids, STRIDES, scales, obb, 0.0, pre, 0.3, post, 0.0, mesh)
    boxes, scores, count = ops.fcos_proposals(d, torch.device("cuda"))
    k = int(count.item())
    ob, os_ = fp.fcos_proposals([c[:, 0].cpu().numpy() for c in cls], [r[:, :code].cpu().numpy() for r in reg],
                                [r[:, code].cpu().numpy() for r in reg], scales, grids, STRIDES, mesh, obb, 0.0, pre, 0.3, post, 0.0)
    assert k == ob.shape[0] and k > 50
    np.testing.assert_array_equal(bits(boxes[:k].cpu().numpy()), bits(ob))
    np.testing.assert_array_equal(bits(scores[:k].cpu().numpy()), bits(os_))


def _ns():
    from nerf_rpn_b200.model import feature_extractor
    from nerf_rpn_b200.model.fcos import fcos

    class NS:
        ResNet_FPN_256 = feature_extractor.ResNet_FPN_256
        Bottleneck = feature_extractor.Bottleneck
        FCOSOverNeRF = fcos.FCOSOverNeRF
    return NS


@pytest.mark.parametrize("name,obb,pre,post", [("fcos_small_aabb", False, 2500, 2500), ("fcos_small_obb", True, 2500, 2500),
                                               ("fcos_small_obb_tight", True, 300, 150)])
@pytest.mark.parametrize("precision", ["bf16", "fp16"])
def test_fcos_end_to_end_vs_reference_golden(golden_dir, name, obb, pre, post, precision):
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    model = recipes.build_fcos_small(_ns(), obb, g, pre, post).cuda().eval()
    model.precision = precision
    x = recipes.seed1000_input().cuda()
    with torch.no_grad():
        boxes, losses, scores = model([x])
    assert losses == {} and boxes[0].shape[1] == (8 if obb else 7)
    eng = model.engine()
    plan = eng._plans[next(iter(eng._plans))]
    code = 8 if obb else 6
    # (a) head outputs vs the reference (bf16 towers + GroupNorm): norm-wise
    for l in range(4):
        lg = plan.pred["cls"][l][0][..., 0].cpu()
        ref = torch.from_numpy(g[f"logits{l}"][0])
        rel = ((lg - ref).norm() / ref.norm()).item()
        print(f"{name} [{precision}]: cls logits level {l} norm-wise rel err {rel:.3e}")
        assert rel < (5e-2 if precision == "bf16" else 6e-3)
    # (b) post-processing bit-identical to the oracle on the engine's own head outputs
    L = eng.layers
    ob, os_ = fp.fcos_proposals([p[0].reshape(-1, p.shape[-1])[:, 0].cpu().numpy() for p in plan.pred["cls"]],
                                [p[0].reshape(-1, p.shape[-1])[:, :code].cpu().numpy() for p in plan.pred["reg"]],
                                [p[0].reshape(-1, p.shape[-1])[:, code].cpu().numpy() for p in plan.pred["reg"]],
                                L["scales"], GRIDS, STRIDES, (32, 48, 40), obb, 0.0, pre, 0.3, post, 0.0)
    np.testing.assert_array_equal(bits(boxes[0].cpu().numpy()), bits(ob))
    np.testing.assert_array_equal(bits(scores[0].cpu().numpy()), bits(os_))
    # (c) agreement with the reference's proposals by overlap
    refb, refs = g["boxes"][:, 1:], g["scores"]
    ours = boxes[0][:, 1:].cpu().numpy()
    top = np.argsort(-refs, kind="stable")[:100]
    hit = (obox.iou_matrix(refb[top], ours).max(axis=1) >= 0.7).mean()
    print(f"{name}: {ours.shape[0]} proposals (reference {refb.shape[0]}); top-100 matched at IoU>=0.7: {hit:.2f}")
    assert hit >= 0.8 and abs(ours.shape[0] - refb.shape[0]) <= 0.2 * refb.shape[0] + 10


@pytest.mark.parametrize("obb", [False, True])
def test_fcos_batch_of_two_padded_scenes(golden_dir, obb):
    """batch > 1 with different extents (fcos.py:252-266 compute_padding_masks): scenes are zero-padded to the batch maximum,
    locations outside a scene's own extent are masked, boxes are clipped to the scene's own size. Post-processing of every scene
    must equal the oracle's on the engine's head outputs."""
    name = "fcos_small_obb" if obb else "fcos_small_aabb"
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    model = recipes.build_fcos_small(_ns(), obb, g, 2500, 2500).cuda().eval()
    x0 = recipes.seed1000_input().cuda()
    x1 = x0[:, :24, :40, :32].contiguous()
    with torch.no_grad():
        boxes, losses, scores = model([x0, x1])
    assert len(boxes) == 2 and losses == {}
    eng = model.engine()
    plan = [p for k, p in eng._plans.items() if k[0] == 2][0]
    code = 8 if obb else 6
    L = eng.layers
    for i, own in enumerate([(32, 48, 40), (24, 40, 32)]):
        ob, os_ = fp.fcos_proposals([p[i].reshape(-1, p.shape[-1])[:, 0].cpu().numpy() for p in plan.pred["cls"]],
                                    [p[i].reshape(-1, p.shape[-1])[:, :code].cpu().numpy() for p in plan.pred["reg"]],
                                    [p[i].reshape(-1, p.shape[-1])[:, code].cpu().numpy() for p in plan.pred["reg"]],
                                    L["scales"], GRIDS, STRIDES, own, obb, 0.0, 2500, 0.3, 2500, 0.0, padded=True)
        np.testing.assert_array_equal(bits(boxes[i].cpu().numpy()), bits(ob))
        np.testing.assert_array_equal(bits(scores[i].cpu().numpy()), bits(os_))
    assert boxes[1].shape[0] > 0 and boxes[0].shape[0] != boxes[1].shape[0]
