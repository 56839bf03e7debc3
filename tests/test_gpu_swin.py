"""GPU tests for the Swin-3D path: the window-attention argument checks, and SwinTransformer_FPN + FCOS end to end against the
reference's golden outputs (config 3, small).  The kernels one by one: tests/test_gpu_swin_gn_kernels.py."""
import os

import numpy as np
import pytest
import torch

from oracle import box as obox
from oracle import fcos_post as fp
from tests import recipes

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def test_window_attention_rejects_unaligned_rows():
    """Rows are moved in 16-byte chunks: an output row pitch that is not a multiple of 8 elements is an invalid argument, refused
    before anything is launched."""
    from nerf_rpn_b200 import ops
    heads, C = 3, 96
    qkv = torch.zeros((1, 4, 4, 4, 3 * C), device="cuda", dtype=torch.bfloat16)
    out = torch.zeros((1, 4, 4, 4, C + 4), device="cuda", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="invalid argument"):
        ops.window_attention(qkv, out, torch.zeros(3 * C, device="cuda"), torch.zeros((343, heads), device="cuda"), C, heads, 0)


@pytest.mark.parametrize("precision", ["bf16", "fp16", "fp16_w2"])
def test_config3_swin_s_fcos_small(golden_dir, precision):
    """Swin-S + FPN + FCOS head (OBB) on a 40x52x34 grid vs the reference's golden feature maps / logits / boxes."""
    from nerf_rpn_b200.model import feature_extractor
    from nerf_rpn_b200.model.fcos import fcos as fcos_mod

    class NS:
        SwinTransformer_FPN = feature_extractor.SwinTransformer_FPN
        FCOSOverNeRF = fcos_mod.FCOSOverNeRF
    g = np.load(os.path.join(golden_dir, "swin_small_fcos_obb.npz"))
    model = recipes.build_swin_fcos_small(NS, g).cuda().eval()
    model.precision = precision
    model.backbone.precision = precision
    x = recipes.seed1000_input((40, 52, 34)).cuda()
    with torch.no_grad():
        boxes, _, scores = model([x])
        feats = model.backbone(x[None])
    for i, f in enumerate(feats):
        ref = torch.from_numpy(g[f"feat{i}"].astype(np.float32)).cuda()
        rel = ((f[0] - ref).norm() / ref.norm()).item()
        print(f"swin config 3 [{precision}]: feature level {i} norm-wise rel err {rel:.3e}")
        assert rel < {"bf16": 4e-2, "fp16": 4e-3, "fp16_w2": 2.5e-3}[precision]
    eng = model.engine()
    plan = eng._plans[next(iter(eng._plans))]
    grids = plan.feat_dims
    L = eng.layers
    ob, os_ = fp.fcos_proposals([p[0].reshape(-1, p.shape[-1])[:, 0].cpu().numpy() for p in plan.pred["cls"]],
                                [p[0].reshape(-1, p.shape[-1])[:, :8].cpu().numpy() for p in plan.pred["reg"]],
                                [p[0].reshape(-1, p.shape[-1])[:, 8].cpu().numpy() for p in plan.pred["reg"]],
                                L["scales"], grids, [4, 8, 16, 32], (40, 52, 34), True, 0.0, 2500, 0.3, 2500, 0.0)
    np.testing.assert_array_equal(bits(boxes[0].cpu().numpy()), bits(ob))
    refb, refs = g["boxes"][:, 1:], g["scores"]
    ours = boxes[0][:, 1:].cpu().numpy()
    top = np.argsort(-refs, kind="stable")[:100]
    hit = (obox.iou_matrix(refb[top], ours).max(axis=1) >= 0.7).mean()
    print(f"swin config 3 [{precision}]: {ours.shape[0]} proposals (reference {refb.shape[0]}); top-100 matched at IoU>=0.7: {hit:.2f}")
    assert hit >= 0.75
