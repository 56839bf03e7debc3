"""GPU tests for the Swin-3D path: LayerNorm / patch-merge / patch-embed / window-attention kernels against plain PyTorch
fp32, GELU epilogue, and SwinTransformer_FPN + FCOS end to end against the reference's golden outputs (config 3, small)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import box as obox
from oracle import fcos_post as fp
from oracle import net as onet
from tests import recipes

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def test_layernorm_and_patch_merge_kernels():
    from nerf_rpn_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(1)
    for C, ld in ((96, 128), (192, 192), (768, 768)):
        x = torch.zeros((2, 5, 7, 3, ld), device="cuda", dtype=torch.bfloat16)
        x[..., :C] = (torch.randn((2, 5, 7, 3, C), device="cuda", generator=g) * 2 + 0.3).to(torch.bfloat16)
        gamma = torch.rand(C, device="cuda", generator=g) + 0.5; beta = torch.randn(C, device="cuda", generator=g)
        out = torch.zeros_like(x)
        ops.layernorm(x, out, C, gamma, beta, 1e-5)
        ref = F.layer_norm(x[..., :C].float(), (C,), gamma, beta, 1e-5)
        assert (out[..., :C].float() - ref).abs().max().item() < 1e-2 * max(1.0, ref.abs().max().item()) + 1e-2, 'layernorm'
        assert ld == C or out[..., C:].abs().max().item() == 0, 'pad channels must stay zero'
        gamma8 = torch.rand(8 * C, device="cuda", generator=g) + 0.5; beta8 = torch.randn(8 * C, device="cuda", generator=g)
        merged = torch.empty((2, 3, 4, 2, 8 * C), device="cuda", dtype=torch.bfloat16)
        ops.patch_merge_ln(x, merged, C, gamma8, beta8, 1e-5)
        xp = F.pad(x[..., :C].float(), (0, 0, 0, 1, 0, 1, 0, 1))
        parts = [xp[:, i::2, j::2, k::2, :] for (i, j, k) in ((0, 0, 0), (1, 0, 0), (0, 1, 0), (1, 1, 0), (0, 0, 1), (1, 0, 1), (0, 1, 1), (1, 1, 1))]
        refm = F.layer_norm(torch.cat(parts, -1), (8 * C,), gamma8, beta8, 1e-5)
        assert (merged.float() - refm).abs().max().item() < 1e-2 * max(1.0, refm.abs().max().item()) + 1e-2, 'patch merge'


def test_patch_embed_pack_and_gelu_gemm():
    from nerf_rpn_b200 import ops, packing
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.rand((1, 4, 21, 18, 14), device="cuda", generator=g)
    w = torch.randn((96, 4, 4, 4, 4), device="cuda", generator=g) * 0.1
    bias = torch.randn(96, device="cuda", generator=g)
    packed = torch.empty((1, 5, 4, 3, 256), device="cuda", dtype=torch.bfloat16)
    ops.patch_embed_pack(x, packed)
    wp, taps = packing.pack_conv_weight(w.reshape(96, 256, 1, 1, 1).cpu()); wp = wp.cuda()
    shift = packing.pad_shift(bias, wp.shape[1])
    y = torch.zeros((1, 5, 4, 3, 128), device="cuda", dtype=torch.float32)
    ops.conv3d_fprop([ops.ConvLevelArgs(packed, y, 1, (5, 4, 3), (5, 4, 3), 128)], wp, shift, 256, 96, taps, relu=2, out_fp32=True)
    ref = F.gelu(F.conv3d(x.to(torch.bfloat16).float(), w.to(torch.bfloat16).float(), bias, stride=4)).permute(0, 2, 3, 4, 1)
    assert (y[..., :96] - ref).abs().max().item() < 2e-3 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("dims,heads,shift", [((8, 8, 8), 3, 0), ((8, 12, 8), 3, 2), ((10, 13, 8), 6, 2), ((3, 4, 2), 12, 2), ((5, 7, 4), 6, 0)])
def test_window_attention_kernel(dims, heads, shift):
    """Against oracle/net.py:_window_attention (bit-identical to the reference on CPU) with identity projection."""
    from nerf_rpn_b200 import ops
    C = heads * 32
    g = torch.Generator(device="cuda").manual_seed(4)
    qkv = (torch.randn((2, *dims, 3 * C), device="cuda", generator=g)).to(torch.bfloat16)
    qkv_bias = torch.randn(3 * C, device="cuda", generator=g) * 0.3
    table = torch.randn((343, heads), device="cuda", generator=g) * 0.5
    out = torch.zeros((2, *dims, C), device="cuda", dtype=torch.bfloat16)
    ops.window_attention(qkv, out, qkv_bias, table, C, heads, shift)
    # reference: feed x = identity-able input: build sd so that F.linear(x, W, b) reproduces the given qkv on real tokens and the
    # bias on padded ones: x = [qkv - bias | 1-hot? ] is not possible in general -> use W = I (3C x 3C) on an input of width 3C
    sd = {"a.qkv.weight": torch.eye(3 * C), "a.qkv.bias": qkv_bias.cpu(), "a.proj.weight": torch.eye(C), "a.proj.bias": torch.zeros(C),
          "a.relative_position_bias_table": table.cpu()}
    from nerf_rpn_b200.model.feature_extractor import ShiftedWindowAttention
    sd["a.relative_position_index"] = ShiftedWindowAttention(C, [4, 4, 4], [shift] * 3, heads).relative_position_index
    xin = qkv.float().cpu() - qkv_bias.cpu()                      # so that linear(xin) = qkv on real tokens, = bias on zero padding
    ref = _attn_ref_wide(xin, sd, heads, shift, C)
    err = (out.float().cpu() - ref).abs().max().item()
    assert err < 3e-2 * max(1.0, ref.abs().max().item()), f"max abs err {err}"


def test_window_attention_rejects_unaligned_rows():
    """Rows are moved in 16-byte chunks: an output row pitch that is not a multiple of 8 elements is an invalid argument, refused
    before anything is launched."""
    from nerf_rpn_b200 import ops
    heads, C = 3, 96
    qkv = torch.zeros((1, 4, 4, 4, 3 * C), device="cuda", dtype=torch.bfloat16)
    out = torch.zeros((1, 4, 4, 4, C + 4), device="cuda", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="invalid argument"):
        ops.window_attention(qkv, out, torch.zeros(3 * C, device="cuda"), torch.zeros((343, heads), device="cuda"), C, heads, 0)


def _attn_ref_wide(xin, sd, heads, shift, C):
    """_window_attention with a 3C-wide input and identity qkv weight (so arbitrary q/k/v can be injected)."""
    import torch
    B, H, W, D, C3 = xin.shape
    win = 4
    ph, pw, pd = (-H) % win, (-W) % win, (-D) % win
    xp = F.pad(xin, (0, 0, 0, pd, 0, pw, 0, ph))
    PH, PW, PD = H + ph, W + pw, D + pd
    sh = [0 if win >= e else shift for e in (PH, PW, PD)]
    if sum(sh) > 0:
        xp = torch.roll(xp, shifts=(-sh[0], -sh[1], -sh[2]), dims=(1, 2, 3))
    nh, nw, nd = PH // win, PW // win, PD // win
    t = xp.view(B, nh, win, nw, win, nd, win, C3).permute(0, 1, 3, 5, 2, 4, 6, 7).reshape(B * nh * nw * nd, 64, C3)
    qkv = (t + sd["a.qkv.bias"]).reshape(t.shape[0], 64, 3, heads, 32).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0] * 32 ** -0.5, qkv[1], qkv[2]
    attn = q @ k.transpose(-2, -1)
    bias = sd["a.relative_position_bias_table"][sd["a.relative_position_index"]].view(64, 64, -1).permute(2, 0, 1)
    attn = attn + bias.unsqueeze(0)
    if sum(sh) > 0:
        region = torch.zeros((PH, PW, PD)); cnt = 0
        for hs in ((0, -win), (-win, -sh[0]), (-sh[0], None)):
            for ws in ((0, -win), (-win, -sh[1]), (-sh[1], None)):
                for ds in ((0, -win), (-win, -sh[2]), (-sh[2], None)):
                    region[hs[0]:hs[1], ws[0]:ws[1], ds[0]:ds[1]] = cnt; cnt += 1
        region = region.view(nh, win, nw, win, nd, win).permute(0, 2, 4, 1, 3, 5).reshape(nh * nw * nd, 64)
        diff = region.unsqueeze(1) - region.unsqueeze(2)
        mask = torch.where(diff != 0, torch.full_like(diff, -100.0), torch.zeros_like(diff))
        attn = (attn.view(B, nh * nw * nd, heads, 64, 64) + mask.unsqueeze(1).unsqueeze(0)).view(-1, heads, 64, 64)
    o = (F.softmax(attn, dim=-1) @ v).transpose(1, 2).reshape(t.shape[0], 64, C)
    o = o.view(B, nh, nw, nd, win, win, win, C).permute(0, 1, 4, 2, 5, 3, 6, 7).reshape(B, PH, PW, PD, C)
    if sum(sh) > 0:
        o = torch.roll(o, shifts=(sh[0], sh[1], sh[2]), dims=(1, 2, 3))
    return o[:, :H, :W, :D, :].contiguous()


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
