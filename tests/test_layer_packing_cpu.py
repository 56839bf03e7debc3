"""CPU: which weight format every packed layer of the engine gets (precision.py, DESIGN.md section 4), and that the stand-alone module
forwards (model/_eager.py) pack a module exactly as the engine does."""
import pytest
import torch

from nerf_rpn_b200.engine import RPNInferenceEngine, _Conv, pack_bottleneck, pack_fcos_head, pack_fpn, pack_rpn_head
from nerf_rpn_b200.model import feature_extractor as FE
from nerf_rpn_b200.model.anchor import RPNHead
from nerf_rpn_b200.model.fcos.fcos import FCOSOverNeRF
from tests import recipes

FCOS = dict(use_obb=True, pre_nms_thresh=0.0, pre_nms_top_n=100, nms_thresh=0.3, post_nms_top_n=100, min_size=0.0, fpn_strides=[4, 8, 16, 32])
HEAD_KEYS = ("head", "pred", "cls_tower", "bbox_tower", "cls_pred", "reg_pred")


def _model(name):
    torch.manual_seed(0)
    if name == "resnet_rpn":
        return FE.ResNet_FPN_256(FE.Bottleneck, [3, 4, 6, 3], input_dim=4, is_max_pool=True), RPNHead(256, 13, 4), None
    if name in ("vgg32_rpn", "vgg256_rpn"):
        return FE.VGG_FPN("EF", 4, True, 32 if name == "vgg32_rpn" else 256), RPNHead(256, 13, 4, rotate=True), None
    bb = FE.VGG_FPN("EF", 4, True, 256) if name == "vgg_fcos" else FE.SwinTransformer_FPN(**recipes.SWIN_S)
    m = FCOSOverNeRF(recipes.fcos_args(True), bb, [4, 8, 16, 32])
    return m.backbone, m.fcos_module.head, FCOS


# Under fp16_w2 these keep single fp16 weights: the stem, the 3^3 64 -> 64 layers (halo-slab kernel), the P2 output conv and every
# head layer.  The 1^3 64 -> 64 c1 of the first ResNet stage is split.
SINGLE = {
    "resnet_rpn": {"stem", "blocks[0].c2", "blocks[1].c2", "blocks[2].c2", "smooth[2]"},
    "vgg32_rpn": {"stem", "vgg_stages[0][0][1]", "vgg_stages[0][1][1]", "fpn[0]"},
    "vgg256_rpn": {"stem", "vgg_stages[0][0][1]", "vgg_stages[0][1][1]", "fpn[0]"},
    "vgg_fcos": {"stem", "vgg_stages[0][0][1]", "vgg_stages[0][1][1]", "fpn[0]"},
    "swin_fcos": {"fpn[0]"},
}
# backbone + laterals + the other output convs: ResNet 1 + 16 x 3 + 4 downsample + 4 + 3 convs; VGG "EF" 1 + 16 + 4 + 4; Swin-S patch
# embedding + 24 blocks x (qkv, proj, 2 MLP) + 3 patch-merging reductions + 4 + 4
SPLIT_COUNT = {"resnet_rpn": 60 - 5, "vgg32_rpn": 25 - 4, "vgg256_rpn": 25 - 4, "vgg_fcos": 25 - 4, "swin_fcos": 1 + 24 * 4 + 3 + 8 - 1}


def _convs(x, path=""):
    if isinstance(x, _Conv):
        yield path, x
    elif isinstance(x, dict):
        for k, v in x.items():
            yield from _convs(v, f"{path}.{k}" if path else k)
    elif isinstance(x, (list, tuple)):
        for i, v in enumerate(x):
            yield from _convs(v, f"{path}[{i}]")


def _assert_same(a, b):
    assert isinstance(b, type(a)) or isinstance(a, type(b))
    if isinstance(a, _Conv):
        for t, u in ((a.w, b.w), (a.shift, b.shift)):
            assert t.dtype == u.dtype and t.shape == u.shape and torch.equal(t, u)
        assert (a.taps, a.cin, a.cout, a.stride, a.relu) == (b.taps, b.cin, b.cout, b.stride, b.relu)
    elif isinstance(a, dict):
        assert a.keys() == b.keys()
        for k in a:
            _assert_same(a[k], b[k])
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b)
        for u, v in zip(a, b):
            _assert_same(u, v)
    elif isinstance(a, torch.Tensor):
        assert a.dtype == b.dtype and torch.equal(a, b)
    else:
        assert a == b


@pytest.fixture(scope="module", params=["resnet_rpn", "vgg32_rpn", "vgg256_rpn", "vgg_fcos", "swin_fcos"])
def model(request):
    return request.param, _model(request.param)


@pytest.mark.parametrize("precision", ["fp16_w2", "fp16", "bf16"])
def test_layer_weight_formats(model, precision):
    name, (bb, hd, fcos) = model
    eng = RPNInferenceEngine(bb.eval(), hd.eval(), num_anchors=13, fcos=fcos, precision=precision)
    eng._pack("cpu")
    convs = dict(_convs(eng.layers))
    dtype = torch.bfloat16 if precision == "bf16" else torch.float16
    assert all(c.w.dtype == dtype for c in convs.values())
    split = {p for p, c in convs.items() if c.w.dim() == 4}           # (taps, 2, CoutPad, Cin): hi + lo planes
    if precision != "fp16_w2":
        assert not split
        return
    head = {p for p in convs if p.split(".")[0].split("[")[0] in HEAD_KEYS}
    assert head and not head & split
    assert set(convs) - split - head == SINGLE[name]
    assert len(split) == SPLIT_COUNT[name]


@pytest.mark.parametrize("precision", ["fp16_w2", "bf16"])
def test_standalone_packers_match_engine(model, precision):
    name, (bb, hd, fcos) = model
    eng = RPNInferenceEngine(bb.eval(), hd.eval(), num_anchors=13, fcos=fcos, precision=precision)
    eng._pack("cpu")
    L = eng.layers
    if name == "resnet_rpn":
        blocks = [b for s in bb.layers for b in s]
        for i in (0, 3, 4):                                            # 64-wide, strided with downsample, plain
            _assert_same(pack_bottleneck(blocks[i], precision, "cpu"), L["blocks"][i])
    else:
        lat, out = pack_fpn(bb.fpn_neck.lateral_convs, bb.fpn_neck.fpn_convs, 0, precision, "cpu")
        _assert_same((lat, out), (L["lat"], L["fpn"]))
    head = pack_rpn_head(hd, precision, "cpu") if fcos is None else pack_fcos_head(hd, precision, "cpu")
    _assert_same(head, {k: L[k] for k in head})
