"""Stand-alone forward() of the sub-modules the reference exposes (SURVEY.md 8(b)): Bottleneck.forward (feature_extractor.py:48-68),
FPN.forward (fpn.py:134-161), RPNHead.forward (anchor.py:206-213), FCOSHead.forward (fcos/fcos.py:104-130).

Inside NeRFRegionProposalNetwork / FCOSOverNeRF these layers run as part of one captured launch sequence (engine.py).  A caller that
uses a sub-module on its own (the reference's detector.py does, a user script may) gets the same kernels, launched eagerly: NCDHW fp32
tensors in and out like the reference, channels-last 16-bit inside (the layout conversions are torch copies -- plumbing --; every
convolution / normalisation is a libnerf_rpn_b200 launch).  Eval-mode semantics (BatchNorm running statistics); in training mode
the whole-model training engine (nerf_rpn_b200/train.py) is the supported path and these functions raise.
"""
from typing import Sequence, Tuple

import torch

from .. import ops
from ..engine import _Conv, bottleneck_launches, fpn_launches, pack_bottleneck, pack_fcos_head, pack_fpn, pack_rpn_head
from ..precision import resolve as _resolve_precision, storage_dtype

_CACHE = {}


def _version(module) -> tuple:
    return tuple((t.data_ptr(), t._version) for t in list(module.parameters()) + list(module.buffers()))


def _packed(module, precision, build):
    """Pre-packed weights of `module`, rebuilt when any parameter / buffer changed (storage or version)."""
    key = (id(module), precision)
    ver = _version(module)
    hit = _CACHE.get(key)
    if hit is None or hit[0] != ver:
        hit = _CACHE[key] = (ver, build())
    return hit[1]


def _check(x: torch.Tensor, training: bool, what: str):
    if training:
        raise NotImplementedError(f"nerf_rpn_b200: {what}.forward in training mode is not a stand-alone path; train through "
                                  "NeRFRegionProposalNetwork (nerf_rpn_b200/train.py)")
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise RuntimeError(f"nerf_rpn_b200: {what}.forward needs CUDA tensors (no CPU path)")


def _to_cl(x: torch.Tensor, dtype) -> torch.Tensor:
    return x.permute(0, 2, 3, 4, 1).to(dtype).contiguous()          # (N,C,X,Y,Z) fp32 -> (N,X,Y,Z,C) 16-bit


def _from_cl(y: torch.Tensor, c: int = None) -> torch.Tensor:
    y = y if c is None else y[..., :c]
    return y.permute(0, 4, 1, 2, 3).float()                           # NCDHW view semantics (channels_last_3d strides) like the engine


def _launch(layer: _Conv, xs, ys, in_dims, out_dims, res=None, res_dims=None, out_fp32=False, name=None):
    """One launch over the levels in xs (shared weights) into ys, issued now: the `conv` callback of the engine's layer orders."""
    args = []
    for i, x in enumerate(xs):
        r = None if res is None else res[i]
        args.append(ops.ConvLevelArgs(x, ys[i], x.shape[0], in_dims[i], out_dims[i], ys[i].shape[-1], res=r,
                                      res_dims=None if r is None else res_dims[i], ldr=0 if r is None else r.shape[-1]))
    ops.conv3d_fprop(args, layer.w, layer.shift, layer.cin, layer.cout, layer.taps, stride=layer.stride, relu=layer.relu, out_fp32=out_fp32)


def _buf_like(x: torch.Tensor):
    return lambda d, c: torch.empty((x.shape[0], *d, c), dtype=x.dtype, device=x.device)


def _conv(layer: _Conv, xs: Sequence[torch.Tensor], out_dims, out_fp32=False):
    """One launch over the levels in xs (shared weights); returns the outputs (N, *out_dims[i], layer.cout)."""
    dt = torch.float32 if out_fp32 else xs[0].dtype
    ys = [torch.empty((xs[0].shape[0], *od, layer.cout), dtype=dt, device=xs[0].device) for od in out_dims]
    _launch(layer, xs, ys, [x.shape[1:4] for x in xs], out_dims, out_fp32=out_fp32)
    return ys


# ---------------------------------------------------------------------------------------------- Bottleneck
def bottleneck_forward(blk, x: torch.Tensor, precision=None) -> torch.Tensor:
    """feature_extractor.py:48-68: relu(bn3(conv3(relu(bn2(conv2(relu(bn1(conv1(x)))))))) + [downsample](x)), BatchNorm folded."""
    _check(x, blk.training, "Bottleneck")
    precision = _resolve_precision(precision)
    L = _packed(blk, precision, lambda: pack_bottleneck(blk, precision, x.device))
    xc = _to_cl(x, storage_dtype(precision))
    o, _ = bottleneck_launches(_launch, _buf_like(xc), L, xc, tuple(xc.shape[1:4]), "bottleneck")
    return _from_cl(o)


# ---------------------------------------------------------------------------------------------- FPN
def fpn_forward(fpn, inputs: Sequence[torch.Tensor], precision=None) -> Tuple[torch.Tensor, ...]:
    """fpn.py:134-161: laterals, in-place top-down nearest-upsample accumulation, one 3^3 conv per level."""
    assert len(inputs) == len(fpn.in_channels)
    _check(inputs[0], fpn.training, "FPN")
    precision = _resolve_precision(precision)
    lat, out = _packed(fpn, precision, lambda: pack_fpn(fpn.lateral_convs, fpn.fpn_convs, 0, precision, inputs[0].device))
    xs = [_to_cl(t, storage_dtype(precision)) for t in inputs]
    feats = fpn_launches(_launch, _buf_like(xs[0]), lat, out, [(x, tuple(x.shape[1:4])) for x in xs])
    return tuple(_from_cl(o) for o, _ in feats)


# ---------------------------------------------------------------------------------------------- RPNHead
def rpn_head_pred(head, feats: Sequence[torch.Tensor], precision=None):
    """The head's fused output: per level fp32 (N, w, l, h, 128) rows [A logits | A*code deltas | zero pad] -- the layout the
    post-processing kernel (nrpn_rpn_proposals) reads."""
    _check(feats[0], head.training, "RPNHead")
    precision = _resolve_precision(precision)
    L = _packed(head, precision, lambda: pack_rpn_head(head, precision, feats[0].device))
    cur = [_to_cl(t, storage_dtype(precision)) for t in feats]
    dims = [tuple(t.shape[1:4]) for t in cur]
    for layer in L["head"]:
        cur = _conv(layer, cur, dims)
    return _conv(L["pred"], cur, dims, out_fp32=True)


def rpn_head_forward(head, feats: Sequence[torch.Tensor], precision=None):
    """anchor.py:206-213: per level conv stack (shared weights, all levels per launch) -> (logits (N,A,w,l,h), bbox_reg (N,A*code,w,l,h))."""
    A = head.cls_logits.weight.shape[0]
    nb = head.bbox_pred.weight.shape[0]
    pred = rpn_head_pred(head, feats, precision)
    logits = [p[..., :A].permute(0, 4, 1, 2, 3).contiguous() for p in pred]
    bbox = [p[..., A:A + nb].permute(0, 4, 1, 2, 3).contiguous() for p in pred]
    return logits, bbox


# ---------------------------------------------------------------------------------------------- FCOSHead
def fcos_head_forward(head, feats: Sequence[torch.Tensor], precision=None):
    """fcos/fcos.py:104-130 (eval): towers of conv + GroupNorm(32) + ReLU shared over levels, 3^3 predictors, per-level Scale, ReLU on the
    first six regressors and x stride -> (logits, bbox_reg, centerness) lists of (N,C,w,l,h) fp32."""
    _check(feats[0], head.training, "FCOSHead")
    precision = _resolve_precision(precision)
    code = head.bbox_pred.weight.shape[0]
    L = _packed(head, precision, lambda: pack_fcos_head(head, precision, feats[0].device))
    x0 = [_to_cl(t, storage_dtype(precision)) for t in feats]
    dims = [tuple(t.shape[1:4]) for t in x0]
    ends = {}
    for name in ("cls_tower", "bbox_tower"):
        cur = x0
        for (layer, gamma, beta, eps) in L[name]:
            cur = _conv(layer, cur, dims)
            ops.groupnorm_relu_(cur, gamma, beta, eps, True, 32)
        ends[name] = cur
    cls = _conv(L["cls_pred"], ends["cls_tower"], dims, out_fp32=True)
    reg = _conv(L["reg_pred"], ends["bbox_tower"], dims, out_fp32=True)
    logits = [c[..., :1].permute(0, 4, 1, 2, 3).contiguous() for c in cls]
    bbox_reg, ctr = [], []
    for l, r in enumerate(reg):
        bp = r[..., :code].permute(0, 4, 1, 2, 3).contiguous() * L["scales"][l]
        bp[:, :6] = torch.relu(bp[:, :6]) * head.fpn_strides[l]
        bbox_reg.append(bp)
        ctr.append(r[..., code:code + 1].permute(0, 4, 1, 2, 3).contiguous())
    return logits, bbox_reg, ctr
