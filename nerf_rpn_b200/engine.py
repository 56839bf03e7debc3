"""Inference engine: ResNet50-3D + FPN + anchor RPN head + proposal post-processing as a fixed list of
libnerf_rpn_b200 kernel launches over pre-allocated channels-last bf16 buffers, captured in a CUDA graph.

Mirrors, layer for layer, the reference forward
  NeRFRegionProposalNetwork.forward      nerf_rpn/model/nerf_rpn.py:166-217
  ResNet_FPN_256.forward / Bottleneck    nerf_rpn/model/feature_extractor.py:31-68,215-235
  RPNHead.forward                        nerf_rpn/model/anchor.py:206-213
  RegionProposalNetwork.forward (eval)   nerf_rpn/model/rpn.py:458-536
but: BatchNorm (eval) is folded into the conv weights, ReLU / residual / FPN nearest-upsample-add are conv
epilogues, the head runs all four pyramid levels in one launch per layer, cls and bbox predictors are one GEMM,
only the top-k candidates are decoded, and NMS never leaves the device.

PyTorch's role here: owning device buffers, the stream and the CUDA graph object.  Training-mode forward
(BatchNorm batch statistics, losses) is not implemented in this round and raises.
"""
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import ops, packing
from .precision import resolve as _resolve_precision, split_weights, storage_dtype


class _Conv:
    """One pre-packed convolution (+ folded BN / bias, optional ReLU).  `precision` gives the 16-bit storage format and, with `role`,
    whether the weights are split into hi + lo planes (precision.split_weights).  Roles "stem" / "stem_s1" pack the 7^3 stem for
    the stride-2 space-to-depth / stride-1 row-packed input."""

    def __init__(self, weight, bias=None, bn=None, *, precision, role="backbone", stride=1, relu=False, cout_pad_to=None, device="cuda"):
        scale = shift = None
        if bn is not None:
            scale, shift = (t.cpu() for t in packing.fold_bn(bn))
            if bias is not None:
                shift = shift + bias.detach().float().cpu() * scale
        elif bias is not None:
            shift = bias.detach().float().cpu()
        cout = weight.shape[0]
        weight = weight.detach().float().cpu()          # packing is host-side work (once per checkpoint), not GPU launches
        if scale is not None:
            scale = scale.cpu()
        if shift is not None:
            shift = shift.cpu()
        dtype = storage_dtype(precision)
        if role == "stem_s1":
            wp, taps = packing.pack_stem_s1_weight(weight, scale, dtype=dtype)
        elif role == "stem":
            wp, taps = packing.pack_stem_weight(weight, scale, dtype=dtype)
        else:
            wp, taps = packing.pack_conv_weight(weight, scale, cout_pad_to=cout_pad_to, dtype=dtype,
                                                split=split_weights(precision, role, weight, stride))
        self.w = wp.to(device)
        self.taps = taps
        self.cin = wp.shape[-1]
        self.cout = ((cout + 7) // 8) * 8 if cout_pad_to is None else cout_pad_to
        if shift is None:
            shift = torch.zeros(cout)
        self.shift = packing.pad_shift(shift, wp.shape[-2]).to(device)
        self.stride, self.relu = stride, relu


def _down(d: Sequence[int]) -> Tuple[int, int, int]:
    return tuple((v - 1) // 2 + 1 for v in d)


def _f32(t, device):
    return t.detach().float().to(device).contiguous()


# ---------------------------------------------------------------- packers: one per module kind, shared by the engine and model/_eager.py
def pack_stem(conv, bn, precision, device):
    """7^3 stem conv + BN + ReLU of ResNet_FPN_256 / VGG_FPN: stride 2 on the space-to-depth packed input, or stride 1 (VGG_FPN
    below 160) on the row-packed input."""
    return _Conv(conv.weight, conv.bias, bn, precision=precision, role="stem" if conv.stride[0] == 2 else "stem_s1", relu=True,
                 device=device)


def pack_bottleneck(blk, precision, device):
    """Bottleneck (feature_extractor.py:31-68) with its BatchNorms folded."""
    def conv(c, bn, stride=1, relu=True):
        return _Conv(c.weight, None, bn, precision=precision, stride=stride, relu=relu, device=device)
    s = blk.stride
    return {"c1": conv(blk.conv1, blk.bn1, s), "c2": conv(blk.conv2, blk.bn2),
            "c3": conv(blk.conv3, blk.bn3),                                           # ReLU after the residual add
            "ds": None if blk.downsample is None else conv(blk.downsample[0], blk.downsample[1], s, relu=False), "stride": s}


def pack_fpn(laterals, outs, p2, precision, device):
    """FPN neck: (1^3 lateral convs, 3^3 output convs); outs[p2] is the P2 output conv."""
    return ([_Conv(m.weight, m.bias, precision=precision, device=device) for m in laterals],
            [_Conv(m.weight, m.bias, precision=precision, role="p2" if i == p2 else "backbone", device=device) for i, m in enumerate(outs)])


def pack_rpn_head(hd, precision, device):
    """RPNHead (anchor.py:177-213): the 3^3 conv + ReLU stack, and the cls (A) and bbox (A*code) predictors fused into one 1^3 GEMM
    zero-padded to 128 output channels."""
    w = torch.cat([hd.cls_logits.weight, hd.bbox_pred.weight], 0)
    b = torch.cat([hd.cls_logits.bias, hd.bbox_pred.bias], 0)
    if w.shape[0] > 128:
        raise ValueError("fused predictor supports at most 128 output channels")
    return {"head": [_Conv(m.weight, m.bias, precision=precision, role="head", relu=True, device=device)
                     for m in hd.conv if isinstance(m, torch.nn.Conv3d)],
            "pred": _Conv(w, b, precision=precision, role="head", cout_pad_to=128, device=device)}


def pack_fcos_head(hd, precision, device):
    """FCOSHead (fcos/fcos.py:43-102): two towers of num_convs x [Conv3d 3^3 + GroupNorm(32) + ReLU] shared over levels, 3^3 predictors
    for class (1) and distances (6|8) | centerness (1, from the bbox tower), one Scale per level."""
    def conv(w, b):
        return _Conv(w, b, precision=precision, role="head", device=device)

    def tower(seq):
        mods = list(seq.children())
        return [(conv(c.weight, c.bias), _f32(gn.weight, device), _f32(gn.bias, device), float(gn.eps)) for c, gn in zip(mods[0::3], mods[1::3])]
    return {"cls_tower": tower(hd.cls_tower), "bbox_tower": tower(hd.bbox_tower), "cls_pred": conv(hd.cls_logits.weight, hd.cls_logits.bias),
            "reg_pred": conv(torch.cat([hd.bbox_pred.weight, hd.centerness.weight], 0), torch.cat([hd.bbox_pred.bias, hd.centerness.bias], 0)),
            "scales": [float(s.scale.detach().item()) for s in hd.scales]}


# ---------------------------------------------------------------- layer orders shared by the plan and model/_eager.py
# conv(layer, xs, ys, in_dims, out_dims, res=, res_dims=, name=) issues one launch; buf(dims, channels) allocates an activation.
def bottleneck_launches(conv, buf, e, x, xd, name):
    """Bottleneck.forward (feature_extractor.py:48-68) on the layers pack_bottleneck made: c1, c2, [ds], c3 + residual.
    Returns (output, dims)."""
    od = _down(xd) if e["stride"] == 2 else xd
    a = buf(od, e["c1"].cout)
    conv(e["c1"], [x], [a], [xd], [od], name=f"{name}.c1")
    b = buf(od, e["c2"].cout)
    conv(e["c2"], [a], [b], [od], [od], name=f"{name}.c2")
    r = x
    if e["ds"] is not None:
        r = buf(od, e["ds"].cout)
        conv(e["ds"], [x], [r], [xd], [od], name=f"{name}.ds")
    o = buf(od, e["c3"].cout)
    conv(e["c3"], [b], [o], [od], [od], res=[r], res_dims=[od], name=f"{name}.c3+res")
    return o, od


def fpn_launches(conv, buf, lat, out, xs):
    """FPN.forward (fpn.py:134-161) on the layers pack_fpn made: laterals top-down, each adding the nearest-upsampled level above in
    its epilogue (the reference's in-place accumulation), then a 3^3 conv on every level.  xs, and the result: [(tensor, dims)] from P2 up."""
    top = len(xs) - 1
    q = [None] * len(xs)
    for i in range(top, -1, -1):
        f, fd = xs[i]
        y = buf(fd, lat[i].cout)
        if i == top:
            conv(lat[i], [f], [y], [fd], [fd], name=f"fpn.lateral{i}")
        else:
            conv(lat[i], [f], [y], [fd], [fd], res=[q[i + 1][0]], res_dims=[q[i + 1][1]], name=f"fpn.lateral{i}+up")
        q[i] = (y, fd)
    feats = []
    for i, (y, yd) in enumerate(q):
        o = buf(yd, out[i].cout)
        conv(out[i], [y], [o], [yd], [yd], name=f"fpn.conv{i}")
        feats.append((o, yd))
    return feats


class RPNInferenceEngine:
    """Executes backbone -> FPN -> head -> proposals for a batch of equally sized scenes."""

    def __init__(self, backbone, head=None, anchor_cells=None, num_anchors: int = 0, rotated: bool = False,
                 pre_nms_top_n: int = 2500, post_nms_top_n: int = 2500, nms_thresh: float = 0.3, score_thresh: float = 0.0,
                 min_size: float = 1e-3, use_graph: bool = True, fcos: Optional[dict] = None, precision: Optional[str] = None,
                 density_to_alpha: bool = False):
        precision = _resolve_precision(precision)            # "bf16" | "fp16" | "fp16_w2" (nerf_rpn_b200/precision.py)
        self.precision = precision
        self.act_dtype = storage_dtype(precision)
        # datasets.py:50-52 (--normalize_density) applied by the stem packing kernel instead of numpy on the host (ResNet / VGG strided stems)
        self.density_to_alpha = bool(density_to_alpha)
        self.backbone, self.head = backbone, head
        self.fcos = fcos                   # None: anchor head (anchor.py:177-213); dict: FCOS head + post-processing settings
        self.cells = anchor_cells          # list (levels) of (A, 6) float arrays
        self.A, self.rotated = num_anchors, rotated
        self.code = 8 if rotated else 6
        self.pre_n, self.post_n = pre_nms_top_n, post_nms_top_n
        self.nms_thresh, self.score_thresh, self.min_size = nms_thresh, score_thresh, min_size
        self.use_graph = use_graph
        self._packed_version = None
        self._plans: Dict[tuple, "_Plan"] = {}
        self.layers = None

    # ---------------------------------------------------------------- weights
    def _param_version(self):
        """(storage, version) of every parameter / buffer: any in-place update, load_state_dict or re-materialisation changes it
        (a tuple, not a sum: nothing can cancel)."""
        out = []
        for m in (self.backbone, self.head):
            if m is not None:
                out.extend((t.data_ptr(), t._version) for t in m.parameters())
                out.extend((t.data_ptr(), t._version) for t in m.buffers())
        return tuple(out)

    def invalidate(self):
        """Force re-packing of the weights (and re-capture of the graphs) at the next forward."""
        self._packed_version = None

    def _pack(self, device):
        bb, hd = self.backbone, self.head
        kinds = {"ResNet_FPN_256": "resnet", "VGG_FPN": "vgg", "SwinTransformer_FPN": "swin"}
        if type(bb).__name__ not in kinds:
            raise NotImplementedError(f"nerf_rpn_b200: backbone {type(bb).__name__} is not implemented by the CUDA engine "
                                      "(ResNet_FPN_256, VGG_FPN, SwinTransformer_FPN are)")
        self.kind = kinds[type(bb).__name__]
        if self.kind == "resnet":          # the layer plan below is the configuration run_rpn.py:276 builds; anything else would run silently wrong
            c1 = getattr(bb, "conv1", None)
            ok = (getattr(bb, "is_max_pool", False) and c1 is not None and tuple(c1.kernel_size) == (7, 7, 7) and tuple(c1.stride) == (2, 2, 2)
                  and c1.in_channels == 4 and c1.out_channels == 64 and [len(s) for s in bb.layers] == [3, 4, 6, 3]
                  and all(type(b).__name__ == "Bottleneck" for s in bb.layers for b in s))
            if not ok:
                raise NotImplementedError("nerf_rpn_b200: the ResNet engine implements ResNet_FPN_256(Bottleneck, [3,4,6,3], input_dim=4, "
                                          "is_max_pool=True) (7^3 stride-2 stem on 4 channels + max-pool), the configuration run_rpn.py:276 builds")
        p = self.precision
        L = {"vgg": self._pack_vgg, "swin": self._pack_swin, "resnet": self._pack_resnet}[self.kind](device)
        if self.kind != "resnet":
            L["lat"], L["fpn"] = pack_fpn(bb.fpn_neck.lateral_convs, bb.fpn_neck.fpn_convs, 0, p, device)
        if hd is not None:
            L.update(pack_rpn_head(hd, p, device) if self.fcos is None else pack_fcos_head(hd, p, device))
        self.layers = L
        self._plans.clear()

    def _pack_swin(self, device):
        """SwinTransformer_FPN (feature_extractor.py:689-789). Every Linear becomes a 1x1x1 conv of the wgmma kernel; widths
        that are not multiples of 64 (96 at stage 0) live in rows padded with zero channels."""
        bb = self.backbone
        ln = lambda m: (_f32(m.weight, device), _f32(m.bias, device), float(m.eps))
        lin = lambda m, act=0: _Conv(m.weight.reshape(m.weight.shape[0], -1, 1, 1, 1), m.bias, precision=self.precision, relu=act,
                                     device=device)
        stages = []
        for si, stage in enumerate(bb.stages):
            mods = list(stage.children())
            st = {"merge": None, "blocks": []}
            if si > 0:
                pm = mods[0]; mods = mods[1:]
                st["merge"] = dict(ln=ln(pm.norm), c_in=pm.dim, red=lin(pm.reduction))
            for blk in mods:
                a = blk.attn
                st["blocks"].append(dict(
                    C=a.qkv.weight.shape[1], heads=a.num_heads, shift=int(a.shift_size[0]), ln1=ln(blk.norm1), ln2=ln(blk.norm2),
                    qkv=lin(a.qkv), qkv_bias=_f32(a.qkv.bias, device), table=_f32(a.relative_position_bias_table, device),
                    proj=lin(a.proj), mlp0=lin(blk.mlp[0], 2), mlp3=lin(blk.mlp[3])))
            stages.append(st)
        return {"pe": lin(bb.patch_partition[0]), "pe_ln": ln(bb.patch_partition[2]), "swin_stages": stages}

    def _pack_resnet(self, device):
        bb, p = self.backbone, self.precision
        lat, smooth = pack_fpn(bb.latlayers, bb.smooths, len(bb.smooths) - 1, p, device)          # the last smooth conv makes P2
        return {"stem": pack_stem(bb.conv1, bb.bn1, p, device), "blocks": [pack_bottleneck(b, p, device) for s in bb.layers for b in s],
                "lat": lat, "smooth": smooth}

    def _pack_vgg(self, device):
        """VGG_FPN (feature_extractor.py:289-377): stem [conv7 (s2 + max-pool when input_size >= 160, else s1), BN, ReLU], then
        four stages of (Conv3d 3^3 + BN + ReLU)* [+ MaxPool3d(2,2,ceil)] and the mmdet-style FPN neck (fpn.py:105-161)."""
        mods = list(self.backbone.layers.children())
        stages = []
        for grp in mods[-4:]:
            seq, items = list(grp.children()), []
            for i, m in enumerate(seq):           # ReLU is fused into the conv epilogue
                if isinstance(m, torch.nn.Conv3d):
                    bn = seq[i + 1] if i + 1 < len(seq) and isinstance(seq[i + 1], torch.nn.BatchNorm3d) else None
                    items.append(("conv", _Conv(m.weight, m.bias, bn, precision=self.precision, relu=True, device=device)))
                elif isinstance(m, torch.nn.MaxPool3d):
                    items.append(("pool", None))
            stages.append(items)
        return {"vgg_strided": mods[0].stride[0] == 2, "stem": pack_stem(mods[0], mods[1], self.precision, device), "vgg_stages": stages}

    # ---------------------------------------------------------------- plan
    def _get_plan(self, n, dims, device, channels_last: bool = False, u8: bool = False):
        ver = self._param_version()
        if self.layers is None or ver != self._packed_version:
            self._pack(device)
            self._packed_version = ver
        # a grid handed over as the dataset's (4,W,L,H) VIEW of the on-disk (W,L,H,4) array is consumed in place by the
        # ResNet stem packing (128-bit loads); the other backbones take a copy into NCDHW first
        cl = bool(channels_last) and self.kind == "resnet" and max(dims) >= 0
        if self.density_to_alpha and (u8 or self.kind == "swin" or (self.kind == "vgg" and not self.layers.get("vgg_strided", False))):
            raise NotImplementedError("density_to_alpha on the device is fused into the fp32 stride-2 stem packing (ResNet_FPN_256, VGG_FPN at >= 160)")
        if u8 and not cl:
            raise NotImplementedError("raw uint8 grids are consumed by the ResNet stem packing only; normalise to fp32 for the other backbones")
        key = (n, tuple(dims), str(device), cl, bool(u8))
        p = self._plans.get(key)
        if p is None:
            p = _Plan(self, n, tuple(dims), device, cl, bool(u8))
            self._plans[key] = p
        return p

    def check_eval(self):
        if self.backbone.training or (self.head is not None and self.head.training):
            raise NotImplementedError(
                "nerf_rpn_b200: training-mode forward (BatchNorm batch statistics, RPN losses, gradients) is not "
                "implemented by the CUDA engine yet; call .eval() (inference) -- there is no PyTorch fallback")

    def forward_device(self, grids: torch.Tensor, valid_dims: Optional[Sequence[Sequence[int]]] = None):
        """grids: (N,4,X,Y,Z) fp32 CUDA.  Returns the plan whose output buffers hold the results (no host sync)."""
        self.check_eval()
        if not grids.is_cuda or grids.dtype not in (torch.float32, torch.uint8):
            raise RuntimeError("nerf_rpn_b200: input grids must be fp32 (or raw uint8, channels-last) CUDA tensors (no CPU path)")
        n, c, X, Y, Z = grids.shape
        u8 = grids.dtype == torch.uint8
        if u8 and not ops.is_channels_last_grid(grids):
            raise ValueError("nerf_rpn_b200: uint8 grids must be (4,W,L,H) views of the on-disk (W,L,H,4) arrays")
        plan = self._get_plan(n, (X, Y, Z), grids.device, channels_last=ops.is_channels_last_grid(grids), u8=u8)
        plan.run(grids, valid_dims)
        return plan

    def flops_per_scene(self, dims) -> float:
        """Algorithmic conv FLOPs (2*MAC on the reference's real filter taps / channels) for one scene."""
        p = self._get_plan(1, tuple(dims), torch.device("cuda"))
        return p.algorithmic_flops


class _Plan:
    def __init__(self, eng: RPNInferenceEngine, n: int, dims: Tuple[int, int, int], device, channels_last: bool = False,
                 u8: bool = False):
        self.eng, self.n, self.dims, self.device = eng, n, dims, device
        self.channels_last = channels_last
        self.input_u8 = u8
        L = eng.layers
        bf = dict(dtype=eng.act_dtype, device=device)
        X, Y, Z = dims
        self._rpn_ws = None
        self._valid = None
        self._graph = None
        self._post = []
        self.names = {}              # id(callable) -> (layer name, algorithmic flops of the launch)
        self.launches = []           # backbone stage: list of zero-arg callables
        self.head_launches = []      # head stage
        self._cur = self.launches
        self.algorithmic_flops = 0.0

        def buf(d, c, dtype=eng.act_dtype):
            return torch.empty((n, *d, c), dtype=dtype, device=device)

        def conv(layer: _Conv, xs, ys, in_dims, out_dims, res=None, res_dims=None, out_fp32=False, real=None, name="conv"):
            args = []
            for i in range(len(xs)):
                r = None if res is None else res[i]
                args.append(ops.ConvLevelArgs(xs[i], ys[i], n, in_dims[i], out_dims[i], ys[i].shape[-1], res=r,
                                              res_dims=None if r is None else res_dims[i], ldr=0 if r is None else r.shape[-1]))
            self._cur.append(lambda a=args, l=layer, f=out_fp32: ops.conv3d_fprop(
                a, l.w, l.shift, l.cin, l.cout, l.taps, stride=l.stride, relu=l.relu, out_fp32=f))
            fl = 0.0
            for od in out_dims:
                vox = n * od[0] * od[1] * od[2]
                rc, rt, rco = real if real else (layer.cin, len(layer.taps), layer.cout)
                fl += 2.0 * vox * rco * rc * rt
            self.algorithmic_flops += fl / n
            self.names[id(self._cur[-1])] = (f"{name} {layer.cin}->{layer.cout} taps={len(layer.taps)} s={layer.stride} "
                                             f"out={'+'.join('x'.join(map(str, d)) for d in out_dims)}", fl)

        if channels_last:            # memory (n,X,Y,Z,4), logical (n,4,X,Y,Z): same strides as the dataset's view, copies stay memcpys
            self.input = torch.empty((n, X, Y, Z, 4), dtype=torch.uint8 if u8 else torch.float32, device=device).permute(0, 4, 1, 2, 3)
        else:
            self.input = torch.empty((n, 4, X, Y, Z), dtype=torch.float32, device=device)
        self._src = self.input
        self._buf, self._conv = buf, conv
        feats = {"vgg": self._build_vgg, "swin": self._build_swin}.get(eng.kind, self._build_resnet)(L, n, dims, bf)
        self.features = [f for f, _ in feats]
        self.feat_dims = [d for _, d in feats]

        # head: all levels per launch
        self.has_head = eng.head is not None
        if not self.has_head:
            return
        self._cur = self.head_launches
        (self._build_anchor_head if eng.fcos is None else self._build_fcos_head)(L, n, buf, conv)
        # post-processing = ~45 tiny kernels per scene: high priority so that they slip into the SMs as conv CTAs retire instead of
        # queueing behind whole layers (the main stream depends on them two steps later through the double-buffered predictions)
        self.side = torch.cuda.Stream(device=self.device, priority=-1)
        self._ev_pred = [torch.cuda.Event() for _ in range(2)]
        self._ev_done = [torch.cuda.Event() for _ in range(2)]
        self._parity = 0
        self._build_post(None)

    def _launch(self, fn, name):
        """Appends a launch that is not a convolution (no algorithmic FLOPs) to the current stage."""
        self._cur.append(fn)
        self.names[id(fn)] = (name, 0.0)

    def _build_strided_stem(self, L, n, dims, bf):
        """Space-to-depth input packing, the 7^3 stride-2 stem and the 3^3 stride-2 max-pool (ResNet, VGG at >= 160)."""
        d1 = _down(dims)
        self.packed = torch.empty((n, d1[0], d1[1], d1[2] + 1, 64), **bf)
        self._launch(lambda: ops.pack_stem_input(self._src, self.packed, density_to_alpha=self.eng.density_to_alpha), "pack_stem_input")
        c1 = self._buf(d1, 64)
        self._conv(L["stem"], [self.packed], [c1], [(d1[0], d1[1], d1[2] + 1)], [d1], real=(4, 343, 64), name="stem7x7x7s2(s2d)")
        d2 = _down(d1)
        x = self._buf(d2, 64)
        self._launch(lambda: ops.maxpool3d_k3s2(c1, x), "maxpool3d_k3s2")
        return x, d2

    def _build_resnet(self, L, n, dims, bf):
        buf, conv = self._buf, self._conv
        x, xd = self._build_strided_stem(L, n, dims, bf)

        # bottom-up
        c_out = []
        blocks = iter(L["blocks"])
        for si, stage in enumerate(self.eng.backbone.layers):
            for _ in stage:
                x, xd = bottleneck_launches(conv, buf, next(blocks), x, xd, f"L{si}")
            c_out.append((x, xd))

        # top-down (feature_extractor.py:224-235): p5 = lat0(c5); p_i = up(p_{i+1}) + lat(c_i); smooth all but p5
        (c5, d5) = c_out[-1]
        p = buf(d5, 256)
        conv(L["lat"][0], [c5], [p], [d5], [d5], name="lat0")
        p_out = [(p, d5)]
        for i in range(1, len(L["lat"])):
            (c, cd) = c_out[-1 - i]
            q = buf(cd, 256)
            conv(L["lat"][i], [c], [q], [cd], [cd], res=[p_out[-1][0]], res_dims=[p_out[-1][1]], name=f"lat{i}+up")
            p_out.append((q, cd))
        feats = [p_out[0]]
        for i, sm in enumerate(L["smooth"]):
            (q, qd) = p_out[i + 1]
            sq = buf(qd, 256)
            conv(sm, [q], [sq], [qd], [qd], name=f"smooth{i}")
            feats.append((sq, qd))
        feats.reverse()                                   # [P2, P3, P4, P5]
        return feats

    def _build_vgg(self, L, n, dims, bf):
        """VGG_FPN.forward (feature_extractor.py:362-377) + FPN.forward (fpn.py:134-161)."""
        buf, conv = self._buf, self._conv
        X, Y, Z = dims
        if L["vgg_strided"]:
            x, xd = self._build_strided_stem(L, n, dims, bf)
        else:
            self.packed = torch.empty((n, X, Y + 1, Z, 64), **bf)
            self._launch(lambda: ops.pack_stem_input_s1(self._src, self.packed), "pack_stem_input_s1")
            xd = dims
            x = buf(xd, 64)
            conv(L["stem"], [self.packed], [x], [(X, Y + 1, Z)], [xd], real=(4, 343, 64), name="stem7x7x7s1(packed)")
        stage_out = []
        for si, items in enumerate(L["vgg_stages"]):
            for kind, layer in items:
                if kind == "conv":
                    y = buf(xd, layer.cout)
                    conv(layer, [x], [y], [xd], [xd], name=f"vgg{si}.conv3x3x3")
                    x = y
                else:
                    od = tuple((v + 1) // 2 for v in xd)
                    y = buf(od, x.shape[-1])
                    self._launch(lambda a=x, b=y: ops.maxpool3d_k2s2_ceil(a, b), "maxpool3d_k2s2_ceil")
                    x, xd = y, od
            stage_out.append((x, xd))
        return fpn_launches(conv, buf, L["lat"], L["fpn"], stage_out)

    def _build_swin(self, L, n, dims, bf):
        """SwinTransformer_FPN.forward (feature_extractor.py:781-789): patch embedding, 4 stages of [PatchMerging] + blocks
        (x + attn(LN x); x + MLP(LN x)), FPN neck. Token grids are (n, H, W, D, ld) with ld = C rounded up to 64."""
        device = self.device
        buf, conv, add = self._buf, self._conv, self._launch
        pad64 = lambda c: (c + 63) // 64 * 64
        zbuf = lambda d, c: torch.zeros((n, *d, c), dtype=self.eng.act_dtype, device=device)      # pad channels must stay zero
        X, Y, Z = dims
        td = (X // 4, Y // 4, Z // 4)
        self.packed = torch.empty((n, *td, 256), **bf)
        add(lambda: ops.patch_embed_pack(self._src, self.packed), "swin.patch_embed_pack")
        C = L["pe"].cout
        e = zbuf(td, pad64(C))
        conv(L["pe"], [self.packed], [e], [td], [td], name="swin.patch_embed(4x4x4 s4 as GEMM)")
        x = zbuf(td, pad64(C))
        g, b, eps = L["pe_ln"]
        add(lambda i=e, o=x, c=C, g=g, b=b, eps=eps: ops.layernorm(i, o, c, g, b, eps), "swin.patch_embed.ln")
        stage_out = []
        for si, st in enumerate(L["swin_stages"]):
            if st["merge"] is not None:
                m = st["merge"]
                od = tuple((v + 1) // 2 for v in td)
                gathered = torch.empty((n, *od, 8 * m["c_in"]), **bf)
                g, b, eps = m["ln"]
                add(lambda i=x, o=gathered, c=m["c_in"], g=g, b=b, eps=eps: ops.patch_merge_ln(i, o, c, g, b, eps), f"swin{si}.patch_merge.gather+ln")
                C = m["red"].cout
                x = zbuf(od, pad64(C))
                conv(m["red"], [gathered], [x], [od], [od], name=f"swin{si}.patch_merge.reduction")
                td = od
            Cp = pad64(C)
            t = zbuf(td, Cp)                                   # LayerNorm output (scratch, reused by every block of the stage)
            qkv = torch.empty((n, *td, 3 * C), **bf)
            att = zbuf(td, Cp)
            hid = torch.empty((n, *td, 4 * C), **bf)
            ring = [zbuf(td, Cp), zbuf(td, Cp), x]             # residual stream rotates through three buffers
            ri = 0
            for bi, blk in enumerate(st["blocks"]):
                g1, b1, e1 = blk["ln1"]; g2, b2, e2 = blk["ln2"]
                add(lambda i=x, o=t, c=C, g=g1, b=b1, eps=e1: ops.layernorm(i, o, c, g, b, eps), f"swin{si}.ln1")
                conv(blk["qkv"], [t], [qkv], [td], [td], name=f"swin{si}.qkv")
                add(lambda q=qkv, o=att, bb_=blk["qkv_bias"], tb=blk["table"], c=C, h=blk["heads"], s=blk["shift"]:
                    ops.window_attention(q, o, bb_, tb, c, h, s), f"swin{si}.window_attention(shift={blk['shift']})")
                x2 = ring[ri % 3]; ri += 1
                if x2 is x:
                    x2 = ring[ri % 3]; ri += 1
                conv(blk["proj"], [att], [x2], [td], [td], res=[x], res_dims=[td], name=f"swin{si}.proj+res")
                add(lambda i=x2, o=t, c=C, g=g2, b=b2, eps=e2: ops.layernorm(i, o, c, g, b, eps), f"swin{si}.ln2")
                conv(blk["mlp0"], [t], [hid], [td], [td], name=f"swin{si}.mlp.fc1+gelu")
                x3 = [r for r in ring if r is not x and r is not x2][0]
                conv(blk["mlp3"], [hid], [x3], [td], [td], res=[x2], res_dims=[td], name=f"swin{si}.mlp.fc2+res")
                x = x3
            # the stage output must survive the next stage's scratch: it is only read (by patch merging and the FPN lateral)
            stage_out.append((x, td))
        return fpn_launches(conv, buf, L["lat"], L["fpn"], stage_out)

    def _build_pred(self, launch):
        """Predictor launches into two output sets (parity), so that the post-processing of scene i, which runs on the side stream,
        overlaps the backbone of scene i+1 without a buffer hazard.  launch(par) issues the predictor convs that write set par."""
        self.pred_launch = []
        for par in range(2):
            self._cur = []
            launch(par)
            fs = self._cur
            self.pred_launch.append(fs[0] if len(fs) == 1 else lambda fs=fs: [g() for g in fs])
        for g in fs:
            self.algorithmic_flops -= self.names[id(g)][1] / self.n         # counted once per scene
        self._cur = self.head_launches

    def _build_anchor_head(self, L, n, buf, conv):
        eng, device = self.eng, self.device
        cur = self.features
        for layer in L["head"]:
            nxt = [buf(d, 256) for d in self.feat_dims]
            conv(layer, cur, nxt, self.feat_dims, self.feat_dims, name="head3x3x3")
            cur = nxt
        self.pred_sets = [[buf(d, 128, torch.float32) for d in self.feat_dims] for _ in range(2)]
        self._build_pred(lambda par: conv(L["pred"], cur, self.pred_sets[par], self.feat_dims, self.feat_dims, out_fp32=True,
                                          real=(256, 1, eng.A * (1 + eng.code)), name="pred(cls|bbox)"))
        # proposals
        self.strides = [tuple(self.dims[k] // d[k] for k in range(3)) for d in self.feat_dims]
        bd = 7 if eng.rotated else 6
        self._out = [dict(boxes=torch.zeros((n, eng.post_n, bd), dtype=torch.float32, device=device),
                          scores=torch.zeros((n, eng.post_n), dtype=torch.float32, device=device),
                          levels=torch.zeros((n, eng.post_n), dtype=torch.float32, device=device),
                          count=torch.zeros((n,), dtype=torch.int32, device=device)) for _ in range(2)]

    def _build_fcos_head(self, L, n, buf, conv):
        eng, device, dims = self.eng, self.device, self.dims
        f = eng.fcos
        self._gn_ws = torch.empty(max(1, ops.lib().nrpn_groupnorm_workspace_bytes(len(self.features), n)), dtype=torch.uint8, device=device)
        ends = {}
        for name in ("cls_tower", "bbox_tower"):
            cur = self.features
            for (layer, gamma, beta, eps) in L[name]:
                nxt = [buf(d, 256) for d in self.feat_dims]
                conv(layer, cur, nxt, self.feat_dims, self.feat_dims, name=f"fcos.{name}.conv3x3x3")
                self._launch(lambda t=nxt, g=gamma, b=beta, e=eps: ops.groupnorm_relu_(t, g, b, e, True, 32, self._gn_ws),
                             f"fcos.{name}.groupnorm+relu")
                cur = nxt
            ends[name] = cur
        code = 8 if f["use_obb"] else 6
        cls_c, reg_c = L["cls_pred"].cout, L["reg_pred"].cout
        self.pred_sets = [dict(cls=[buf(d, cls_c, torch.float32) for d in self.feat_dims],
                               reg=[buf(d, reg_c, torch.float32) for d in self.feat_dims]) for _ in range(2)]

        def pred(par):
            conv(L["cls_pred"], ends["cls_tower"], self.pred_sets[par]["cls"], self.feat_dims, self.feat_dims, out_fp32=True,
                 real=(256, 27, 1), name="fcos.cls_logits")
            conv(L["reg_pred"], ends["bbox_tower"], self.pred_sets[par]["reg"], self.feat_dims, self.feat_dims, out_fp32=True,
                 real=(256, 27, code + 1), name="fcos.bbox_pred|centerness")
        self._build_pred(pred)
        self.strides = list(f["fpn_strides"])[: len(self.feat_dims)]
        cap = ops.lib().nrpn_fcos_max_proposals(__import__("ctypes").byref(self._post_desc(0, 0, dims)))
        dim = 7 if f["use_obb"] else 6
        self._out = [dict(boxes=torch.zeros((n, cap, 1 + dim), dtype=torch.float32, device=device),
                          scores=torch.zeros((n, cap), dtype=torch.float32, device=device),
                          count=torch.zeros((n,), dtype=torch.int32, device=device)) for _ in range(2)]

    # results of the most recent run (valid once `done` has completed)
    @property
    def pred(self):
        return self.pred_sets[self._parity]

    @property
    def out_boxes(self):
        return self._out[self._parity]["boxes"]

    @property
    def out_scores(self):
        return self._out[self._parity]["scores"]

    @property
    def out_levels(self):
        return self._out[self._parity]["levels"]

    @property
    def out_count(self):
        return self._out[self._parity]["count"]

    @property
    def done(self):
        return self._ev_done[self._parity]

    def _post_desc(self, par, i, valid):
        """Post-processing descriptor of scene i's predictions in output set par; valid: the scene's own extent (None: the plan's)."""
        eng, L, f = self.eng, self.eng.layers, self.eng.fcos
        if f is None:
            return ops.make_rpn_desc([p[i].reshape(-1, 128) for p in self.pred_sets[par]], self.feat_dims, self.strides, eng.cells, eng.A,
                                     eng.rotated, eng.pre_n, eng.post_n, eng.nms_thresh, eng.score_thresh, eng.min_size, self.dims, valid=valid)
        cls_c, reg_c = L["cls_pred"].cout, L["reg_pred"].cout
        return ops.make_fcos_desc([p[i].reshape(-1, cls_c) for p in self.pred_sets[par]["cls"]],
                                  [p[i].reshape(-1, reg_c) for p in self.pred_sets[par]["reg"]], self.feat_dims, self.strides,
                                  L["scales"], f["use_obb"], f["pre_nms_thresh"], f["pre_nms_top_n"], f["nms_thresh"],
                                  f["post_nms_top_n"], f["min_size"], valid or self.dims, padded=self.n > 1)

    def _build_post(self, valid_dims):
        """Per parity and scene, one post-processing chain (top-k, decode, NMS) writing that scene's rows of the output set."""
        import ctypes
        from ._lib import lib
        anchor = self.eng.fcos is None
        self._descs = [self._post_desc(par, i, None if valid_dims is None else valid_dims[i]) for par in range(2) for i in range(self.n)]
        ws_query = lib().nrpn_rpn_workspace_bytes if anchor else lib().nrpn_fcos_workspace_bytes
        ws_bytes = max(ws_query(ctypes.byref(d)) for d in self._descs)
        if self._rpn_ws is None or self._rpn_ws[0].numel() < ws_bytes or len(self._rpn_ws) != self.n:
            self._rpn_ws = [torch.empty(ws_bytes, dtype=torch.uint8, device=self.device) for _ in range(self.n)]
        run = ops.rpn_proposals if anchor else ops.fcos_proposals
        keys = ("boxes", "scores", "levels") if anchor else ("boxes", "scores")
        self._post = [[], []]
        for par in range(2):
            o = self._out[par]
            for i in range(self.n):
                out = tuple(o[k][i] for k in keys) + (o["count"][i:i + 1],)
                self._post[par].append(lambda d=self._descs[par * self.n + i], out=out, i=i:
                                       run(d, self.device, out=out, workspace=self._rpn_ws[i]))
        self._valid = valid_dims
        self._post_graph = [None, None]

    def _run_main_eager(self, skip_pack: bool = False):
        # launches[0] is always the kernel that consumes the fp32 input grid (stem packing / patch-embedding packing); it reads
        # self._src, the caller's tensor, so no staging copy of the 168 MB grid is needed.  The captured graph starts after it.
        for f in self.launches[1:] if skip_pack else self.launches:
            f()
        if self.has_head:
            for f in self.head_launches:
                f()

    def _run_post_eager(self, par):
        """Post-processing of every scene of the batch: independent chains of ~45 small kernels (top-k, decode, NMS), run one
        after the other on the current stream.  The chains are off the critical path already (high-priority side stream), and
        running them concurrently would only take SM slots from the convolutions."""
        for f in self._post[par]:
            f()

    def _run_eager(self):
        """Everything for one batch on the current stream (warm-up, launch counting, profiling)."""
        self._run_main_eager()
        if self.has_head:
            self.pred_launch[self._parity]()
            self._run_post_eager(self._parity)

    def run(self, grids: torch.Tensor, valid_dims=None):
        if valid_dims is not None and all(tuple(v) == tuple(self.dims) for v in valid_dims):
            valid_dims = None
        vd = None if valid_dims is None else tuple(tuple(v) for v in valid_dims)
        if self.has_head and vd != self._valid:
            torch.cuda.synchronize()
            self._build_post(vd)
        if self.channels_last != ops.is_channels_last_grid(grids) or (not self.channels_last and not grids.is_contiguous()):
            self.input.copy_(grids, non_blocking=True)      # foreign memory order: one conversion copy into the plan's own buffer
            grids = self.input
        self._src = grids
        use_graph = self.eng.use_graph
        if use_graph and self._graph is None:
            self._run_eager()                      # warm-up: cudaFuncSetAttribute, lazy init
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._run_main_eager(skip_pack=True)
            self._graph = g
        if use_graph:
            self.launches[0]()                     # input packing, eager: the only kernel whose source pointer changes per call
            self._graph.replay()
        else:
            self._run_main_eager()
        if not self.has_head:
            return
        cur = torch.cuda.current_stream(self.device)
        par = self._parity ^ 1
        cur.wait_event(self._ev_done[par])          # the post-processing that used this buffer set two runs ago
        self.pred_launch[par]()
        self._ev_pred[par].record(cur)
        self.side.wait_event(self._ev_pred[par])
        with torch.cuda.stream(self.side):
            if use_graph:
                if self._post_graph[par] is None:
                    self._run_post_eager(par)
                    self.side.synchronize()
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g, stream=self.side):
                        self._run_post_eager(par)
                    self._post_graph[par] = g
                self._post_graph[par].replay()
            else:
                self._run_post_eager(par)
            self._ev_done[par].record(self.side)
        self._parity = par

    def num_launches(self) -> int:
        """Kernels per forward (conv / pack / pool launches + the post-processing pipeline), counted, not guessed."""
        from ._lib import lib
        before = lib().nrpn_launch_count()
        self._run_eager()
        return int(lib().nrpn_launch_count() - before)
