"""Backbones. Mirrors nerf_rpn/model/feature_extractor.py for the hot path:
  Bottleneck        feature_extractor.py:31-68
  ResNet_FPN_256    feature_extractor.py:145-235   (ResNet50-3D + inline FPN; run_rpn.py:276)
The modules own ordinary nn.Conv3d / nn.BatchNorm3d parameters, created in the reference's order so that
torch.manual_seed(s) reproduces the reference's initial weights and state_dict keys are identical
(conv1.weight, bn1.*, layers.{s}.{b}.conv{1,2,3}.weight, ..., smooths.{i}.*, latlayers.{i}.*; SURVEY.md section 5).
forward() never calls those nn modules: it runs the pre-packed wgmma engine (nerf_rpn_b200/engine.py).
VGG_FPN (config 1) and SwinTransformer_FPN (config 3) follow below on the same engine.
"""
from typing import List

import torch
from torch import nn

from ..precision import EngineHolder, resolve as _resolve_precision


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv3d(inplanes, planes, kernel_size=1, stride=stride, bias=False)   # stride sits on the 1^3 conv
        self.bn1 = nn.BatchNorm3d(planes)
        self.conv2 = nn.Conv3d(planes, planes, kernel_size=3, stride=1, padding=1, bias=False)
        self.bn2 = nn.BatchNorm3d(planes)
        self.conv3 = nn.Conv3d(planes, planes * self.expansion, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm3d(planes * self.expansion)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        """(N, inplanes, W, L, H) fp32 CUDA -> (N, 4*planes, w, l, h): feature_extractor.py:48-68 on the wgmma kernels (eval mode).
        Inside ResNet_FPN_256 the same layers run as part of the captured engine; this is the stand-alone entry point."""
        from ._eager import bottleneck_forward
        return bottleneck_forward(self, x, getattr(self, "precision", None))


class ResNet_FPN_256(EngineHolder, nn.Module):
    """ResNet-FPN backbone, same constructor / attributes as the reference (feature_extractor.py:159-194)."""

    def __init__(self, block, layers, input_dim=4, is_max_pool=False, precision=None):
        super().__init__()
        self.precision = _resolve_precision(precision)
        if input_dim != 4 or not is_max_pool or block is not Bottleneck:
            raise NotImplementedError("the CUDA engine implements the configuration run_rpn.py builds: "
                                      "ResNet_FPN_256(Bottleneck, [3,4,6,3], input_dim=4, is_max_pool=True)")
        self.in_planes = 64
        self.out_channels = 256
        self.conv1 = nn.Conv3d(input_dim, self.in_planes, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm3d(self.in_planes)
        self.layers = nn.ModuleList()
        self.start_deep = self.in_planes
        self.is_max_pool = is_max_pool
        for i in range(len(layers)):
            self.layers.append(self._make_layer(block, self.start_deep * (2 ** i), layers[i], stride=1 if i == 0 else 2))
        self.smooths = nn.ModuleList()
        for i in range(len(layers) - 1):
            self.smooths.append(nn.Conv3d(256, 256, kernel_size=3, stride=1, padding=1))
        self.latlayers = nn.ModuleList()
        for i in range(len(layers) - 1, -1, -1):
            self.latlayers.append(nn.Conv3d(block.expansion * self.start_deep * (2 ** i), self.out_channels,
                                            kernel_size=1, stride=1, padding=0))
        for m in self.modules():             # same init walk as the reference (feature_extractor.py:188-194)
            if isinstance(m, nn.Conv3d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm3d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)
        self._engine = None

    def _make_layer(self, block, planes, blocks, stride=1):
        downsample = None
        if stride != 1 or self.in_planes != planes * block.expansion:
            downsample = nn.Sequential(
                nn.Conv3d(self.in_planes, planes * block.expansion, kernel_size=1, stride=stride, bias=False),
                nn.BatchNorm3d(planes * block.expansion),
            )
        layers = [block(self.in_planes, planes, stride, downsample)]
        self.in_planes = planes * block.expansion
        for _ in range(1, blocks):
            layers.append(block(self.in_planes, planes))
        return nn.Sequential(*layers)

    def forward(self, x: torch.Tensor) -> List[torch.Tensor]:
        """x: (N,4,W,L,H) fp32 CUDA -> [P2,P3,P4,P5], each (N,256,w,l,h) fp32 (channels_last_3d strides)."""
        return self._engine_features(x)


def _not_built(name):
    class _Missing(nn.Module):
        def __init__(self, *a, **k):
            raise NotImplementedError(f"nerf_rpn_b200: backbone {name} is not implemented by the CUDA engine (built: ResNet_FPN_256, VGG_FPN, "
                                      "SwinTransformer_FPN -- the backbones of BASELINE.json's configurations; the name is importable because "
                                      "run_rpn.py:18-20 imports it)")
    _Missing.__name__ = name
    return _Missing


vgg_cfgs = {     # feature_extractor.py:278-286
    "A": [64, "M", 128, "M", 256, 256, "M", 512, 512, "M", 512, 512, "M"],
    "B": [64, 64, "M", 128, 128, "M", 256, 256, "M", 512, 512, "M", 512, 512, "M"],
    "D": [64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512, "M"],
    "E": [64, 64, "M", 128, 128, "M", 256, 256, 256, 256, "M", 512, 512, 512, 512, "M", 512, 512, 512, 512, "M"],
    "AF": [64, 128, "F", 256, 256, "M", "F", 512, 512, "M", "F", 512, 512, "M", "F"],
    "DF": [64, 64, 128, 128, "F", 256, 256, 256, "M", "F", 512, 512, 512, "M", "F", 512, 512, 512, "M", "F"],
    "EF": [64, 64, 128, 128, "F", 256, 256, 256, 256, "M", "F", 512, 512, 512, 512, "M", "F", 512, 512, 512, 512, "M", "F"],
}


class VGG_FPN(EngineHolder, nn.Module):
    """VGG-FPN backbone (feature_extractor.py:289-377), cfgs "AF" / "DF" / "EF" (run_rpn.py:277-280 builds AF and EF):
    stem Conv3d(4,64,7) [stride 2 + max-pool when input_size >= 160, else stride 1] + BN + ReLU, four stages of
    (Conv3d 3^3 + BN + ReLU)* [+ MaxPool3d(2,2,ceil_mode=True)], FPN neck on the four stage outputs."""

    def __init__(self, cfg: str = "AF", in_channels: int = 4, batch_norm: bool = True, input_size: int = 256,
                 conv_at_start: bool = False, precision=None):
        super().__init__()
        self.precision = _resolve_precision(precision)
        if conv_at_start or in_channels != 4 or not cfg.endswith("F"):
            raise NotImplementedError("the CUDA engine implements VGG_FPN(cfg in {AF,DF,EF}, 4, batch_norm, input_size)")
        from .fpn import FPN
        self.out_channels = 256
        self.layers = self.make_layers(vgg_cfgs[cfg], in_channels, batch_norm, input_size)
        stage_channels = [[v for v in grp if isinstance(v, int)][-1] for grp in self._groups(vgg_cfgs[cfg])]
        if stage_channels != [128, 256, 512, 512]:
            raise NotImplementedError("FPN input widths are fixed to [128,256,512,512] in the reference (feature_extractor.py:304)")
        self.fpn_neck = FPN([128, 256, 512, 512], self.out_channels, 4)
        self.conv_at_start = conv_at_start
        self.starting_layers = None
        self.ds_layers = None
        self._engine = None

    @staticmethod
    def _groups(cfg):
        out, cur = [], []
        for v in cfg:
            if v == "F":
                out.append(cur); cur = []
            else:
                cur.append(v)
        return out

    def make_layers(self, cfg, in_channels, batch_norm, input_size) -> nn.Sequential:
        layers, curr = [], []
        if input_size >= 160:
            layers += [nn.Conv3d(in_channels, 64, kernel_size=7, stride=2, padding=3), nn.BatchNorm3d(64), nn.ReLU(inplace=True),
                       nn.MaxPool3d(kernel_size=3, stride=2, padding=1)]
        else:
            layers += [nn.Conv3d(in_channels, 64, kernel_size=7, stride=1, padding=3), nn.BatchNorm3d(64), nn.ReLU(inplace=True)]
        c = 64
        for v in cfg:
            if v == "M":
                curr += [nn.MaxPool3d(kernel_size=2, stride=2, ceil_mode=True)]
            elif v == "F":
                layers += [nn.Sequential(*curr)]
                curr = []
            else:
                conv3d = nn.Conv3d(c, v, kernel_size=3, padding=1)
                curr += [conv3d, nn.BatchNorm3d(v), nn.ReLU(inplace=True)] if batch_norm else [conv3d, nn.ReLU(inplace=True)]
                c = v
        return nn.Sequential(*layers)

    def forward(self, X):
        """(N,4,W,L,H) fp32 CUDA -> tuple of 4 (N,256,w,l,h) fp32 feature maps (channels_last_3d strides)."""
        return tuple(self._engine_features(X))


class ShiftedWindowAttention(nn.Module):
    """Parameter container for 3-D shifted-window attention (feature_extractor.py:504-590): qkv / proj Linear layers, the
    (2w-1)^3 x heads relative-position bias table and its index buffer, created and initialised in the reference's order."""

    def __init__(self, dim, window_size, shift_size, num_heads, qkv_bias=True, proj_bias=True, attention_dropout=0.0, dropout=0.0):
        super().__init__()
        if len(window_size) != 3 or len(shift_size) != 3:
            raise ValueError("window_size and shift_size must be of length 3")
        self.window_size, self.shift_size, self.num_heads = window_size, shift_size, num_heads
        self.attention_dropout, self.dropout = attention_dropout, dropout
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim, bias=proj_bias)
        w = window_size
        self.relative_position_bias_table = nn.Parameter(torch.zeros((2 * w[0] - 1) * (2 * w[1] - 1) * (2 * w[2] - 1), num_heads))
        nn.init.trunc_normal_(self.relative_position_bias_table, std=0.02)
        coords = torch.stack(torch.meshgrid(torch.arange(w[0]), torch.arange(w[1]), torch.arange(w[2]), indexing="ij"))
        flat = torch.flatten(coords, 1)
        rel = (flat[:, :, None] - flat[:, None, :]).permute(1, 2, 0).contiguous()
        rel[:, :, 0] += w[0] - 1; rel[:, :, 1] += w[1] - 1; rel[:, :, 2] += w[2] - 1
        rel[:, :, 0] *= (2 * w[2] - 1) * (2 * w[1] - 1)
        rel[:, :, 1] *= (2 * w[2] - 1)
        self.register_buffer("relative_position_index", rel.sum(-1).flatten())


class SwinTransformerBlock(nn.Module):
    """feature_extractor.py:593-644: x + attn(norm1 x); x + mlp(norm2 x), MLP = Linear(C,4C) -> GELU -> Linear(4C,C)."""

    def __init__(self, dim, num_heads, window_size, shift_size, mlp_ratio=4.0, dropout=0.0, attention_dropout=0.0,
                 stochastic_depth_prob=0.0, norm_layer=nn.LayerNorm, attn_layer=ShiftedWindowAttention):
        super().__init__()
        self.norm1 = norm_layer(dim)
        self.attn = attn_layer(dim, window_size, shift_size, num_heads, attention_dropout=attention_dropout, dropout=dropout)
        self.stochastic_depth = nn.Identity()          # StochasticDepth("row") is the identity in eval mode
        self.norm2 = norm_layer(dim)
        hidden = int(dim * mlp_ratio)
        # torchvision.ops.misc.MLP(dim, [hidden, dim], activation_layer=nn.GELU, inplace=None): indices 0 and 3 carry parameters
        self.mlp = nn.Sequential(nn.Linear(dim, hidden), nn.GELU(), nn.Dropout(dropout), nn.Linear(hidden, dim), nn.Dropout(dropout))
        for m in self.mlp.modules():
            if isinstance(m, nn.Linear):
                nn.init.xavier_uniform_(m.weight)
                if m.bias is not None:
                    nn.init.normal_(m.bias, std=1e-6)


class PatchMerging(nn.Module):
    """feature_extractor.py:647-686: 2x2x2 gather (parity order 000,100,010,110,001,101,011,111 over H,W,D) -> LN(8C) -> Linear."""

    def __init__(self, dim, norm_layer=nn.LayerNorm, expand_dim=True):
        super().__init__()
        self.dim = dim
        self.reduction = nn.Linear(8 * dim, dim * 2 if expand_dim else dim, bias=False)
        self.norm = norm_layer(8 * dim)


class SwinTransformer_FPN(EngineHolder, nn.Module):
    """3-D Swin Transformer + FPN (feature_extractor.py:689-789), same constructor as the reference; run_rpn.py:281-292 builds
    Swin-T/S/B/L with patch 4^3, window 4^3."""

    def __init__(self, patch_size, embed_dim, depths, num_heads, window_size, mlp_ratio=4.0, dropout=0.0, attention_dropout=0.0,
                 stochastic_depth_prob=0.1, norm_layer=None, block=None, downsample_layer=None, expand_dim=True,
                 out_channels=256, input_dim=4, precision=None):
        super().__init__()
        self.precision = _resolve_precision(precision)
        from functools import partial
        from .fpn import FPN
        if list(patch_size) != [4, 4, 4] or list(window_size) != [4, 4, 4] or input_dim != 4 or not expand_dim or dropout or attention_dropout:
            raise NotImplementedError("the CUDA engine implements patch 4^3 / window 4^3 / 4 input channels (run_rpn.py:286-292)")
        norm_layer = norm_layer or partial(nn.LayerNorm, eps=1e-5)
        block = block or SwinTransformerBlock
        downsample_layer = downsample_layer or PatchMerging
        self.out_channels = out_channels
        self.patch_size, self.window_size, self.depths, self.num_heads, self.embed_dim = list(patch_size), list(window_size), list(depths), list(num_heads), embed_dim
        self.patch_partition = nn.Sequential(
            nn.Conv3d(input_dim, embed_dim, kernel_size=tuple(patch_size), stride=tuple(patch_size)),
            nn.Identity(),                                  # Permute([0,2,3,4,1]) in the reference: no parameters, index 1
            norm_layer(embed_dim),
        )
        self.stages = nn.ModuleList()
        total, bid, fpn_in = sum(depths), 0, []
        for i_stage in range(len(depths)):
            stage = []
            dim = embed_dim * 2 ** i_stage
            fpn_in.append(dim)
            if i_stage > 0:
                stage.append(downsample_layer(fpn_in[-2], norm_layer, expand_dim))
            for i_layer in range(depths[i_stage]):
                sd = stochastic_depth_prob * float(bid) / (total - 1)
                stage.append(block(dim, num_heads[i_stage], window_size=list(window_size),
                                   shift_size=[0 if i_layer % 2 == 0 else w // 2 for w in window_size], mlp_ratio=mlp_ratio,
                                   dropout=dropout, attention_dropout=attention_dropout, stochastic_depth_prob=sd, norm_layer=norm_layer))
                bid += 1
            self.stages.append(nn.Sequential(*stage))
        self.fpn_neck = FPN(fpn_in, out_channels, len(fpn_in))
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.trunc_normal_(m.weight, std=0.02)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
        self._engine = None

    def forward(self, x):
        return tuple(self._engine_features(x))


ResNet_FPN_64 = _not_built("ResNet_FPN_64")
ResNetSimplified_64 = _not_built("ResNetSimplified_64")
ResNetSimplified_256 = _not_built("ResNetSimplified_256")
