"""Anchor generator and RPN head. Mirrors nerf_rpn/model/anchor.py:
  AnchorGenerator3D   anchor.py:14-174
  RPNHead             anchor.py:177-213
In the CUDA engine anchors are never materialised (2.43 M x 6 floats per scene in the reference): the decode
kernel rebuilds the anchor of a selected candidate from its flat index.  AnchorGenerator3D therefore only has to
produce the per-level cell anchors in the reference's order -- which comes from iterating a Python set of
permutations (anchor.py:40-46,57-60) and is reproduced by evaluating the same expression.
"""
import itertools
from typing import List

import numpy as np
import torch
from torch import nn, Tensor


class AnchorGenerator3D(nn.Module):
    def __init__(self, sizes, aspect_ratios, is_normalized=False):
        super().__init__()
        self.sizes = sizes
        self.aspect_ratios = aspect_ratios
        self.is_normalized = is_normalized
        self.aspect_ratios_unique = []
        for size in self.aspect_ratios:
            cur = set()
            for ratio in size:
                cur.update(set(itertools.permutations(ratio)))
            self.aspect_ratios_unique.append(list(cur))

    def num_anchors_per_location(self):
        return [len(s) * len(a) for s, a in zip(self.sizes, self.aspect_ratios_unique)]

    def cell_anchors_np(self) -> List[np.ndarray]:
        """Per level (A, 6) fp32 [-w,-h,-d,w,h,d]/2, rounded half-to-even (anchor.py:51-82)."""
        out = []
        for scales, ratios in zip(self.sizes, self.aspect_ratios):
            sc = np.asarray(scales, dtype=np.float32)
            cols = [[], [], []]
            for ratio in ratios:
                perms = np.asarray(list(set(itertools.permutations(ratio))), dtype=np.float32)
                if self.is_normalized:
                    wgt = np.float32(1.0)
                    for i in range(3):
                        wgt = np.float32(wgt * np.float32(ratio[i]))
                    perms = perms / np.float32(np.power(wgt, np.float32(1.0 / 3.0)))
                for k in range(3):
                    cols[k].append(perms[:, k])
            w, h, d = [(np.concatenate(c)[:, None] * sc[None, :]).reshape(-1) for c in cols]
            base = np.stack([-w, -h, -d, w, h, d], axis=1).astype(np.float32) / np.float32(2)
            out.append(np.round(base).astype(np.float32))
        return out

    def forward(self, meshes: Tensor, feature_maps: List[Tensor]):
        """Materialised anchors, (anchors per mesh, per-level lists) like the reference (anchor.py:154-174).
        Only used by callers that want the tensors; the engine does not call this."""
        grid_sizes = [fm.shape[-3:] for fm in feature_maps]
        mesh_size = meshes.shape[-3:]
        device = feature_maps[0].device
        cells = [torch.from_numpy(c).to(device) for c in self.cell_anchors_np()]
        per_level = []
        for size, cell in zip(grid_sizes, cells):
            stride = [mesh_size[i] // size[i] for i in range(3)]
            sh = [torch.arange(0, size[i], dtype=torch.float32, device=device) * stride[i] for i in range(3)]
            gx, gy, gz = torch.meshgrid(sh[0], sh[1], sh[2], indexing="ij")
            shifts = torch.stack((gx.reshape(-1), gy.reshape(-1), gz.reshape(-1)) * 2, dim=1)
            per_level.append((shifts.view(-1, 1, 6) + cell.view(1, -1, 6)).reshape(-1, 6))
        non_cat = [list(per_level) for _ in range(meshes.shape[0])]
        return [torch.cat(a) for a in non_cat], non_cat


class RPNHead(nn.Module):
    """4 x (Conv3d 3^3 + ReLU) shared over levels, then 1^3 objectness and box-delta predictors."""

    def __init__(self, in_channels, num_anchors, conv_depth=1, rotate=False):
        super().__init__()
        convs = []
        for _ in range(conv_depth):
            convs.append(nn.Conv3d(in_channels, in_channels, kernel_size=3, padding=1))
            convs.append(nn.ReLU(inplace=True))
        self.conv = nn.Sequential(*convs)
        self.cls_logits = nn.Conv3d(in_channels, num_anchors, kernel_size=1, stride=1)
        self.bbox_pred = nn.Conv3d(in_channels, num_anchors * (8 if rotate else 6), kernel_size=1, stride=1)
        self.num_anchors, self.rotate = num_anchors, rotate
        for layer in self.modules():
            if isinstance(layer, nn.Conv3d):
                torch.nn.init.normal_(layer.weight, std=0.01)
                if layer.bias is not None:
                    torch.nn.init.constant_(layer.bias, 0)

    def forward(self, x: List[Tensor]):
        """anchor.py:206-213 stand-alone: list of (N,256,w,l,h) fp32 CUDA -> (logits [(N,A,w,l,h)], bbox_reg [(N,A*6|8,w,l,h)]).
        One launch per layer over all levels; inside NeRFRegionProposalNetwork the same layers are part of the captured engine."""
        from ._eager import rpn_head_forward
        return rpn_head_forward(self, x, getattr(self, "precision", None))
