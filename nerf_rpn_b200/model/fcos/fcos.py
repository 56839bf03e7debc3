"""Anchor-free head. Mirrors nerf_rpn/model/fcos/fcos.py (Scale :18-24, FCOSHead :27-130, FCOSModule :133-284,
FCOSOverNeRF :287-386) and fcos/inference.py:11-46 (FCOSPostProcessor's hyper-parameters): same class names, constructor
arguments, attribute / parameter names (state_dict keys `fcos_module.head.{cls_tower,bbox_tower}.{i}.*`, `cls_logits.*`,
`bbox_pred.*`, `centerness.*`, `scales.{i}.scale`) and creation / init order, so seeds and checkpoints line up.
Inference (`--norm_reg_targets --centerness_on_reg`, the flags of test_fcos.sh) runs on the fused CUDA engine.  The training LOSS
(fcos/loss.py) is built (`FCOSModule.loss_evaluator`, model/fcos/loss.py: two kernels + one autograd node over the head outputs);
the backward pass of the FCOS towers (GroupNorm) and a captured FCOS training step are not, so `FCOSOverNeRF.forward` still raises
in training mode."""
import math
from typing import List

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from ...precision import EngineHolder, resolve as _resolve_precision
from .loss import FCOSLossComputation


class Scale(nn.Module):
    def __init__(self, init_value=1.0):
        super().__init__()
        self.scale = nn.Parameter(torch.FloatTensor([init_value]))

    def forward(self, input):
        return input * self.scale


class FCOSHead(nn.Module):
    def __init__(self, in_channels, num_convs, fpn_strides, norm_reg_targets=True, centerness_on_reg=True, use_obb=False):
        super().__init__()
        if not (norm_reg_targets and centerness_on_reg):
            raise NotImplementedError("nerf_rpn_b200 implements the reference's evaluated FCOS configuration: "
                                      "--norm_reg_targets --centerness_on_reg (test_fcos.sh)")
        if in_channels != 256:
            raise NotImplementedError("FCOS towers are built for 256 channels (GroupNorm(32, 256))")
        self.fpn_strides = fpn_strides
        self.norm_reg_targets, self.centerness_on_reg = norm_reg_targets, centerness_on_reg
        self.num_convs, self.use_obb = num_convs, use_obb
        cls_tower, bbox_tower = [], []
        for _ in range(num_convs):
            cls_tower += [nn.Conv3d(in_channels, in_channels, kernel_size=3, stride=1, padding=1, bias=True),
                          nn.GroupNorm(32, in_channels), nn.ReLU()]
            bbox_tower += [nn.Conv3d(in_channels, in_channels, kernel_size=3, stride=1, padding=1, bias=True),
                           nn.GroupNorm(32, in_channels), nn.ReLU()]
        self.add_module('cls_tower', nn.Sequential(*cls_tower))
        self.add_module('bbox_tower', nn.Sequential(*bbox_tower))
        self.cls_logits = nn.Conv3d(in_channels, 1, kernel_size=3, stride=1, padding=1)
        self.bbox_pred = nn.Conv3d(in_channels, 8 if use_obb else 6, kernel_size=3, stride=1, padding=1)
        self.centerness = nn.Conv3d(in_channels, 1, kernel_size=3, stride=1, padding=1)
        for modules in [self.cls_tower, self.bbox_tower, self.cls_logits, self.bbox_pred, self.centerness]:
            for l in modules.modules():
                if isinstance(l, nn.Conv3d):
                    torch.nn.init.normal_(l.weight, std=0.01)
                    torch.nn.init.constant_(l.bias, 0)
        prior_prob = 0.01
        torch.nn.init.constant_(self.cls_logits.bias, -math.log((1 - prior_prob) / prior_prob))
        self.scales = nn.ModuleList([Scale(init_value=1.0) for _ in range(5)])

    def forward(self, x):
        """fcos/fcos.py:104-130 stand-alone (eval): list of (N,256,w,l,h) fp32 CUDA -> (logits, bbox_reg, centerness) lists."""
        from .._eager import fcos_head_forward
        return fcos_head_forward(self, x, getattr(self, "precision", None))


class FCOSPostProcessor(nn.Module):
    """Hyper-parameter holder with the reference's attribute names (fcos/inference.py:18-46)."""

    def __init__(self, pre_nms_thresh, pre_nms_top_n, nms_thresh, fpn_post_nms_top_n, min_size, num_classes,
                 bbox_aug_enabled=False, use_obb=False):
        super().__init__()
        self.pre_nms_thresh, self.pre_nms_top_n, self.nms_thresh = pre_nms_thresh, pre_nms_top_n, nms_thresh
        self.fpn_post_nms_top_n, self.min_size, self.num_classes = fpn_post_nms_top_n, min_size, num_classes
        self.bbox_aug_enabled, self.use_obb = bbox_aug_enabled, use_obb


class FCOSModule(nn.Module):
    def __init__(self, args, in_channels, fpn_strides, world_size=1):
        super().__init__()
        self.head = FCOSHead(in_channels, args.num_convs, fpn_strides, norm_reg_targets=args.norm_reg_targets,
                             centerness_on_reg=args.centerness_on_reg, use_obb=args.rotated_bbox)
        self.box_selector_test = FCOSPostProcessor(args.pre_nms_thresh, args.pre_nms_top_n, args.nms_thresh,
                                                   args.fpn_post_nms_top_n, args.min_size, 1, use_obb=args.rotated_bbox)
        # fcos.py:152-158; the defaults are run_fcos.py:103-111's for callers that build `args` for inference only
        self.loss_evaluator = FCOSLossComputation(
            fpn_strides, getattr(args, "center_sampling_radius", 1.5), getattr(args, "iou_loss_type", "iou"), args.norm_reg_targets,
            world_size=world_size, use_obb=args.rotated_bbox, use_additional_l1_loss=getattr(args, "use_additional_l1_loss", False),
            proj2d_loss_weight=getattr(args, "proj2d_loss_weight", 0.0))
        self.fpn_strides = fpn_strides
        self.world_size = world_size

    def forward(self, grid_sizes, features, targets=None, objectness_output_paths=None):
        raise RuntimeError("nerf_rpn_b200.FCOSModule runs inside FCOSOverNeRF.forward (one captured launch sequence)")

    def _forward_train(self, locations, box_cls, box_regression, centerness, targets, padding_masks):
        """fcos.py:200-210: the three losses of the head outputs (differentiable w.r.t. them)."""
        loss_box_cls, loss_box_reg, loss_centerness = self.loss_evaluator(locations, box_cls, box_regression, centerness, targets,
                                                                          padding_masks=padding_masks)
        return None, None, {"loss_cls": loss_box_cls, "loss_reg": loss_box_reg, "loss_centerness": loss_centerness}

    def compute_locations(self, features):
        """fcos.py:221-250: per level (w * l * h, 3), z fastest, voxel index * stride + stride // 2."""
        locations = []
        for level, feature in enumerate(features):
            w, l, h = feature.size()[-3:]
            stride = self.fpn_strides[level]
            axes = [torch.arange(0, n * stride, step=stride, dtype=torch.float32, device=feature.device) for n in (w, l, h)]
            grid = torch.stack(torch.meshgrid(*axes, indexing="ij"), dim=-1).reshape(-1, 3)
            locations.append(grid + stride // 2)
        return locations

    def output_objectness(self, box_cls, centerness, ori_sizes, output_paths):
        """--output_voxel_scores of run_fcos.py (fcos.py:268-284): per scene an npz with one array per level, sqrt(sigmoid(cls) * sigmoid(centerness))
        cropped to the scene's own extent ceil(size / stride).  File export: host-side plumbing on the head's outputs."""
        for i in range(len(ori_sizes)):
            all_levels = {}
            for level in range(len(box_cls)):
                score = torch.sqrt(box_cls[level][i].sigmoid() * centerness[level][i].sigmoid())
                w, l, h = np.ceil(np.array(ori_sizes[i]) / self.fpn_strides[level]).astype(int)
                all_levels[str(level)] = score[0, :w, :l, :h].cpu().numpy()
            np.savez_compressed(output_paths[i], **all_levels)

    def compute_padding_masks(self, locations, ori_sizes):
        """fcos.py:252-266: per level (N, P_l) bool, True where the location lies inside the scene's own extent."""
        masks = []
        for loc in locations:
            size = torch.tensor([list(s) for s in ori_sizes], dtype=loc.dtype, device=loc.device)          # (N, 3)
            masks.append((loc[None] < size[:, None]).all(dim=-1))
        return masks


class FCOSOverNeRF(EngineHolder, nn.Module):
    def __init__(self, args, backbone, fpn_strides, world_size=1, precision=None) -> None:
        if not hasattr(backbone, "out_channels"):
            raise ValueError("backbone should contain an attribute out_channels specifying the number of output "
                             "channels (assumed to be the same for all the levels)")
        super().__init__()
        self.args = args
        self.world_size = world_size
        self.backbone = backbone
        self.fcos_module = FCOSModule(args, backbone.out_channels, fpn_strides, world_size=world_size)
        self.precision = _resolve_precision(precision)
        self._engine = None

    def transform(self, meshes):
        shapes = [mesh.shape for mesh in meshes]
        target_shape = np.max(shapes, axis=0)
        for i, mesh in enumerate(meshes):
            meshes[i] = F.pad(mesh, (0, target_shape[-1] - mesh.shape[-1], 0, target_shape[-2] - mesh.shape[-2],
                                     0, target_shape[-3] - mesh.shape[-3]), mode="constant", value=0)
        return meshes

    def engine(self):
        from ...engine import RPNInferenceEngine
        precision = _resolve_precision(getattr(self, "precision", None))
        if self._engine is None or self._engine.precision != precision:
            m, sel = self.fcos_module, self.fcos_module.box_selector_test
            self._engine = RPNInferenceEngine(self.backbone, m.head, fcos=dict(
                use_obb=sel.use_obb, pre_nms_thresh=sel.pre_nms_thresh, pre_nms_top_n=sel.pre_nms_top_n,
                nms_thresh=sel.nms_thresh, post_nms_top_n=sel.fpn_post_nms_top_n, min_size=sel.min_size,
                fpn_strides=list(m.fpn_strides)), precision=precision)
        return self._engine

    def forward(self, meshes, targets=None, objectness_output_paths=None):
        if self.training:
            raise NotImplementedError("nerf_rpn_b200: the FCOS training step (backward through the GroupNorm towers) is not built; the loss itself is: "
                                      "fcos_module.loss_evaluator(locations, box_cls, box_regression, centerness, targets, padding_masks)")
        original_mesh_sizes = []
        for mesh in meshes:
            val = mesh.shape[-3:]
            torch._assert(len(val) == 3, f"expecting the last three dimensions of the Tensor to be W, L and H instead got {mesh.shape[-3:]}")
            original_mesh_sizes.append((val[0], val[1], val[2]))
        if len(meshes) > 1:
            meshes = self.transform(meshes)
        mesh_tensors = meshes[0].unsqueeze(0) if len(meshes) == 1 else torch.stack(meshes, dim=0)
        if not mesh_tensors.is_contiguous():
            mesh_tensors = mesh_tensors.contiguous()
        if objectness_output_paths is not None:
            # the export reads the head's class / centerness maps: the stand-alone (eager) forwards of the backbone and the head produce them as
            # NCDHW fp32 tensors, next to the fused run below that produces the proposals (an export option, not the timed path)
            with torch.no_grad():
                feats = list(self.backbone(mesh_tensors))
                box_cls, _, ctrness = self.fcos_module.head(feats)
            self.fcos_module.output_objectness(box_cls, ctrness, original_mesh_sizes, objectness_output_paths)
        plan = self.engine().forward_device(mesh_tensors, original_mesh_sizes)
        torch.cuda.current_stream().wait_event(plan.done)
        counts = plan.out_count.tolist()
        boxes = [plan.out_boxes[i, :k].clone() for i, k in enumerate(counts)]
        scores = [plan.out_scores[i, :k].clone() for i, k in enumerate(counts)]
        return boxes, {}, scores
