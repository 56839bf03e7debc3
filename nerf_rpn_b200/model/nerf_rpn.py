"""NeRFRegionProposalNetwork. Mirrors nerf_rpn/model/nerf_rpn.py:22-217: same constructor keywords, same
forward(meshes, targets=None, objectness_output_paths=None) -> ([features, proposals, level_index], losses, scores).
"""
from typing import List, Tuple

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from ..precision import resolve as _resolve_precision
from .anchor import AnchorGenerator3D, RPNHead
from .rpn import RegionProposalNetwork, write_objectness


def _default_anchorgen():
    anchor_sizes = ((8,), (16,), (32,), (64,),)
    aspect_ratios = (((1., 1., 1.), (1., 1., 2.), (1., 2., 2.), (1., 1., 3.), (1., 3., 3.)),) * len(anchor_sizes)
    return AnchorGenerator3D(anchor_sizes, aspect_ratios)


class _RPNTrainStep(torch.autograd.Function):
    """One autograd node around the engine's forward / backward launch lists (see NeRFRegionProposalNetwork._forward_train)."""

    @staticmethod
    def forward(ctx, eng, grids, targets, *params):
        plan = eng.plan_for(grids)
        plan.forward_loss(grids, targets, 1.0, 1.0, 0.0, eval_2d=True)          # the 2-D projection loss is reported like the reference does
        ctx.eng, ctx.plan, ctx.forward_count = eng, plan, eng.forward_count
        losses = eng.losses.clone()
        return losses[0].clone(), losses[1].clone(), eng.loss_2d.clone()          # fresh 0-dim tensors (run_rpn.py:385-386 scales them in place)

    @staticmethod
    def backward(ctx, g_obj, g_reg, g_2d):
        eng, plan = ctx.eng, ctx.plan
        if eng.forward_count != ctx.forward_count:
            # every batch shape trains in the engine's one set of activation buffers: a later forward has overwritten this one's
            raise RuntimeError("nerf_rpn_b200: another training forward ran on this model before this loss's backward; the CUDA training engine "
                               "keeps the activations of one forward at a time -- call backward() after each forward (accumulate gradients "
                               "over several backward() calls instead of summing the losses of several forwards)")
        plan.loss_grad(float(g_obj), float(g_reg), float(g_2d))          # the loss weights arrive as the upstream gradients (run_rpn.py:385-387)
        plan.backward()
        inv = 1.0 / eng.loss_scale
        grads = []
        for p in (list(eng.bb.parameters()) if not plan.frozen else []) + list(eng.head.parameters()):
            g = eng.grad_of(p).view(p.shape)
            grads.append(g * inv if inv != 1.0 else g.clone())
        return (None, None, None, *grads)


class NeRFRegionProposalNetwork(nn.Module):
    def __init__(self, backbone, rpn_anchor_generator=None, rpn_head=None, rpn_pre_nms_top_n_train=2000,
                 rpn_pre_nms_top_n_test=1000, rpn_post_nms_top_n_train=2000, rpn_post_nms_top_n_test=1000,
                 rpn_nms_thresh=0.7, rpn_fg_iou_thresh=0.7, rpn_bg_iou_thresh=0.3, rpn_batch_size_per_image=256,
                 rpn_positive_fraction=0.5, rpn_score_thresh=0.0, iou_batch_size=16, rotated_bbox=False,
                 reg_loss_type="smooth_l1", precision=None, density_to_alpha_on_device=False, **kwargs):
        if not hasattr(backbone, "out_channels"):
            raise ValueError("backbone should contain an attribute out_channels specifying the number of output "
                             "channels (assumed to be the same for all the levels)")
        if not isinstance(rpn_anchor_generator, (AnchorGenerator3D, type(None))):
            raise TypeError(f"rpn_anchor_generator should be of type AnchorGenerator or None instead of {type(rpn_anchor_generator)}")
        out_channels = backbone.out_channels
        if rpn_anchor_generator is None:
            rpn_anchor_generator = _default_anchorgen()
        if rpn_head is None:
            rpn_head = RPNHead(out_channels, rpn_anchor_generator.num_anchors_per_location()[0], rotated_bbox)
        rpn = RegionProposalNetwork(
            rpn_anchor_generator, rpn_head, rpn_fg_iou_thresh, rpn_bg_iou_thresh, rpn_batch_size_per_image,
            rpn_positive_fraction, dict(training=rpn_pre_nms_top_n_train, testing=rpn_pre_nms_top_n_test),
            dict(training=rpn_post_nms_top_n_train, testing=rpn_post_nms_top_n_test), rpn_nms_thresh,
            score_thresh=rpn_score_thresh, iou_batch_size=iou_batch_size, rotated_bbox=rotated_bbox,
            reg_loss_type=reg_loss_type)
        super().__init__()
        self.backbone = backbone
        self.rpn = rpn
        self.precision = _resolve_precision(precision)     # "bf16" | "fp16" | "fp16_w2" (nerf_rpn_b200/precision.py); explicit, in repr
        # True: feed RAW densities (dataset built with normalize_density=False) and let the stem packing kernel apply datasets.py:165-167
        self.density_to_alpha_on_device = bool(density_to_alpha_on_device)
        self._engine = None
        self._engine_key = None
        self._train_engine = None

    # engines hold CUDA graphs, streams and ctypes objects: keep them out of pickles / deep copies (torch.save(model), spawn-based DDP)
    def __getstate__(self):
        d = self.__dict__.copy()
        d["_engine"], d["_engine_key"], d["_train_engine"] = None, None, None
        return d

    def extra_repr(self):
        return f"precision={self.precision!r}"

    # nerf_rpn.py:129-146
    def transform(self, meshes, targets=None):
        if len(meshes) > 1:
            shapes = [mesh.shape for mesh in meshes]
            target_shape = np.max(shapes, axis=0)
            for i, mesh in enumerate(meshes):
                meshes[i] = F.pad(mesh, (0, target_shape[-1] - mesh.shape[-1], 0, target_shape[-2] - mesh.shape[-2],
                                         0, target_shape[-3] - mesh.shape[-3]), mode="constant", value=0)
        return meshes, targets

    def engine(self):
        from ..engine import RPNInferenceEngine
        r = self.rpn
        precision = _resolve_precision(self.precision)
        key = (r._pre_nms_top_n["testing"], r._post_nms_top_n["testing"], r.nms_thresh, r.score_thresh, r.rotate, precision,
               self.density_to_alpha_on_device)
        if self._engine is None or key != self._engine_key:
            ag = r.anchor_generator
            self._engine = RPNInferenceEngine(
                self.backbone, r.head, ag.cell_anchors_np(), ag.num_anchors_per_location()[0], r.rotate,
                r._pre_nms_top_n["testing"], r._post_nms_top_n["testing"], r.nms_thresh, r.score_thresh, r.min_size,
                precision=precision, density_to_alpha=self.density_to_alpha_on_device)
            self._engine_key = key
        return self._engine

    # ------------------------------------------------------------------------------------------------ training
    def train_engine(self, **kw):
        """The CUDA training engine bound to this model (nerf_rpn_b200/train.py).  Created on first use; keyword arguments (precision,
        lr, weight_decay, clip_grad_norm, reg_loss_weight, process_group ...) configure a NEW engine."""
        from ..train import RPNTrainEngine
        if self._train_engine is None or kw:
            self._train_engine = RPNTrainEngine(self, **kw)
        return self._train_engine

    def frozen_backbone(self) -> bool:
        """True when no backbone parameter (FPN included) requires a gradient and every head parameter does: the pattern of run_rpn.py
        --freeze_backbone, which the training forward runs as the shorter frozen-backbone step.  Read at every training forward."""
        return not any(p.requires_grad for p in self.backbone.parameters()) and all(p.requires_grad for p in self.rpn.head.parameters())

    def _forward_train(self, meshes, targets):
        """Training-mode forward as the reference defines it (nerf_rpn.py:166-217 + rpn.py:514-534): returns losses that carry a
        grad_fn, so the UNMODIFIED loop of run_rpn.py:384-395 (`loss.backward(); clip_grad_norm_; optimizer.step()`) and a DDP
        wrapper drive the CUDA forward / backward kernels: torch.autograd only sees ONE node whose backward runs the engine's launch
        list and hands every parameter its gradient.  A backbone whose every parameter has requires_grad = False under a fully trainable
        head (run_rpn.py --freeze_backbone) runs the engine's frozen-backbone step: only the head's backward, and only the head's
        parameters enter the node, so their gradients are all that autograd, clip_grad_norm_, the optimiser and DDP see."""
        if targets is None:
            raise ValueError("targets should not be None")
        eng = self.train_engine()
        eng.overlap_allreduce = False               # gradients are returned to autograd; a DDP wrapper all-reduces them itself
        eng.freeze_backbone = self.frozen_backbone()
        eng.sync_parameters()
        # meshes of any sizes go to the engine as they are (each in its own memory order): it trains the batch padded to their element-wise
        # maximum like transform() does, without materialising it -- and without padding the caller's list in place, as transform() would
        grids = [m if (m.is_cuda and m.dtype == torch.float32) else m.cuda().float() for m in meshes]
        head = list(self.rpn.head.parameters())
        params = head if eng.freeze_backbone else list(self.backbone.parameters()) + head
        l_obj, l_reg, l_2d = _RPNTrainStep.apply(eng, grids, [t for t in targets], *params)
        return [None, None, None], {"loss_objectness": l_obj, "loss_rpn_box_reg": l_reg, "loss_rpn_box_reg_2d": l_2d}, None

    def forward(self, meshes, targets=None, objectness_output_paths=None):
        if self.training:
            return self._forward_train(meshes, targets)
        original_mesh_sizes: List[Tuple[int, int, int]] = []
        for mesh in meshes:
            val = mesh.shape[-3:]
            torch._assert(len(val) == 3, f"expecting the last three dimensions of the Tensor to be W, H and D instead got {mesh.shape[-3:]}")
            original_mesh_sizes.append((val[0], val[1], val[2]))
        meshes, targets = self.transform(meshes, targets)
        # The reference's dataset yields each mesh as a (4,W,L,H) VIEW of the on-disk (W,L,H,4) array (datasets.py:55-56). Such
        # meshes are kept in that memory order (the stem packing reads it with one 128-bit load per voxel); anything else is
        # made contiguous NCDHW like the reference's torch.stack does.
        if all(m.dim() == 4 and not m.is_contiguous() and m.permute(1, 2, 3, 0).is_contiguous() for m in meshes):
            mesh_tensors = torch.stack([m.permute(1, 2, 3, 0) for m in meshes], dim=0).permute(0, 4, 1, 2, 3)
        else:
            mesh_tensors = meshes[0].unsqueeze(0) if len(meshes) == 1 else torch.stack(meshes, dim=0)
            if not mesh_tensors.is_contiguous():
                mesh_tensors = mesh_tensors.contiguous()
        valid = original_mesh_sizes if len(meshes) > 1 else None     # padding masks only when batch > 1 (rpn.py:501)
        plan = self.engine().forward_device(mesh_tensors, valid)
        torch.cuda.current_stream().wait_event(plan.done)            # post-processing runs on the engine's side stream
        counts = plan.out_count.tolist()                              # the one host sync: data-dependent output sizes
        features = [f.permute(0, 4, 1, 2, 3).float() for f in plan.features]
        if objectness_output_paths is not None:
            write_objectness(plan.pred, self.rpn.anchor_generator.num_anchors_per_location()[0], original_mesh_sizes,
                             objectness_output_paths)
        proposals = [plan.out_boxes[i, :k].clone() for i, k in enumerate(counts)]
        level_index = [plan.out_levels[i, :k].clone() for i, k in enumerate(counts)]
        scores = [plan.out_scores[i, :k].clone() for i, k in enumerate(counts)]
        return [features, proposals, level_index], {}, scores
