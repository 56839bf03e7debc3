"""RegionProposalNetwork. Mirrors nerf_rpn/model/rpn.py:167-229,458-536 (constructor, attributes, eval forward).
The eval branch (head -> decode -> per-level top-k -> clip/filter -> per-level NMS -> top post_nms_top_n,
rpn.py:485-512) is executed by the fused engine owned by NeRFRegionProposalNetwork; this class carries the
hyper-parameters and the sub-modules under the reference's attribute names so checkpoints and DDP wrap alike.
Training (rpn.py:514-534): the anchor <-> ground-truth assignment (`assign_targets_to_anchors`, rpn.py:240-290) runs on the
device (`nrpn_assign_targets`); sampling, the losses, the backward pass and the optimiser step are not implemented in this round.
"""
from typing import Dict, List, Optional, Tuple

import torch
from torch import Tensor, nn

from .. import ops


class RegionProposalNetwork(nn.Module):
    def __init__(self, anchor_generator, head, fg_iou_thresh: float, bg_iou_thresh: float, batch_size_per_mesh: int,
                 positive_fraction: float, pre_nms_top_n: Dict[str, int], post_nms_top_n: Dict[str, int],
                 nms_thresh: float, score_thresh: float = 0.0, iou_batch_size: int = 16, rotated_bbox: bool = False,
                 reg_loss_type: str = "smooth_l1"):
        super().__init__()
        self.anchor_generator = anchor_generator
        self.head = head
        self.rotate = rotated_bbox
        self.num_bbox_digits = 6 if not rotated_bbox else 7
        self.num_delta_digits = 6 if not rotated_bbox else 8
        self.fg_iou_thresh, self.bg_iou_thresh = fg_iou_thresh, bg_iou_thresh
        self.batch_size_per_mesh, self.positive_fraction = batch_size_per_mesh, positive_fraction
        self.iou_batch_size = iou_batch_size
        self._pre_nms_top_n = pre_nms_top_n
        self._post_nms_top_n = post_nms_top_n
        self.nms_thresh = nms_thresh
        self.score_thresh = score_thresh
        self.reg_loss_type = reg_loss_type
        self.min_size = 1e-3

    def pre_nms_top_n(self) -> int:
        return self._pre_nms_top_n["training" if self.training else "testing"]

    def post_nms_top_n(self) -> int:
        return self._post_nms_top_n["training" if self.training else "testing"]

    @torch.no_grad()
    def assign_targets_to_anchors(self, anchors: List[Tensor], targets: List[Tensor],
                                  padding_masks: Optional[List[Tensor]] = None) -> Tuple[List[Tensor], List[Tensor]]:
        """rpn.py:240-290 with the same arguments and results (labels in {1, 0, -1} and the matched ground-truth box of every
        anchor), computed by one fused device pass per mesh: no (G, num_anchors) IoU matrix, no chunking over ground truth."""
        labels, matched_gt_boxes = [], []
        for i, (anchors_per_mesh, gt_boxes) in enumerate(zip(anchors, targets)):
            dev = anchors_per_mesh.device
            a = anchors_per_mesh.to(device="cuda", dtype=torch.float32).contiguous()
            if gt_boxes.numel() == 0:                       # background mesh (rpn.py:246-250)
                matched_gt_boxes.append(torch.zeros(anchors_per_mesh.shape, dtype=torch.float32, device=dev))
                lab = torch.zeros((anchors_per_mesh.shape[0],), dtype=torch.float32, device=dev)
                if padding_masks is not None:
                    lab[~padding_masks[i].to(dev)] = -1.0
                labels.append(lab)
                continue
            gt = gt_boxes.to(device="cuda", dtype=torch.float32).contiguous()
            valid = None if padding_masks is None else padding_masks[i].to("cuda")
            lab, idx = ops.assign_targets(a, gt, valid, self.fg_iou_thresh, self.bg_iou_thresh, True)
            labels.append(lab.to(dev))
            matched_gt_boxes.append(gt[idx.clamp(min=0)].to(dev))
        return labels, matched_gt_boxes

    def forward(self, meshes, features, original_mesh_sizes, targets=None, objectness_output_paths=None):
        """rpn.py:458-536, eval branch, stand-alone: meshes (N,4,W,L,H), features = 4 x (N,256,w,l,h) fp32 CUDA ->
        (boxes [K_i x 6|7], level_indexes [K_i], losses {}, scores [K_i]).  Head = model/_eager.py (one launch per layer over all
        levels), then the fused device post-processing (anchors, decode, per-level top-k, clip / filter, per-level NMS, top
        post_nms_top_n) -- the same kernels NeRFRegionProposalNetwork.forward runs inside its captured engine."""
        if self.training:
            raise NotImplementedError("nerf_rpn_b200: RegionProposalNetwork.forward in training mode is not a stand-alone path; the losses "
                                      "are computed by the whole-model training engine (NeRFRegionProposalNetwork.forward / train.py)")
        from ._eager import rpn_head_pred
        pred = rpn_head_pred(self.head, features, getattr(self, "precision", None))
        if objectness_output_paths is not None:
            write_objectness(pred, self.head.cls_logits.weight.shape[0], original_mesh_sizes, objectness_output_paths)
        n = pred[0].shape[0]
        mesh = tuple(int(v) for v in meshes.shape[-3:])
        fdims = [tuple(p.shape[1:4]) for p in pred]
        strides = [tuple(mesh[k] // d[k] for k in range(3)) for d in fdims]
        ag = self.anchor_generator
        cells, A = ag.cell_anchors_np(), ag.num_anchors_per_location()[0]
        boxes, levels, scores = [], [], []
        for i in range(n):
            valid = tuple(int(v) for v in original_mesh_sizes[i]) if n > 1 else None       # padding masks only when batch > 1 (rpn.py:501)
            desc = ops.make_rpn_desc([p[i].reshape(-1, 128) for p in pred], fdims, strides, cells, A, self.rotate, self.pre_nms_top_n(),
                                     self.post_nms_top_n(), self.nms_thresh, self.score_thresh, self.min_size, mesh, valid=valid)
            b, s, lv, cnt = ops.rpn_proposals(desc, pred[0].device)
            k = int(cnt.item())
            boxes.append(b[:k]); scores.append(s[:k]); levels.append(lv[:k])
        return boxes, levels, {}, scores


def write_objectness(pred, A, ori_sizes, output_paths):
    """--output_voxel_scores (rpn.py:538-549): per scene and level the maximum objectness LOGIT over the anchors, cropped to the
    un-padded extent ceil(size / 2^(level+2)), written as npz with keys '0'..'3'.  pred: per level the head's fused channels-last
    output (N, w, l, h, >= A) whose first A channels are the logits."""
    import numpy as np
    for i in range(len(ori_sizes)):
        all_levels = {}
        for level, p in enumerate(pred):
            score = p[i][..., :A].max(dim=-1)[0]
            w, l, h = np.ceil(np.array(ori_sizes[i]) / 2 ** (level + 2)).astype(int)
            all_levels[str(level)] = score[:w, :l, :h].cpu().numpy()
        np.savez_compressed(output_paths[i], **all_levels)
