"""FCOS training loss. Mirrors nerf_rpn/model/fcos/loss.py:185-591 (`FCOSLossComputation`: same constructor arguments, `prepare_targets`,
`compute_centerness_targets`, `__call__(locations, box_cls, box_regression, centerness, targets, padding_masks)` -> (cls_loss, reg_loss,
centerness_loss)), computed by two kernels of libnerf_rpn_b200.so instead of the reference's (locations, G, 8) tensors:

  nrpn_fcos_targets   per scene: every location against every ground-truth box (AABB or OBB midpoint-offset encoding), centre sampling,
                      size-of-interest range, smallest box wins                                              (loss.py:213-441)
  nrpn_fcos_loss      focal loss over every unmasked location; on the positives the centerness target, its BCE, the centerness-weighted
                      regression loss (smooth-L1, or -log IoU / 1 - IoU / 1 - GIoU of the axis-aligned head), the alpha / beta smooth-L1 of
                      the OBB head, all with their gradients in the head's NCDHW layout; fp64 sums                (loss.py:487-591)

The three losses come out of ONE autograd node whose backward hands the stored gradients (scaled by the normalisers) to the head outputs.
The rotated-IoU term of the OBB head (RotatedIOULoss, loss.py:134-181) is evaluated on the gathered positives with the differentiable
decode (model/coder_torch.py decode_fcos_obb) + cal_iou_3d / cal_giou_3d / cal_diou_3d (fused IoU kernel and its backward), and its gradient is added to
the regression gradient of the node.  The two normalisers (positives, sum of centerness targets; `reduce_sum`, loss.py:202-208) are all-reduced
as ONE two-element fp64 tensor and stay on the device: the axis-aligned / smooth-L1 paths never synchronise the host.
The 2-D projection loss of the OBB head (proj2d_loss_weight > 0, loss.py:452-485; model/proj2d.py) rides on the same gathered positives.
No CPU path: CUDA tensors only."""
from typing import List, Optional

import torch

from ... import ops
from ..coder_torch import decode_fcos_obb
from ..proj2d import fcos_projection_loss

INF = 100000000


def _all_reduce_sum(t: torch.Tensor, world_size: int) -> torch.Tensor:
    """reduce_sum (loss.py:202-208) for both normalisers at once."""
    if world_size <= 1:
        return t
    import torch.distributed as dist
    t = t.clone()
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t


def normalisers(local: torch.Tensor, world_size: int):
    """local = [positives, sum of centerness targets] of this rank (fp64, any device) -> (num_pos_avg_per_gpu, sum_centerness_targets_avg_per_gpu)
    of loss.py:541-556: totals over the ranks / world size, the first clamped to >= 1."""
    total = _all_reduce_sum(local, world_size)
    w = float(max(world_size, 1))
    return torch.clamp(total[0] / w, min=1.0), total[1] / w


def rotated_iou_losses(pred: torch.Tensor, target: torch.Tensor, loss_type: str) -> torch.Tensor:
    """RotatedIOULoss.forward (loss.py:142-170) per box, before the weighted sum: pred / target (K, 8) regression vectors."""
    from ..rotated_iou.oriented_iou_loss import cal_diou_3d, cal_giou_3d, cal_iou_3d
    zero = torch.zeros(pred.shape[0], 3, device=pred.device)
    pb, tb = decode_fcos_obb(zero, pred).unsqueeze(0), decode_fcos_obb(zero, target).unsqueeze(0)
    if loss_type in ("iou", "linear_iou"):
        ious, _, _, _, unions = cal_iou_3d(pb, tb, verbose=True)
        ious = (ious * unions + 1.0) / (unions + 1.0)
        losses = -torch.log(ious) if loss_type == "iou" else 1 - ious
    elif loss_type == "giou":
        losses = cal_giou_3d(pb, tb)[0]
    elif loss_type == "diou":
        losses = cal_diou_3d(pb, tb)[0]
    else:
        raise NotImplementedError(loss_type)
    return losses.squeeze(0)


class _FCOSLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, ev, labels, reg_targets, mask, n_levels, *heads):
        box_cls, box_reg, ctrness = heads[:n_levels], heads[n_levels:2 * n_levels], heads[2 * n_levels:]
        rotated_iou = ev.use_obb and ev.iou_loss_type != "smooth_l1"
        proj2d = ev.use_obb and ev.proj2d_loss_weight > 0
        kernel_type = "iou" if ev.iou_loss_type == "diou" else ev.iou_loss_type          # diou exists for the rotated head only (ignored by the kernel there)
        want_grad = any(ctx.needs_input_grad[5:])
        sums, ct, grads = ops.fcos_loss_sums([t.detach() for t in box_cls], [t.detach() for t in box_reg], [t.detach() for t in ctrness], labels,
                                             reg_targets, mask, kernel_type, ev.use_obb, ev.use_additional_l1_loss, want_grad=want_grad)
        reg_raw = sums[3] + sums[5]
        if rotated_iou or proj2d:
            reg_raw = reg_raw + _FCOSLoss._positives_term(ev, rotated_iou, proj2d, box_reg, labels, reg_targets, mask, ct, grads)
        num_pos_avg, sum_ct_avg = normalisers(torch.stack([sums[1], sums[2]]), ev.world_size)
        loss_cls = sums[0] / num_pos_avg
        loss_ctr = sums[4] / num_pos_avg
        has = sum_ct_avg > 0
        inv_ct = torch.where(has, 1.0 / torch.where(has, sum_ct_avg, torch.ones_like(sum_ct_avg)), torch.zeros_like(sum_ct_avg))
        loss_reg = reg_raw * inv_ct                                                      # no positives anywhere: 0 (loss.py:583-586)
        if want_grad:
            ctx.grads = grads
            ctx.scale = ((1.0 / num_pos_avg).float(), inv_ct.float())
        ctx.n_levels = n_levels
        return loss_cls.float(), loss_reg.float(), loss_ctr.float()

    @staticmethod
    def _positives_term(ev, rotated_iou, proj2d, box_reg, labels, reg_targets, mask, ct, grads):
        """The terms of the OBB head evaluated on the gathered positives: sum_i w_i * RotatedIOULoss_i and / or proj2d_loss_weight * the 2-D
        projection loss; the gradient w.r.t. the 8 regression channels is accumulated into grads[1]."""
        pos = labels > 0 if mask is None else (labels > 0) & (mask != 0)
        idx = torch.nonzero(pos)                                                         # host sync: the positives' count sizes the gather
        if idx.shape[0] == 0:
            return torch.zeros((), dtype=torch.float64, device=labels.device)
        n_idx, q_idx = idx[:, 0], idx[:, 1]
        begin = [0]
        for t in box_reg:
            begin.append(begin[-1] + t[0, 0].numel())
        lvl = torch.bucketize(q_idx, torch.tensor(begin[1:-1], device=q_idx.device), right=True) if len(box_reg) > 1 else torch.zeros_like(q_idx)
        preds, sel = [], []
        for l, t in enumerate(box_reg):
            m = lvl == l
            sel.append(m)
            flat = t.detach().reshape(t.shape[0], 8, -1).permute(0, 2, 1)                # (N, P_l, 8) view of the NCDHW output
            preds.append(flat[n_idx[m], q_idx[m] - begin[l]])
        order = torch.cat([torch.nonzero(m).squeeze(1) for m in sel])                    # positives level by level
        pred = torch.cat(preds).requires_grad_(grads is not None)
        tgt, w = reg_targets[n_idx[order], q_idx[order]], ct[n_idx[order], q_idx[order]]
        with torch.enable_grad():
            raw = pred.sum() * 0
            if rotated_iou:
                raw = raw + (rotated_iou_losses(pred, tgt, ev.iou_loss_type) * w).sum()
            if proj2d:
                zero = torch.zeros(pred.shape[0], 3, device=pred.device)
                raw = raw + ev.proj2d_loss_weight * fcos_projection_loss(decode_fcos_obb(zero, pred), decode_fcos_obb(zero, tgt), w)
            if grads is not None:
                g, = torch.autograd.grad(raw, pred)
        if grads is not None:
            off = 0
            for l, t in enumerate(box_reg):
                k = int(sel[l].sum())                                                    # (already synchronised above)
                if k:
                    o = order[off:off + k]
                    view = grads[1][l].reshape(t.shape[0], 8, -1).permute(0, 2, 1)
                    view.index_put_((n_idx[o], q_idx[o] - begin[l]), g[off:off + k].to(view.dtype), accumulate=True)
                off += k
        return raw.detach().double()

    @staticmethod
    def backward(ctx, g_cls, g_reg, g_ctr):
        n = ctx.n_levels
        dcls, dreg, dctr = ctx.grads
        inv_pos, inv_ct = ctx.scale
        out = [None] * 5
        out += [d * (g_cls * inv_pos) for d in dcls]
        out += [d * (g_reg * inv_ct) for d in dreg]
        out += [d * (g_ctr * inv_pos) for d in dctr]
        assert len(out) == 5 + 3 * n
        return tuple(out)


class FCOSLossComputation(object):
    """This class computes the FCOS losses (3-D, binary objectness) on the CUDA kernels; see the module docstring."""

    def __init__(self, fpn_strides, center_sampling_radius, iou_loss_type, norm_reg_targets, world_size, use_obb, use_additional_l1_loss,
                 proj2d_loss_weight=0.0):
        if iou_loss_type not in ("smooth_l1", "iou", "linear_iou", "giou") and not (use_obb and iou_loss_type == "diou"):
            raise NotImplementedError(f"iou_loss_type {iou_loss_type!r}: the reference implements iou / linear_iou / giou (+ diou for OBB) and smooth_l1")
        if len(fpn_strides) > 4:
            raise NotImplementedError("object_sizes_of_interest has four rows (fcos/loss.py:263-268): at most 4 levels")
        self.fpn_strides = list(fpn_strides)
        self.center_sampling_radius = center_sampling_radius
        self.iou_loss_type = iou_loss_type
        self.norm_reg_targets = norm_reg_targets
        self.world_size = world_size
        self.use_obb = use_obb
        self.use_additional_l1_loss = use_additional_l1_loss
        self.proj2d_loss_weight = proj2d_loss_weight

    # -------------------------------------------------------------------------------------------- targets
    def _targets(self, points: List[torch.Tensor], targets: List[torch.Tensor]):
        """-> labels (N, P) f32, reg_targets (N, P, 6|8) f32, levels concatenated per scene (the kernels' layout)."""
        n_per = [int(p.shape[0]) for p in points]
        self.num_points_per_level = n_per
        loc = torch.cat([p.to(device="cuda", dtype=torch.float32) for p in points], 0).contiguous()
        dim = 7 if self.use_obb else 6
        labels, regs = [], []
        for boxes in targets:
            gt = boxes.to(device=loc.device, dtype=torch.float32).reshape(-1, dim).contiguous()
            lab, reg = ops.fcos_targets(loc, n_per, self.fpn_strides[:len(n_per)], gt, self.center_sampling_radius, self.norm_reg_targets)
            labels.append(lab); regs.append(reg)
        return torch.stack(labels), torch.stack(regs)

    def prepare_targets(self, points, targets):
        """loss.py:262-316: level-first lists -- labels[l] (N * P_l,), reg_targets[l] (N * P_l, 6|8), scenes concatenated inside a level."""
        labels, regs = self._targets(points, targets)
        out_l, out_r, off = [], [], 0
        for pl in self.num_points_per_level:
            out_l.append(labels[:, off:off + pl].reshape(-1))
            out_r.append(regs[:, off:off + pl].reshape(-1, regs.shape[-1]))
            off += pl
        return out_l, out_r

    def compute_centerness_targets(self, reg_targets):
        """loss.py:443-450 (a helper of the reference's API; the loss kernel computes the same per positive)."""
        pairs = [reg_targets[:, [0, 3]], reg_targets[:, [1, 4]], reg_targets[:, [2, 5]]]
        c = [p.min(dim=-1)[0] / p.max(dim=-1)[0] for p in pairs]
        return torch.sqrt(c[0] * c[1] * c[2])

    # -------------------------------------------------------------------------------------------- losses
    def __call__(self, locations, box_cls, box_regression, centerness, targets, padding_masks: Optional[List[torch.Tensor]]):
        """locations: list[(P_l, 3)]; box_cls / box_regression / centerness: list[(N, 1 | 6|8 | 1, w, l, h)] CUDA fp32 (may require grad);
        targets: list[(G_n, 6|7)] per scene; padding_masks: None or list[(N, P_l) bool].  -> cls_loss, reg_loss, centerness_loss (0-d, fp32)."""
        if box_cls[0].size(1) != 1:
            raise AssertionError("binary objectness only (num_classes == 1), like the reference")
        if not all(t.is_cuda for t in list(box_cls) + list(box_regression) + list(centerness)):
            raise RuntimeError("nerf_rpn_b200: FCOSLossComputation needs CUDA tensors (this package has no CPU path)")
        labels, reg_targets = self._targets(locations, targets)
        mask = None
        if padding_masks is not None:
            mask = torch.cat([m.reshape(m.shape[0], -1) for m in padding_masks], 1).to(device=labels.device, dtype=torch.uint8).contiguous()
        heads = [t if t.is_contiguous() else t.contiguous() for t in list(box_cls) + list(box_regression) + list(centerness)]
        heads = [t if t.dtype == torch.float32 else t.float() for t in heads]
        return _FCOSLoss.apply(self, labels, reg_targets, mask, len(box_cls), *heads)
