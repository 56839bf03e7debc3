"""Training step of the anchor RPN on the CUDA kernels (SURVEY.md 8(a) a18, BASELINE config 4).

Mirrors what `losses = model(rgbsigma, boxes); loss.backward(); clip_grad_norm_; optimizer.step()` computes in the reference
  NeRFRegionProposalNetwork.forward (train)   nerf_rpn/model/nerf_rpn.py:166-217
  ResNet_FPN_256.forward / Bottleneck         nerf_rpn/model/feature_extractor.py:48-68,215-235   (BatchNorm3d with batch statistics)
  RegionProposalNetwork.forward (train)       nerf_rpn/model/rpn.py:514-534  (assign targets, sample 256, BCE + smooth-L1)
  Trainer.train_epoch                         nerf_rpn/run_rpn.py:372-412    (AdamW, clip_grad_norm_ 0.1, DDP gradient all-reduce)
as a fixed list of libnerf_rpn_b200 launches:
  forward   conv (wgmma implicit GEMM, raw output) -> batch statistics -> normalise (+ residual) + ReLU, FPN / head as in inference
  backward  per conv: wgrad (wgmma, voxel-major contraction, written straight into the flat fp32 gradient bucket in nn.Conv3d's own
            layout) and dgrad (the forward kernel on mirrored / transposed weights, branch gradients added in its epilogue);
            BatchNorm / ReLU / max-pool / up-sampling backward are bandwidth kernels (csrc/train.cu)
  update    the flat gradient bucket is all-reduced over NCCL in chunks, each launched as soon as the backward pass has produced it
            (head -> FPN -> stage 4..1 -> stem), overlapping the remaining dgrad / wgrad; then global norm, clip and AdamW in one pass.
Parameters live in ONE flat fp32 buffer (the nn.Parameters of the module mirrors are views of it, checkpoints / state_dict unchanged);
16-bit GEMM operands are re-packed from it after every update by a device kernel.

PyTorch here: buffers, streams, torch.distributed (NCCL) and the RNG of the sampler (the reference's own torch.randperm calls).
There is no autograd graph and no eager-PyTorch compute on this path.
"""
import ctypes
import os
import math
from typing import List, Optional, Sequence

import torch

from . import ops, packing
from ._lib import RpnDesc, WgradDesc, check, lib


_TRAIN_GRAPH = os.environ.get("NRPN_TRAIN_GRAPH", "1") != "0"          # static launch lists of the training step replayed as CUDA graphs
_WGRAD_PLANAR = os.environ.get("NRPN_WGRAD_PLANAR", "0") == "1"      # earlier wgrad operand path (transposed staging copies), for A/B runs



def _replay_static(state: dict, name: str, fns, enabled: bool = True):
    """Runs a STATIC launch list (fixed kernels, shapes and pointers): eagerly the first two times -- scratch buffers and workspaces are allocated
    lazily --, then captured once into a CUDA graph and replayed (the ~700 launches of a training step otherwise cost ~5 ms of ctypes calls and
    leave gaps between the many few-microsecond kernels of the deep stages).  A failed capture falls back to eager launches for good."""
    st = state.setdefault(name, {"runs": 0, "graph": None, "failed": False})
    if st["graph"] is not None:
        st["graph"].replay()
        return
    if not (enabled and _TRAIN_GRAPH) or st["failed"] or st["runs"] < 2:
        for f in fns:
            f()
        st["runs"] += 1
        return
    try:
        g = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        with torch.cuda.graph(g):
            for f in fns:
                f()
        st["graph"] = g
        g.replay()
    except Exception:                                         # noqa: BLE001 -- anything that cannot be captured: stay eager
        st["failed"] = True
        torch.cuda.synchronize()
        for f in fns:
            f()


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def _ru(v, m):
    return (v + m - 1) // m * m


def _down(d):
    return tuple((v - 1) // 2 + 1 for v in d)


def bucket_schedule(bwd_lo: Sequence[int], n_params: int, bucket_elems: int):
    """All-reduce ranges of the flat gradient bucket, in launch order.  bwd_lo[i] = lowest flat offset that is final once backward stage i
    (construction order: stem, blocks..., FPN, head) has run; stages execute in REVERSE, so gradients become final from the end of the bucket
    towards its start.  A range [lo, hi) is launched after a stage as soon as at least bucket_elems new elements are final (or the bucket is
    complete).  Returns [(stage index in execution order, lo, hi)]: disjoint, covering [0, n_params) exactly once."""
    out, hi = [], n_params
    for k, lo in enumerate(reversed(list(bwd_lo))):
        if hi > lo and (hi - lo >= bucket_elems or lo == 0):
            out.append((k, lo, hi))
            hi = lo
    return out


class _TConv:
    """One trainable convolution: views of the master weight (+ bias), its 16-bit forward / data-gradient operands and tap table."""

    def __init__(self, eng, conv: torch.nn.Conv3d, need_dgrad=True, stem=False):
        self.eng = eng
        self.weight, self.bias = conv.weight, conv.bias
        cout, cin, k = conv.weight.shape[0], conv.weight.shape[1], conv.weight.shape[2]
        self.cout, self.cin_real, self.k = cout, cin, k
        self.stride = conv.stride[0]
        dt, dev = eng.act_dtype, eng.device
        self.stem = stem
        if stem:
            probe = torch.arange(1, conv.weight.numel() + 1, dtype=torch.float32).view_as(conv.weight)
            wp, taps = packing.pack_stem_weight(probe, None, dtype=torch.float32)                  # (32, 64, 64): source index + 1, 0 = structural zero
            self.taps = taps
            self.cin, self.cout_pad = 64, 64
            self.gather_idx = (wp.reshape(-1).to(torch.int64) - 1).to(torch.int32).to(dev)       # packed position -> master index
            inv = torch.full((conv.weight.numel(),), -1, dtype=torch.int32)
            pos = torch.nonzero(wp.reshape(-1) > 0).reshape(-1)
            inv[(wp.reshape(-1)[pos] - 1).to(torch.int64)] = pos.to(torch.int32)
            assert int((inv < 0).sum()) == 0
            self.scatter_idx = inv.to(dev)                                                        # master index -> packed position
            self.fwd = torch.zeros((len(taps), 64, 64), dtype=dt, device=dev)
            self.bwd = None
            self.stride = 1
        else:
            self.taps = [(a - k // 2, b - k // 2, c - k // 2) for a in range(k) for b in range(k) for c in range(k)]
            self.cin = _ru(cin, 64)
            c8 = _ru(cout, 8)
            self.cout_pad = _ru(c8, packing.conv_block_n(c8))
            self.fwd = torch.zeros((len(self.taps), self.cout_pad, self.cin), dtype=dt, device=dev)
            self.bwd = None
            if need_dgrad:
                n8 = _ru(cin, 8)
                self.bwd_rows = _ru(n8, packing.conv_block_n(n8))
                self.bwd_cols = _ru(cout, 64)
                self.bwd = torch.zeros((len(self.taps), self.bwd_rows, self.bwd_cols), dtype=dt, device=dev)
                self.bwd_shift = torch.zeros(self.bwd_rows, dtype=torch.float32, device=dev)
        self.zero_shift = torch.zeros(self.cout_pad, dtype=torch.float32, device=dev)

    @property
    def shift(self):
        # a bias of 8-multiple length is read in place by the conv epilogue (it only touches channels < cout)
        if self.bias is not None and self.cout % 8 == 0:
            return self.bias.data
        return self.zero_shift

    def repack(self):
        f16 = 1 if self.eng.act_dtype == torch.float16 else 0
        L = lib()
        if self.stem:
            check(L.nrpn_gather_pack(_p(self.weight.data), _p(self.gather_idx), self.gather_idx.numel(), _p(self.fwd), None, 1.0, f16, _stream()),
                  "gather_pack(stem)")
            return
        taps = len(self.taps)
        check(L.nrpn_pack_weights(_p(self.weight.data), self.cout, self.cin_real, taps, _p(self.fwd), self.cout_pad, self.cin,
                                  _p(self.bwd), 0 if self.bwd is None else self.bwd_rows, 0 if self.bwd is None else self.bwd_cols, f16, _stream()),
              "pack_weights")


class _BN:
    def __init__(self, eng, bn: torch.nn.BatchNorm3d):
        self.m = bn
        c = bn.num_features
        self.c = c
        assert bn.bias.data_ptr() == bn.weight.data_ptr() + 4 * c, "bn.weight / bn.bias must be adjacent in the flat parameter buffer"
        self.stats = torch.zeros(3 * c, dtype=torch.float32, device=eng.device)


class RPNTrainEngine:
    """Forward + backward + update for ResNet_FPN_256 + RPNHead (+ RegionProposalNetwork hyper-parameters)."""

    def __init__(self, model, precision: str = "bf16", lr: float = 1e-4, weight_decay: float = 0.01, betas=(0.9, 0.999), eps: float = 1e-8,
                 clip_grad_norm: float = 0.1, reg_loss_weight: float = 5.0, process_group=None, bucket_mb: float = 32.0,
                 loss_scale: Optional[float] = None, seed: Optional[int] = None, reg_loss_weight_2d: float = 0.0):
        if precision not in ("bf16", "fp16"):
            raise ValueError("training runs with bf16 (default) or fp16 (with a static loss scale) 16-bit activations / gradients")
        bb, rpn = model.backbone, model.rpn
        if type(bb).__name__ != "ResNet_FPN_256":
            raise NotImplementedError("nerf_rpn_b200: the training engine implements ResNet_FPN_256 + RPNHead (BASELINE config 4)")
        if rpn.reg_loss_type not in ("smooth_l1", "iou", "linear_iou", "giou", "diou"):
            raise NotImplementedError(f"nerf_rpn_b200: unknown reg_loss_type {rpn.reg_loss_type!r}")
        if rpn.reg_loss_type != "smooth_l1" and not rpn.rotate:
            raise NotImplementedError("nerf_rpn_b200: the IoU-type regression losses exist for --rotated_bbox only (as in the reference, rpn.py:216-217)")
        self.reg_loss_type = rpn.reg_loss_type
        self.model, self.bb, self.head, self.rpn = model, bb, rpn.head, rpn
        self.device = next(bb.parameters()).device
        if self.device.type != "cuda":
            raise RuntimeError("nerf_rpn_b200: training needs the model on a CUDA device (no CPU path)")
        self.precision = precision
        self.act_dtype = torch.float16 if precision == "fp16" else torch.bfloat16
        self.f16 = 1 if precision == "fp16" else 0
        self.loss_scale = float(loss_scale) if loss_scale is not None else (1024.0 if precision == "fp16" else 1.0)
        self.lr, self.wd, self.betas, self.eps, self.clip = lr, weight_decay, betas, eps, clip_grad_norm
        self.w_reg = reg_loss_weight
        self.w_2d = reg_loss_weight_2d      # --reg_loss_weight_2d (run_rpn.py:91, default 0): the 2-D projection loss is evaluated only when it is non-zero
        self.pg = process_group
        self.world = torch.distributed.get_world_size(process_group) if (process_group is not None or
                                                                         (torch.distributed.is_available() and torch.distributed.is_initialized())) else 1
        self.step_count = 0
        self.rotated = rpn.rotate
        self.code = 8 if self.rotated else 6
        ag = rpn.anchor_generator
        self.cells = ag.cell_anchors_np()
        self.A = ag.num_anchors_per_location()[0]
        self._flatten_parameters()
        self._build_layers()
        self.bucket_elems = int(bucket_mb * (1 << 20) / 4)
        self._plans = {}
        self._graphs = {}                      # captured static launch lists (repack)
        self.comm_stream = torch.cuda.Stream(device=self.device)
        self._norm = torch.zeros(1, dtype=torch.float32, device=self.device)
        self._norm_ws = torch.empty(lib().nrpn_grad_norm_workspace_bytes(), dtype=torch.uint8, device=self.device)
        self._red_ws = torch.empty(lib().nrpn_chan_reduce_workspace_bytes(2048), dtype=torch.uint8, device=self.device)
        self.losses = torch.zeros(2, dtype=torch.float32, device=self.device)
        self.loss_2d = torch.zeros((), dtype=torch.float32, device=self.device)        # loss_rpn_box_reg_2d (unweighted), when evaluated
        self.overlap_allreduce = True       # False: leave the gradient all-reduce to the caller (DDP wrapping the autograd compat path)
        self.gen = None
        if seed is not None:
            self.gen = torch.Generator(device=self.device); self.gen.manual_seed(seed)
        self.repack()

    # ------------------------------------------------------------------------------------------------ parameters
    def _flatten_parameters(self):
        """All parameters of backbone + head as views of one flat fp32 buffer, in BACKWARD-COMPLETION order reversed (module order):
        the gradient bucket of the layers that finish first in the backward pass (head, FPN) sits at the END of the buffer."""
        params = list(self.bb.parameters()) + list(self.head.parameters())
        total = sum(p.numel() for p in params)
        self.flat_p = torch.empty(total, dtype=torch.float32, device=self.device)
        self.flat_g = torch.zeros(total, dtype=torch.float32, device=self.device)
        self.flat_m = torch.zeros(total, dtype=torch.float32, device=self.device)
        self.flat_v = torch.zeros(total, dtype=torch.float32, device=self.device)
        off = 0
        self.offsets = {}
        for p in params:
            n = p.numel()
            self.flat_p[off:off + n].copy_(p.data.reshape(-1))
            p.data = self.flat_p[off:off + n].view(p.shape)
            self.offsets[id(p)] = (off, n)
            off += n
        self.n_params = total
        self._params = params
        self._packed_ver = None

    def sync_parameters(self):
        """Drop-in path (torch optimiser / load_state_dict between steps): re-point parameters that were re-materialised back into the flat
        buffer and re-pack the 16-bit operands when any master weight changed since the last packing."""
        ver = tuple(p._version for p in self._params)
        moved = False
        for p in self._params:
            off, n = self.offsets[id(p)]
            if p.data.data_ptr() != self.flat_p.data_ptr() + 4 * off:
                self.flat_p[off:off + n].copy_(p.data.reshape(-1)); p.data = self.flat_p[off:off + n].view(p.shape); moved = True
        if moved or ver != self._packed_ver:
            self.repack()

    def grad_of(self, p):
        off, n = self.offsets[id(p)]
        return self.flat_g[off:off + n]

    def _build_layers(self):
        bb, hd = self.bb, self.head
        self.stem = _TConv(self, bb.conv1, need_dgrad=False, stem=True)
        self.stem_bn = _BN(self, bb.bn1)
        self.blocks = []
        for stage in bb.layers:
            for blk in stage:
                e = dict(c1=_TConv(self, blk.conv1), bn1=_BN(self, blk.bn1), c2=_TConv(self, blk.conv2), bn2=_BN(self, blk.bn2),
                         c3=_TConv(self, blk.conv3), bn3=_BN(self, blk.bn3), ds=None, bnd=None, stride=blk.stride)
                if blk.downsample is not None:
                    e["ds"] = _TConv(self, blk.downsample[0]); e["bnd"] = _BN(self, blk.downsample[1])
                self.blocks.append(e)
        self.lat = [_TConv(self, m) for m in bb.latlayers]
        self.smooth = [_TConv(self, m) for m in bb.smooths]
        self.hconv = [_TConv(self, m) for m in hd.conv if isinstance(m, torch.nn.Conv3d)]
        # fused cls | bbox predictor (anchor.py:196-198): one 1^3 GEMM with 128 (padded) output channels
        self.n_pred = self.A * (1 + self.code)
        if self.n_pred > 128:
            raise ValueError("fused predictor supports at most 128 output channels")
        dt = self.act_dtype
        self.pred_fwd = torch.zeros((1, 128, 256), dtype=dt, device=self.device)
        self.pred_bwd = torch.zeros((1, 256, 128), dtype=dt, device=self.device)
        self.pred_shift = torch.zeros(128, dtype=torch.float32, device=self.device)
        self.pred_bwd_shift = torch.zeros(256, dtype=torch.float32, device=self.device)
        self.pred_w32 = torch.zeros((128, 256), dtype=torch.float32, device=self.device)
        self.pred_dw = torch.zeros((128, 256), dtype=torch.float32, device=self.device)
        self.pred_db = torch.zeros(128, dtype=torch.float32, device=self.device)
        self.all_convs = [self.stem] + [e[k] for e in self.blocks for k in ("c1", "c2", "c3", "ds") if e[k] is not None] + self.lat + self.smooth + self.hconv

    def repack(self):
        """fp32 master weights -> 16-bit GEMM operands (after every optimiser step / checkpoint load)."""
        self._packed_ver = tuple(p._version for p in self._params)
        _replay_static(self._graphs, "repack", [self._repack_launches])

    def _repack_launches(self):
        for c in self.all_convs:
            c.repack()
        hd, A = self.head, self.A
        self.pred_w32[:A].copy_(hd.cls_logits.weight.data.view(A, 256))
        self.pred_w32[A:self.n_pred].copy_(hd.bbox_pred.weight.data.view(-1, 256))
        self.pred_shift[:A].copy_(hd.cls_logits.bias.data); self.pred_shift[A:self.n_pred].copy_(hd.bbox_pred.bias.data)
        check(lib().nrpn_pack_weights(_p(self.pred_w32), 128, 256, 1, _p(self.pred_fwd), 128, 256, _p(self.pred_bwd), 256, 128, self.f16, _stream()),
              "pack_weights(pred)")

    # ------------------------------------------------------------------------------------------------ plan
    def plan(self, n, dims):
        key = (n, tuple(dims))
        p = self._plans.get(key)
        if p is None:
            p = _TrainPlan(self, n, tuple(dims))
            self._plans[key] = p
        return p

    # ------------------------------------------------------------------------------------------------ step
    def forward_backward(self, grids: torch.Tensor, targets: Sequence[torch.Tensor]):
        """grids (N,4,X,Y,Z) fp32 CUDA, targets: N tensors (G,6|7).  Runs forward, losses, backward (+ the overlapped gradient
        all-reduce when a process group is active).  Returns the loss tensor (2,) = [loss_objectness, loss_rpn_box_reg] (device)."""
        n, c, X, Y, Z = grids.shape
        plan = self.plan(n, (X, Y, Z))
        plan.run(grids, targets)
        return self.losses

    def optimizer_step(self, lr: Optional[float] = None):
        """clip_grad_norm_(clip) + AdamW on the flat buffers (after the all-reduce has drained), then re-pack the 16-bit operands."""
        torch.cuda.current_stream().wait_stream(self.comm_stream)
        self.step_count += 1
        inv = 1.0 / (self.loss_scale * self.world)
        L = lib()
        check(L.nrpn_grad_norm(_p(self.flat_g), self.n_params, inv, _p(self._norm), _p(self._norm_ws), self._norm_ws.numel(), _stream()), "grad_norm")
        check(L.nrpn_adamw_step(_p(self.flat_p), _p(self.flat_g), _p(self.flat_m), _p(self.flat_v), self.n_params, _p(self._norm), float(self.clip),
                                inv, float(self.lr if lr is None else lr), self.betas[0], self.betas[1], self.eps, self.wd, self.step_count, _stream()),
              "adamw_step")
        self.repack()

    def train_step(self, grids, targets, lr: Optional[float] = None):
        losses = self.forward_backward(grids, targets)
        self.optimizer_step(lr)
        return losses


class _TrainPlan:
    """Buffers and the launch lists (forward, backward) for n scenes of one size."""

    def __init__(self, eng: RPNTrainEngine, n: int, dims):
        self.eng, self.n, self.dims = eng, n, dims
        dev, dt = eng.device, eng.act_dtype
        self.fwd: List = []
        self.bwd: List = []                      # built in forward order, executed reversed
        self.bwd_lo: List[int] = []              # lowest flat-parameter offset whose gradient is final once bwd[i] has run
        self.f16 = eng.f16
        self._scratch = {}
        self._graphs = {}
        self._ws = None
        X, Y, Z = dims
        L = lib()

        def buf(d, c, dtype=dt, zero=False):
            f = torch.zeros if zero else torch.empty
            return f((n, *d, c), dtype=dtype, device=dev)

        self.input = None
        d1 = _down(dims)
        self.packed = torch.empty((n, d1[0], d1[1], d1[2] + 1, 64), dtype=dt, device=dev)
        self.fwd.append(lambda: ops.pack_stem_input(self._src, self.packed))
        y0 = buf(d1, 64); a0 = buf(d1, 64)
        self._conv_fwd(eng.stem, self.packed, (d1[0], d1[1], d1[2] + 1), y0, d1)
        self._bn_fwd(eng.stem_bn, y0, None, a0, True)
        d2 = _down(d1)
        p0 = buf(d2, 64)
        self.pool_idx = torch.empty((n, *d2, 64), dtype=torch.uint8, device=dev)
        self.fwd.append(lambda: check(L.nrpn_maxpool3d_k3s2_argmax(_p(a0), n, d1[0], d1[1], d1[2], 64, _p(p0), _p(self.pool_idx), self.f16, _stream()), "maxpool_argmax"))
        dp0 = buf(d2, 64)                          # gradient w.r.t. the pooled map
        da0 = buf(d1, 64); dy0 = buf(d1, 64)

        # backward of the stem (runs LAST): pool backward -> BN backward -> stem wgrad (on the packed input)
        def stem_bwd():
            check(L.nrpn_maxpool3d_k3s2_backward(_p(dp0), _p(self.pool_idx), n, d1[0], d1[1], d1[2], 64, _p(da0), self.f16, _stream()), "maxpool_backward")
            self._bn_bwd(eng.stem_bn, da0, a0, y0, dy0, None, True)
            self._wgrad_stem(dy0, d1)
        self.bwd.append(stem_bwd)
        self.bwd_lo.append(0)

        # ---- bottom-up
        x, xd, dx = p0, d2, dp0                    # block input, its dims, and the buffer that receives its gradient
        c_out = []
        bi = 0
        for si, stage in enumerate(eng.bb.layers):
            for _ in stage:
                e = eng.blocks[bi]; bi += 1
                s = e["stride"]
                od = _down(xd) if s == 2 else xd
                planes, outc = e["c1"].cout, e["c3"].cout
                y1, a1 = buf(od, planes), buf(od, planes)
                y2, a2 = buf(od, planes), buf(od, planes)
                y3, out = buf(od, outc), buf(od, outc)
                self._conv_fwd(e["c1"], x, xd, y1, od)
                self._bn_fwd(e["bn1"], y1, None, a1, True)
                self._conv_fwd(e["c2"], a1, od, y2, od)
                self._bn_fwd(e["bn2"], y2, None, a2, True)
                self._conv_fwd(e["c3"], a2, od, y3, od)
                if e["ds"] is not None:
                    yd, r = buf(od, outc), buf(od, outc)
                    self._conv_fwd(e["ds"], x, xd, yd, od)
                    self._bn_fwd(e["bnd"], yd, None, r, False)
                else:
                    yd, r = None, x
                self._bn_fwd(e["bn3"], y3, r, out, True)
                dout = buf(od, outc)               # gradient w.r.t. the block output (filled by the consumer's backward)
                # the input of the first block of stages 1..3 is a stage output that also feeds an FPN lateral: fpn_bwd (which runs
                # earlier in the backward pass) has already written the lateral part into dx, so this block ADDS its data gradient
                add_lateral = (si > 0 and _ is stage[0])
                self.bwd.append(self._make_block_bwd(e, x, xd, dx, od, y1, a1, y2, a2, y3, out, yd, dout, s, add_lateral))
                self.bwd_lo.append(min(eng.offsets[id(p_)][0] for k_ in ("c1", "c2", "c3", "ds") if e[k_] is not None for p_ in [e[k_].weight]))
                x, xd, dx = out, od, dout
            c_out.append((x, xd, dx))

        # ---- FPN top-down (feature_extractor.py:224-235)
        (c5, d5, dc5) = c_out[-1]
        q = [None] * 4; dq = [None] * 4; qd = [None] * 4
        q[0] = buf(d5, 256); dq[0] = buf(d5, 256); qd[0] = d5
        self._conv_fwd(eng.lat[0], c5, d5, q[0], d5)
        for i in range(1, 4):
            (c, cd, _) = c_out[-1 - i]
            q[i] = buf(cd, 256); dq[i] = buf(cd, 256); qd[i] = cd
            self._conv_fwd(eng.lat[i], c, cd, q[i], cd, res=q[i - 1], res_dims=qd[i - 1])
        feats, dfeats, fdims = [q[0]], [dq[0]], [d5]           # P5 = q5 (no smooth conv); its gradient accumulates in dq[0]
        for i, sm in enumerate(eng.smooth):
            f = buf(qd[i + 1], 256); df = buf(qd[i + 1], 256)
            self._conv_fwd(sm, q[i + 1], qd[i + 1], f, qd[i + 1])
            feats.append(f); dfeats.append(df); fdims.append(qd[i + 1])
        feats.reverse(); dfeats.reverse(); fdims.reverse()      # [P2, P3, P4, P5]
        self.features, self.feat_dims = feats, fdims

        # FPN backward (executed after the head's backward): smooth convs, top-down merge, laterals
        def fpn_bwd():
            # dfeats = [dP2, dP3, dP4, dP5(=dq[0])]
            for i in (2, 1, 0):                                 # smooth[i] acts on q[i+1]; finest level first
                lvl_feat = 2 - i                                # index into feats / dfeats ([P2,P3,P4,P5]): smooth[2]->P2, [1]->P3, [0]->P4
                self._conv_bwd(eng.smooth[i], q[i + 1], qd[i + 1], dfeats[lvl_feat], qd[i + 1], dq[i + 1], bias=True)
                if i < 2:                                       # the finer level's merged map took up(q[i+1]) as its residual
                    fd, cd_ = qd[i + 2], qd[i + 1]
                    check(L.nrpn_upsample_nearest_backward(_p(dq[i + 2]), n, fd[0], fd[1], fd[2], cd_[0], cd_[1], cd_[2], 256, _p(dq[i + 1]), 1, self.f16, _stream()),
                          "upsample_backward")
            fd, cd_ = qd[1], qd[0]
            check(L.nrpn_upsample_nearest_backward(_p(dq[1]), n, fd[0], fd[1], fd[2], cd_[0], cd_[1], cd_[2], 256, _p(dq[0]), 1, self.f16, _stream()),
                  "upsample_backward")
            for i in range(4):
                (c, cd, dc) = c_out[-1 - i]
                self._conv_bwd(eng.lat[i], c, cd, dq[i], cd, dc, bias=True)      # dc = gradient of the stage output from the lateral branch
        # NOTE: the stage outputs c2..c4 also receive the next stage's data gradient: _make_block_bwd ADDS into dx for the first block
        # of stages 1..3 (flag below), because fpn_bwd (which runs earlier) has already written the lateral part.
        self.bwd.append(fpn_bwd)
        self.bwd_lo.append(min(eng.offsets[id(c.weight)][0] for c in eng.lat + eng.smooth))

        # ---- head: all levels in one launch per layer, activations of all levels in ONE buffer (bias gradients are one reduction)
        vox = [d[0] * d[1] * d[2] for d in fdims]
        self.total_vox = n * sum(vox)

        def level_views(t):
            out, o = [], 0
            for d, v in zip(fdims, vox):
                out.append(t[o:o + n * v].view(n, *d, t.shape[-1])); o += n * v
            return out
        hs = [torch.empty((self.total_vox, 256), dtype=dt, device=dev) for _ in eng.hconv]
        dhs = [torch.empty((self.total_vox, 256), dtype=dt, device=dev) for _ in eng.hconv]
        self.pred = torch.empty((self.total_vox, 128), dtype=torch.float32, device=dev)
        self.dpred = torch.zeros((self.total_vox, 128), dtype=dt, device=dev)
        cur = feats
        for k, layer in enumerate(eng.hconv):
            nxt = level_views(hs[k])
            self._conv_fwd_levels(layer.fwd, layer.shift, layer.taps, 256, 256, cur, nxt, fdims, relu=True)
            cur = nxt
        self._conv_fwd_levels(eng.pred_fwd, eng.pred_shift, [(0, 0, 0)], 256, 128, cur, level_views(self.pred), fdims, relu=False, out_fp32=True)
        self.pred_levels = level_views(self.pred)
        self.dbg = dict(hs=[level_views(h) for h in hs], dhs=[level_views(h) for h in dhs], dfeats=dfeats, q=q, dq=dq, c_out=c_out)   # tools/debug_train.py
        self.dpred_levels = level_views(self.dpred)
        self.strides = [tuple(dims[k] // d[k] for k in range(3)) for d in fdims]

        def head_bwd():
            h_last = level_views(hs[-1])
            # predictor: wgrad / bias grad into scratch (cls and bbox rows are separate parameters), dgrad -> dh4
            self._wgrad(self.dpred_levels, h_last, fdims, [(0, 0, 0)], 128, 256, eng.pred_dw, layout=0)
            ws = self._workspace(L.nrpn_bias_grad_workspace_bytes(128))
            check(L.nrpn_bias_grad(_p(self.dpred), self.total_vox, 128, 128, self.f16, _p(eng.pred_db), _p(ws), ws.numel(), _stream()), "bias_grad")
            A, hd = eng.A, eng.head
            eng.grad_of(hd.cls_logits.weight).copy_(eng.pred_dw[:A].reshape(-1)); eng.grad_of(hd.bbox_pred.weight).copy_(eng.pred_dw[A:eng.n_pred].reshape(-1))
            eng.grad_of(hd.cls_logits.bias).copy_(eng.pred_db[:A]); eng.grad_of(hd.bbox_pred.bias).copy_(eng.pred_db[A:eng.n_pred])
            self._conv_fwd_levels(eng.pred_bwd, eng.pred_bwd_shift, [(0, 0, 0)], 128, 256, self.dpred_levels, level_views(dhs[-1]), fdims, relu=False, run=True)
            for k in range(len(eng.hconv) - 1, -1, -1):
                layer = eng.hconv[k]
                check(L.nrpn_relu_backward(_p(dhs[k]), _p(hs[k]), dhs[k].numel(), self.f16, _stream()), "relu_backward")
                xin = feats if k == 0 else level_views(hs[k - 1])
                self._wgrad(level_views(dhs[k]), xin, fdims, layer.taps, 256, 256, eng.grad_of(layer.weight), layout=1)
                ws = self._workspace(L.nrpn_bias_grad_workspace_bytes(256))
                check(L.nrpn_bias_grad(_p(dhs[k]), self.total_vox, 256, 256, self.f16, _p(eng.grad_of(layer.bias)), _p(ws), ws.numel(), _stream()), "bias_grad")
                dst = dfeats if k == 0 else level_views(dhs[k - 1])
                self._conv_fwd_levels(layer.bwd, layer.bwd_shift, layer.taps, 256, 256, level_views(dhs[k]), dst, fdims, relu=False, run=True)
        self.bwd.append(head_bwd)
        self.bwd_lo.append(min(eng.offsets[id(p_)][0] for p_ in eng.head.parameters()))
        self._src = None
        self.anchors = None

    # ------------------------------------------------------------------------------------------------ helpers
    def _workspace(self, nbytes):
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = torch.empty(max(int(nbytes), 1 << 20), dtype=torch.uint8, device=self.eng.device)
        return self._ws

    def _scratch_buf(self, name, numel, dtype):
        t = self._scratch.get(name)
        if t is None or t.numel() < numel or t.dtype != dtype:
            t = torch.empty(int(numel), dtype=dtype, device=self.eng.device)
            self._scratch[name] = t
        return t[:numel]

    def _conv_call(self, w, shift, taps, cin, cout, levels, stride=1, relu=False, out_fp32=False):
        ops.conv3d_fprop(levels, w, shift, cin, cout, taps, stride=stride, relu=relu, out_fp32=out_fp32)

    def _conv_fwd(self, layer: _TConv, x, xd, y, od, res=None, res_dims=None, relu=False):
        n = self.n
        args = [ops.ConvLevelArgs(x, y, n, xd, od, y.shape[-1], res=res, res_dims=res_dims, ldr=0 if res is None else res.shape[-1])]
        self.fwd.append(lambda: self._conv_call(layer.fwd, layer.shift, layer.taps, layer.cin, y.shape[-1], args, stride=layer.stride, relu=relu))

    def _conv_fwd_levels(self, w, shift, taps, cin, cout, xs, ys, dims_l, relu, out_fp32=False, run=False):
        n = self.n
        args = [ops.ConvLevelArgs(xs[i], ys[i], n, dims_l[i], dims_l[i], ys[i].shape[-1]) for i in range(len(xs))]
        f = lambda: self._conv_call(w, shift, taps, cin, cout, args, relu=relu, out_fp32=out_fp32)
        if run:
            f()
        else:
            self.fwd.append(f)

    def _bn_fwd(self, bn: _BN, y, res, out, relu):
        rows = y.numel() // bn.c
        m = bn.m
        L = lib()

        def f():
            ws = self.eng._red_ws
            check(L.nrpn_bn_stats(_p(y), rows, bn.c, self.f16, float(m.eps), _p(bn.stats), _p(m.running_mean), _p(m.running_var),
                                  float(m.momentum if m.momentum is not None else 0.1), _p(ws), ws.numel(), _stream()), "bn_stats")
            check(L.nrpn_bn_apply(_p(y), _p(res), _p(out), rows, bn.c, _p(bn.stats), _p(m.weight.data), _p(m.bias.data), int(relu), self.f16, _stream()), "bn_apply")
        self.fwd.append(f)

    def _bn_bwd(self, bn: _BN, dout, act, y, dy, dres, relu):
        rows = y.numel() // bn.c
        ws = self.eng._red_ws
        sums = self.eng.grad_of(bn.m.weight)           # {dgamma[c], dbeta[c]}: bn.weight.grad | bn.bias.grad are adjacent in the flat bucket
        check(lib().nrpn_bn_backward(_p(dout), _p(act), _p(y), _p(dy), _p(dres), rows, bn.c, _p(bn.stats), _p(bn.m.weight.data), _p(sums), int(relu),
                                     self.f16, _p(ws), ws.numel(), _stream()), "bn_backward")

    def _planar(self, name, x, zp, z_shift, z_logical=None):
        """channels-last (n,X,Y,Z,C) -> planar (n,C,X,Y,zp) in a zero-filled scratch buffer."""
        n, X, Y, Z, C = x.shape
        buf = self._scratch_buf(name, n * C * X * Y * zp, x.dtype)
        buf.zero_()
        check(lib().nrpn_transpose_to_planar(_p(x), n, X, Y, Z, C, C, _p(buf), zp, int(z_shift), _stream()), "transpose_to_planar")
        return buf

    def _wgrad(self, dys, xs, dims_l, taps, cout, cin, dw, layout, z_extra=0, accumulate=False):
        """dW of a stride-1 'same' conv from per-level channels-last (dY, X) pairs, written to `dw` (fp32) in `layout`."""
        d = WgradDesc()
        d.cout, d.cin, d.n_taps = int(cout), int(cin), len(taps)
        for t, off in enumerate(taps):
            for k in range(3):
                d.tap_off[t][k] = int(off[k])
        dzs = sorted({int(off[2]) for off in taps})
        d.n_levels = len(dys)
        if not _WGRAD_PLANAR:                       # operands where they live: channels-last tensors through MN-major descriptors
            for i, (dy, x) in enumerate(zip(dys, xs)):
                lv = d.level[i]
                lv.dy_cl, lv.x_cl, lv.ld_dy, lv.ld_x = dy.data_ptr(), x.data_ptr(), int(dy.shape[-1]), int(x.shape[-1])
                lv.n, lv.x, lv.y, lv.z = int(dy.shape[0]), int(dy.shape[1]), int(dy.shape[2]), int(dy.shape[3])
                lv.xx, lv.xy, lv.xz = int(x.shape[1]), int(x.shape[2]), int(x.shape[3])
            d.operand_layout = 1
        for i, (dy, x) in enumerate(zip(dys, xs) if _WGRAD_PLANAR else ()):
            n, X, Y, Zx = x.shape[0], x.shape[1], x.shape[2], x.shape[3]
            zl = max(Zx, dy.shape[3])
            zp = _ru(zl + 1, 8)
            pdy = self._planar(f"pdy{i}", dy, zp, 0)
            lv = d.level[i]
            lv.dy_planar = pdy.data_ptr()
            for z in dzs:
                lv.x_planar[z + 1] = self._planar(f"px{i}_{z}", x, zp, z).data_ptr()
            lv.n, lv.x, lv.y, lv.z, lv.z_pitch = int(n), int(X), int(Y), int(zl), int(zp)
        d.act_fp16 = self.f16
        d.dw_layout, d.accumulate = int(layout), int(bool(accumulate))
        need = lib().nrpn_conv3d_wgrad_workspace_bytes(ctypes.byref(d))
        if need == 0:
            raise ValueError(f"conv3d_wgrad: unsupported shape cout={cout} cin={cin}")
        ws = self._workspace(need)
        d.dw, d.workspace, d.workspace_bytes = dw.data_ptr(), ws.data_ptr(), ws.numel()
        check(lib().nrpn_conv3d_wgrad(ctypes.byref(d), _stream()), "conv3d_wgrad")

    def _wgrad_stem(self, dy0, d1):
        eng = self.eng
        st = eng.stem
        dwp = self._scratch_buf("stem_dw", len(st.taps) * 64 * 64, torch.float32)
        self._wgrad([dy0], [self.packed], [d1], st.taps, 64, 64, dwp, layout=0)
        g = eng.grad_of(st.weight)
        check(lib().nrpn_gather_pack(_p(dwp), _p(st.scatter_idx), g.numel(), None, _p(g), 1.0, self.f16, _stream()), "gather_pack(stem grad)")

    def _conv_bwd(self, layer: _TConv, x, xd, dy, od, dx, bias=False, dx_res=None, accumulate_dx=False):
        """wgrad (+ bias grad) of a stride-1 layer and its data gradient into dx (optionally + dx_res through the conv epilogue)."""
        eng, L, n = self.eng, lib(), self.n
        self._wgrad([dy], [x], [od], layer.taps, layer.cout, layer.cin_real, eng.grad_of(layer.weight), layout=1)
        if bias:
            ws = self._workspace(L.nrpn_bias_grad_workspace_bytes(layer.cout))
            rows = dy.numel() // layer.cout
            check(L.nrpn_bias_grad(_p(dy), rows, layer.cout, layer.cout, self.f16, _p(eng.grad_of(layer.bias)), _p(ws), ws.numel(), _stream()), "bias_grad")
        if dx is not None:
            args = [ops.ConvLevelArgs(dy, dx, n, od, xd, dx.shape[-1], res=dx_res, res_dims=None if dx_res is None else xd,
                                      ldr=0 if dx_res is None else dx_res.shape[-1])]
            self._conv_call(layer.bwd, layer.bwd_shift, layer.taps, layer.bwd_cols, dx.shape[-1], args)

    def _make_block_bwd(self, e, x, xd, dx, od, y1, a1, y2, a2, y3, out, yd, dout, s, add_lateral):
        eng, L, n = self.eng, lib(), self.n
        planes, outc, cin = e["c1"].cout, e["c3"].cout, e["c1"].cin_real
        dt, dev = eng.act_dtype, eng.device

        def f():
            g = self._scratch_buf("g_skip", out.numel(), dt).view_as(out)        # masked gradient of the block output = skip-branch gradient
            dy3 = self._scratch_buf("dy3", y3.numel(), dt).view_as(y3)
            self._bn_bwd(e["bn3"], dout, out, y3, dy3, g, True)
            da2 = self._scratch_buf("da2", a2.numel(), dt).view_as(a2)
            self._conv_bwd(e["c3"], a2, od, dy3, od, da2)
            dy2 = self._scratch_buf("dy2", y2.numel(), dt).view_as(y2)
            self._bn_bwd(e["bn2"], da2, a2, y2, dy2, None, True)
            da1 = self._scratch_buf("da1", a1.numel(), dt).view_as(a1)
            self._conv_bwd(e["c2"], a1, od, dy2, od, da1)
            dy1 = self._scratch_buf("dy1", y1.numel(), dt).view_as(y1)
            self._bn_bwd(e["bn1"], da1, a1, y1, dy1, None, True)
            if s == 1:
                xs = x
            else:                                                               # stride-2 1^3 convs read the even voxels of x
                xs = self._scratch_buf("x_s2", n * od[0] * od[1] * od[2] * cin, dt).view(n, *od, cin)
                check(L.nrpn_stride2(_p(x), _p(xs), n, xd[0], xd[1], xd[2], cin, 0, _stream()), "stride2 gather")
            # dx accumulates: [lateral branch, already written by fpn_bwd for stage outputs] + skip / downsample branch + conv1 branch
            if e["ds"] is None:
                # identity skip: dx = dgrad_c1(dy1) + g   (stride 1 always)
                self._wgrad([dy1], [xs], [od], e["c1"].taps, planes, cin, eng.grad_of(e["c1"].weight), layout=1)
                tgt = dx if not add_lateral else self._scratch_buf("dx_tmp", dx.numel(), dt).view_as(dx)
                args = [ops.ConvLevelArgs(dy1, tgt, n, od, od, cin, res=g, res_dims=od, ldr=outc)]
                self._conv_call(e["c1"].bwd, e["c1"].bwd_shift, e["c1"].taps, e["c1"].bwd_cols, cin, args)
                if add_lateral:
                    check(L.nrpn_add_inplace(_p(dx), _p(tgt), dx.numel(), self.f16, _stream()), "add_inplace")
            else:
                dyd = self._scratch_buf("dyd", yd.numel(), dt).view_as(yd)
                self._bn_bwd(e["bnd"], g, None, yd, dyd, None, False)
                self._wgrad([dy1], [xs], [od], e["c1"].taps, planes, cin, eng.grad_of(e["c1"].weight), layout=1)
                self._wgrad([dyd], [xs], [od], e["ds"].taps, outc, cin, eng.grad_of(e["ds"].weight), layout=1)
                t1 = self._scratch_buf("t1", n * od[0] * od[1] * od[2] * cin, dt).view(n, *od, cin)
                args = [ops.ConvLevelArgs(dy1, t1, n, od, od, cin)]
                self._conv_call(e["c1"].bwd, e["c1"].bwd_shift, e["c1"].taps, e["c1"].bwd_cols, cin, args)
                direct = (s == 1 and not add_lateral)
                t2 = dx if direct else self._scratch_buf("t2", n * od[0] * od[1] * od[2] * cin, dt).view(n, *od, cin)
                args = [ops.ConvLevelArgs(dyd, t2, n, od, od, cin, res=t1, res_dims=od, ldr=cin)]
                self._conv_call(e["ds"].bwd, e["ds"].bwd_shift, e["ds"].taps, e["ds"].bwd_cols, cin, args)
                if s == 2:
                    full = dx if not add_lateral else self._scratch_buf("dx_tmp", dx.numel(), dt).view_as(dx)
                    check(L.nrpn_stride2(_p(t2), _p(full), n, xd[0], xd[1], xd[2], cin, 1, _stream()), "stride2 scatter")
                    if add_lateral:
                        check(L.nrpn_add_inplace(_p(dx), _p(full), dx.numel(), self.f16, _stream()), "add_inplace")
                elif add_lateral:
                    check(L.nrpn_add_inplace(_p(dx), _p(t2), dx.numel(), self.f16, _stream()), "add_inplace")
        return f

    # ------------------------------------------------------------------------------------------------ run
    def _anchors(self):
        """Materialised anchors of one mesh (2.43 M x 6 fp32 at 160x256x256), built once per plan for the target assignment kernel."""
        if self.anchors is None:
            dev = self.eng.device
            per = []
            for d, s, cell in zip(self.feat_dims, self.strides, self.eng.cells):
                sh = [torch.arange(0, d[i], dtype=torch.float32, device=dev) * s[i] for i in range(3)]
                gx, gy, gz = torch.meshgrid(sh[0], sh[1], sh[2], indexing="ij")
                shifts = torch.stack((gx.reshape(-1), gy.reshape(-1), gz.reshape(-1)) * 2, dim=1)
                per.append((shifts.view(-1, 1, 6) + torch.from_numpy(cell).to(dev).view(1, -1, 6)).reshape(-1, 6))
            self.anchors = torch.cat(per).contiguous()
        return self.anchors

    def _sample(self, labels):
        """BalancedPositiveNegativeSampler (utils.py:35-96) with the reference's own torch.randperm draws."""
        rpn = self.eng.rpn
        positive = torch.where(labels >= 1)[0]
        negative = torch.where(labels == 0)[0]
        num_pos = min(positive.numel(), int(rpn.batch_size_per_mesh * rpn.positive_fraction))
        num_neg = min(negative.numel(), rpn.batch_size_per_mesh - num_pos)
        g = self.eng.gen
        perm1 = torch.randperm(positive.numel(), device=positive.device, generator=g)[:num_pos]
        perm2 = torch.randperm(negative.numel(), device=negative.device, generator=g)[:num_neg]
        return positive[perm1].contiguous(), negative[perm2].contiguous()

    def forward_loss(self, grids, targets, w_obj=1.0, w_reg=None, w_2d=None, eval_2d=False):
        """Forward launches, target assignment, sampling, losses; fills d(pred) for the weighted sum w_obj * L_obj + w_reg * L_reg (+ w_2d * L_2d)."""
        eng, n = self.eng, self.n
        if ops.is_channels_last_grid(grids) or grids.is_contiguous():
            self._src = grids
        else:
            self._src = grids.contiguous()
        self.fwd[0]()                                               # stem packing reads the caller's grid: its pointer changes from step to step
        _replay_static(self._graphs, "fwd", self.fwd[1:])
        anchors = self._anchors()
        samples = []
        forced = getattr(self, "forced_samples", None)         # tests: (pos, neg) index tensors per mesh instead of the sampler's draw
        for i in range(n):
            gt = targets[i].to(device=eng.device, dtype=torch.float32).contiguous()
            if gt.numel() == 0:                                     # background mesh (rpn.py:246-250): every anchor is a negative
                labels = torch.zeros(anchors.shape[0], dtype=torch.float32, device=eng.device)
                pos, neg = self._sample(labels)
                samples.append((pos, neg, torch.zeros((0, 7 if eng.rotated else 6), dtype=torch.float32, device=eng.device)))
                continue
            labels, idx = ops.assign_targets(anchors, gt, None, eng.rpn.fg_iou_thresh, eng.rpn.bg_iou_thresh, True)
            pos, neg = self._sample(labels) if forced is None else (forced[i][0].contiguous(), forced[i][1].contiguous())
            samples.append((pos, neg, gt[idx[pos].clamp(min=0)].contiguous()))
        self.last_samples = samples
        self.loss_grad(w_obj, eng.w_reg if w_reg is None else w_reg, eng.w_2d if w_2d is None else w_2d, eval_2d)

    def loss_grad(self, w_obj, w_reg, w_2d=0.0, eval_2d=False):
        """(Re)computes the losses and d(w_obj * L_obj + w_reg * L_reg + w_2d * L_2d)/d(pred) * loss_scale for the samples of the last forward.
        The 2-D projection loss (rpn.py:421-453) is evaluated when its weight is non-zero or eval_2d asks for its value."""
        eng, L, n = self.eng, lib(), self.n
        samples = self.last_samples
        norm = float(sum(p.numel() + q.numel() for p, q, _ in samples))
        eng.losses.zero_()
        self.dpred.zero_()
        for i, (pos, neg, gtp) in enumerate(samples):
            preds = [p[i].reshape(-1, 128) for p in self.pred_levels]
            dpreds = [p[i].reshape(-1, 128) for p in self.dpred_levels]
            desc = ops.make_rpn_desc(preds, self.feat_dims, self.strides, eng.cells, eng.A, eng.rotated, 1, 1, 0.5, 0.0, 1e-3, self.dims)
            arr = (ctypes.c_void_p * len(dpreds))(*[t.data_ptr() for t in dpreds])
            check(L.nrpn_rpn_loss(ctypes.byref(desc), arr, _p(pos), int(pos.numel()), _p(neg), int(neg.numel()), _p(gtp), max(norm, 1.0), float(w_obj),
                                  float(w_reg) if eng.reg_loss_type == "smooth_l1" else 0.0, float(eng.loss_scale), _p(eng.losses), None, self.f16, _stream()),
                  "rpn_loss")
        if eng.reg_loss_type != "smooth_l1":
            self._iou_reg_loss(float(w_reg), max(norm, 1.0))
        eng.loss_2d.zero_()
        if float(w_2d) != 0.0 or eval_2d:
            self._proj2d_loss(float(w_2d))

    def _gather_deltas(self, i, pos):
        """The head's regression deltas (fp32 predictor output) of the flat anchor indices `pos` of mesh i, and where they live."""
        A, code = self.eng.A, self.eng.code
        level, vox, a = self._split_anchor_index(pos)
        cols = (A + a * code).view(-1, 1) + torch.arange(code, device=pos.device).view(1, -1)
        deltas = torch.empty((pos.numel(), code), dtype=torch.float32, device=self.eng.device)
        for l, p in enumerate(self.pred_levels):
            m = level == l
            if m.any():
                deltas[m] = p[i].reshape(-1, 128)[vox[m].view(-1, 1), cols[m]]
        return deltas, level, vox, cols

    def _proj2d_loss(self, w_2d):
        """loss_rpn_box_reg_2d (rpn.py:421-453): the sampled positives' DECODED boxes and their matched ground truth, two points each, projected into
        four cameras, smooth-L1 / positives / max mesh dimension (model/proj2d.py); with a non-zero weight its gradient w.r.t. the deltas (autograd
        through the torch decode) is ADDED to d(pred).  A step without any positive gives 0 here (0 / 0 = NaN in the reference)."""
        from .model.coder_torch import decode_aabb, decode_obb
        from .model.proj2d import rpn_projection_loss
        eng = self.eng
        n_pos = sum(int(p.numel()) for p, _, _ in self.last_samples)
        if n_pos == 0:
            return
        res = float(max(self.dims))
        anchors = self._anchors()
        total = torch.zeros((), dtype=torch.float32, device=eng.device)
        for i, (pos, neg, gtp) in enumerate(self.last_samples):
            if pos.numel() == 0:
                continue
            deltas, level, vox, cols = self._gather_deltas(i, pos)
            with torch.enable_grad():
                d = deltas.detach().requires_grad_(w_2d != 0.0)
                boxes = decode_obb(anchors[pos], d) if eng.rotated else decode_aabb(anchors[pos], d)
                loss = rpn_projection_loss(boxes, gtp, n_pos, res)
                if w_2d != 0.0:
                    (g,) = torch.autograd.grad(loss, d)
            total = total + loss.detach()
            if w_2d != 0.0:
                g = g * (w_2d * eng.loss_scale)
                for l, dp in enumerate(self.dpred_levels):
                    m = level == l
                    if m.any():
                        view = dp[i].reshape(-1, 128)
                        rows = vox[m].view(-1, 1)
                        view[rows, cols[m]] = (view[rows, cols[m]].float() + g[m]).to(view.dtype)
        eng.loss_2d.copy_(total)

    # ---- IoU-type regression losses (RotatedIOULoss, rpn.py:133-165: "iou", "linear_iou", "giou", "diou") on the <= 128 sampled positives per mesh
    def _split_anchor_index(self, idx):
        """flat anchor index of one mesh -> (level, voxel within the level, anchor): index = level offset + voxel * A + a (rpn.py:20-27)."""
        A = self.eng.A
        vox = [d[0] * d[1] * d[2] for d in self.feat_dims]
        bounds = torch.tensor([0] + [v * A for v in vox], device=idx.device).cumsum(0)
        level = torch.bucketize(idx, bounds[1:], right=True)
        local = idx - bounds[level]
        return level, local // A, local % A

    def _iou_reg_loss(self, w_reg, norm):
        """loss = sum over sampled positives of -log((I + 1) / (U + 1)) (or 1 - ..., or the GIoU / DIoU loss) / number of sampled anchors, on the boxes DECODED from the head's
        deltas; its gradient w.r.t. the deltas (autograd through decode + the IoU Function) is written into d(pred) like the fused kernel does."""
        from .model.coder_torch import decode_obb
        from .model.rotated_iou.oriented_iou_loss import cal_diou_3d, cal_giou_3d, cal_iou_3d
        eng = self.eng
        A, code = eng.A, 8
        anchors = self._anchors()
        total = torch.zeros((), dtype=torch.float32, device=eng.device)
        for i, (pos, neg, gtp) in enumerate(self.last_samples):
            if pos.numel() == 0:
                continue
            level, vox, a = self._split_anchor_index(pos)
            cols = (A + a * code).view(-1, 1) + torch.arange(code, device=pos.device).view(1, -1)
            deltas = torch.empty((pos.numel(), code), dtype=torch.float32, device=eng.device)
            for l, p in enumerate(self.pred_levels):
                m = level == l
                if m.any():
                    deltas[m] = p[i].reshape(-1, 128)[vox[m].view(-1, 1), cols[m]]
            with torch.enable_grad():
                d = deltas.detach().requires_grad_(True)
                boxes = decode_obb(anchors[pos], d)
                if eng.reg_loss_type == "giou":
                    losses = cal_giou_3d(boxes.unsqueeze(0), gtp.unsqueeze(0))[0]
                elif eng.reg_loss_type == "diou":
                    losses = cal_diou_3d(boxes.unsqueeze(0), gtp.unsqueeze(0))[0]
                else:
                    iou, _, _, _, union = cal_iou_3d(boxes.unsqueeze(0), gtp.unsqueeze(0), verbose=True)
                    ratio = (iou * union + 1.0) / (union + 1.0)
                    losses = -torch.log(ratio) if eng.reg_loss_type == "iou" else 1.0 - ratio
                loss = losses.sum() / norm
                (g,) = torch.autograd.grad(loss, d)
            total = total + loss.detach()
            if w_reg != 0.0:
                g = (g * (w_reg * eng.loss_scale)).to(self.dpred.dtype)
                for l, dp in enumerate(self.dpred_levels):
                    m = level == l
                    if m.any():
                        dp[i].reshape(-1, 128)[vox[m].view(-1, 1), cols[m]] = g[m]
        eng.losses[1] = total

    def backward(self):
        """Backward launches in reverse construction order.  Gradients become final from the END of the flat bucket (head, FPN) towards
        its start (stem): every time >= bucket_elems new elements are final their all-reduce is launched on the comm stream, overlapping
        the dgrad / wgrad of the layers below (run_rpn.py:235-236: DDP's bucketed all-reduce during loss.backward())."""
        eng = self.eng
        if not (eng.world > 1 and eng.overlap_allreduce):
            self.allreduce_calls = 0
            _replay_static(self._graphs, "bwd", list(reversed(self.bwd)))
            return
        sched = {k: (lo, hi) for k, lo, hi in bucket_schedule(self.bwd_lo, eng.n_params, eng.bucket_elems)}
        self.allreduce_calls = 0
        order = list(reversed(self.bwd))
        start = 0
        for seg, k in enumerate(sorted(sched) + ([len(order) - 1] if (len(order) - 1) not in sched else [])):
            _replay_static(self._graphs, f"bwd{seg}", order[start:k + 1])      # the launches between two all-reduce points: one graph each
            start = k + 1
            if k in sched:
                lo, hi = sched[k]
                ev = torch.cuda.Event()
                ev.record()
                eng.comm_stream.wait_event(ev)
                with torch.cuda.stream(eng.comm_stream):
                    torch.distributed.all_reduce(eng.flat_g[lo:hi], group=eng.pg)
                self.allreduce_calls += 1

    def run(self, grids, targets, backward=True):
        self.forward_loss(grids, targets)
        if backward:
            self.backward()
