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
from collections import OrderedDict
from typing import List, Optional, Sequence

import torch

from . import ops, packing
from ._lib import RpnDesc, check, lib
from .engine import _down


_TRAIN_GRAPH = os.environ.get("NRPN_TRAIN_GRAPH", "1") != "0"          # static launch lists of the training step replayed as CUDA graphs
PLAN_CACHE = 4          # batch shapes whose per-shape state (launch lists, anchors, CUDA graphs) is kept, least recently used first out



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


def bucket_schedule(bwd_lo: Sequence[int], n_params: int, bucket_elems: int, lowest: int = 0):
    """All-reduce ranges of the flat gradient bucket, in launch order.  bwd_lo[i] = lowest flat offset that is final once backward stage i
    (construction order: stem, blocks..., FPN, head) has run; stages execute in REVERSE, so gradients become final from the end of the bucket
    towards its start.  A range [lo, hi) is launched after a stage as soon as at least bucket_elems new elements are final (or the bucket is
    complete down to `lowest`, the start of the part the backward pass produces: the head's offset when the backbone is frozen).
    Returns [(stage index in execution order, lo, hi)]: disjoint, covering [lowest, n_params) exactly once."""
    out, hi = [], n_params
    for k, lo in enumerate(reversed(list(bwd_lo))):
        if hi > lo and (hi - lo >= bucket_elems or lo <= lowest):
            out.append((k, lo, hi))
            hi = lo
    return out


class _TConv:
    """One trainable convolution: its fp32 weight (+ bias), their gradient destinations (by default the parameters' views of the flat
    gradient bucket), its 16-bit forward / data-gradient operands and tap table."""

    def __init__(self, eng, weight, bias, stride=1, need_dgrad=True, stem=False, dw=None, db=None):
        self.eng = eng
        self.weight, self.bias = weight, bias
        self.dw = eng.grad_of(weight) if dw is None else dw
        self.db = eng.grad_of(bias) if db is None and bias is not None else db
        cout, cin, k = weight.shape[0], weight.shape[1], weight.shape[2]
        self.cout, self.cin_real, self.k = cout, cin, k
        self.stride = stride
        dt, dev = eng.act_dtype, eng.device
        self.stem = stem
        if stem:
            probe = torch.arange(1, weight.numel() + 1, dtype=torch.float32).view_as(weight)
            wp, taps = packing.pack_stem_weight(probe, None, dtype=torch.float32)                  # (32, 64, 64): source index + 1, 0 = structural zero
            self.taps = taps
            self.cin, self.cout_pad = 64, 64
            self.gather_idx = (wp.reshape(-1).to(torch.int64) - 1).to(torch.int32).to(dev)       # packed position -> master index
            inv = torch.full((weight.numel(),), -1, dtype=torch.int32)
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
            check(L.nrpn_gather_pack(_p(self.weight.data), _p(self.gather_idx), self.gather_idx.numel(), _p(self.fwd), None, f16, _stream()),
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
    """Forward + backward + update for ResNet_FPN_256 or VGG_FPN (strided stem) + RPNHead (+ RegionProposalNetwork hyper-parameters)."""

    def __init__(self, model, precision: str = "bf16", lr: float = 1e-4, weight_decay: float = 0.01, betas=(0.9, 0.999), eps: float = 1e-8,
                 clip_grad_norm: float = 0.1, reg_loss_weight: float = 5.0, process_group=None, bucket_mb: float = 32.0,
                 loss_scale: Optional[float] = None, seed: Optional[int] = None, reg_loss_weight_2d: float = 0.0, freeze_backbone: bool = False):
        if precision not in ("bf16", "fp16"):
            raise ValueError("training runs with bf16 (default) or fp16 (with a static loss scale) 16-bit activations / gradients")
        bb, rpn = model.backbone, model.rpn
        built = ("nerf_rpn_b200: the training engine implements RPNHead on ResNet_FPN_256 (BASELINE config 4) or on VGG_FPN with cfg AF / DF / EF, "
                 "batch_norm=True and the strided stem (input_size >= 160)")
        if type(bb).__name__ == "VGG_FPN":
            mods = list(bb.layers.children())
            convs = [(grp, i) for grp in mods[-4:] for i, m in enumerate(grp) if isinstance(m, torch.nn.Conv3d)]
            if mods[0].stride[0] != 2 or not all(i + 1 < len(grp) and isinstance(grp[i + 1], torch.nn.BatchNorm3d) for grp, i in convs):
                raise NotImplementedError(built)
        elif type(bb).__name__ != "ResNet_FPN_256":
            raise NotImplementedError(built)
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
        # Per-shape plans are few (PLAN_CACHE, LRU); their activation / gradient buffers are views of ONE pool shared by every shape:
        # the k-th buffer a plan requests is the first bytes of slot k, and every plan requests its buffers in the same order.  Scratch and
        # workspaces of the backward pass are shared the same way.  A slot (or scratch buffer) only grows -- to the largest batch seen so far --
        # and growing drops every other cached plan and graph, because they hold the old pointers.
        self._plans = OrderedDict()
        self._pool: List[torch.Tensor] = []
        self._scratch = {}
        self.pool_growths = 0
        self.scratch_growths = 0
        self.forward_count = 0              # training forwards run so far: a backward checks that its activations were not overwritten since
        self._graphs = {}                      # captured static launch lists (repack)
        self.comm_stream = torch.cuda.Stream(device=self.device)
        self._norm = torch.zeros(1, dtype=torch.float32, device=self.device)
        self._norm_ws = torch.empty(lib().nrpn_grad_norm_workspace_bytes(), dtype=torch.uint8, device=self.device)
        self._red_ws = torch.empty(lib().nrpn_chan_reduce_workspace_bytes(2048), dtype=torch.uint8, device=self.device)
        self.losses = torch.zeros(2, dtype=torch.float32, device=self.device)
        self.loss_2d = torch.zeros((), dtype=torch.float32, device=self.device)        # loss_rpn_box_reg_2d (unweighted), when evaluated
        self.overlap_allreduce = True       # False: leave the gradient all-reduce to the caller (DDP wrapping the autograd compat path)
        # True: run_rpn.py --freeze_backbone.  The backbone (FPN included) keeps training-mode BatchNorm but gets no gradient: the step runs the
        # head's backward only, and clip, AdamW and the all-reduce cover the head's range [head_lo, n_params) of the flat buffers.  Read when a
        # step plans its batch and when it updates, so it may change between steps.
        self.freeze_backbone = bool(freeze_backbone)
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
        self.head_lo = total - sum(p.numel() for p in self.head.parameters())      # the head is the contiguous tail of the flat buffers
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
            n_bb = len(self._params) - len(list(self.head.parameters()))
            self.repack(head_only=self.freeze_backbone and not moved and ver[:n_bb] == self._packed_ver[:n_bb])

    def grad_of(self, p):
        off, n = self.offsets[id(p)]
        return self.flat_g[off:off + n]

    def _build_layers(self):
        """The backbone's trainable layers.  ResNet: self.blocks (Bottleneck dicts).  VGG: self.vgg_stages, four lists of
        ("conv", _TConv, _BN) / ("pool",) items.  Either neck: self.lat, the lateral convs coarsest level first, and self.fpn_out, the output
        conv of each of those levels, None where the level is its lateral (ResNet's P5)."""
        bb, hd = self.bb, self.head

        def conv(m: torch.nn.Conv3d, **kw):
            return _TConv(self, m.weight, m.bias, stride=m.stride[0], **kw)
        self.blocks, self.vgg_stages = [], None
        if type(bb).__name__ == "ResNet_FPN_256":
            self.stem = conv(bb.conv1, need_dgrad=False, stem=True)
            self.stem_bn = _BN(self, bb.bn1)
            for stage in bb.layers:
                for blk in stage:
                    e = dict(c1=conv(blk.conv1), bn1=_BN(self, blk.bn1), c2=conv(blk.conv2), bn2=_BN(self, blk.bn2),
                             c3=conv(blk.conv3), bn3=_BN(self, blk.bn3), ds=None, bnd=None, stride=blk.stride)
                    if blk.downsample is not None:
                        e["ds"] = conv(blk.downsample[0]); e["bnd"] = _BN(self, blk.downsample[1])
                    self.blocks.append(e)
            body = [e[k] for e in self.blocks for k in ("c1", "c2", "c3", "ds") if e[k] is not None]
            self.lat = [conv(m) for m in bb.latlayers]
            self.fpn_out = [None] + [conv(m) for m in bb.smooths]
        else:                                           # VGG_FPN with a strided stem and BatchNorm (checked by __init__)
            mods = list(bb.layers.children())
            self.stem = conv(mods[0], need_dgrad=False, stem=True)
            self.stem_bn = _BN(self, mods[1])
            self.vgg_stages = []
            for grp in mods[-4:]:
                seq, items = list(grp.children()), []
                for i, m in enumerate(seq):
                    if isinstance(m, torch.nn.Conv3d):
                        items.append(("conv", conv(m), _BN(self, seq[i + 1])))
                    elif isinstance(m, torch.nn.MaxPool3d):
                        items.append(("pool",))
                # cfgs AF / DF / EF: a pool only ever ends a stage, so a stage's backward needs two scratch buffers
                assert all(it[0] == "conv" for it in items[:-1]), "unexpected VGG stage layout"
                self.vgg_stages.append(items)
            body = [it[1] for items in self.vgg_stages for it in items if it[0] == "conv"]
            self.lat = [conv(m) for m in reversed(bb.fpn_neck.lateral_convs)]
            self.fpn_out = [conv(m) for m in reversed(bb.fpn_neck.fpn_convs)]
        self.hconv = [conv(m) for m in hd.conv if isinstance(m, torch.nn.Conv3d)]
        # fused cls | bbox predictor (anchor.py:196-198): one 1^3 conv with 128 (padded) output channels on fp32 staging copies of the two
        # layers' weights and biases (_repack_head); its gradients land in staging buffers that head_bwd splits into the two layers' gradients
        self.n_pred = self.A * (1 + self.code)
        if self.n_pred > 128:
            raise ValueError("fused predictor supports at most 128 output channels")
        f32 = dict(dtype=torch.float32, device=self.device)
        self.predictor = _TConv(self, torch.zeros((128, 256, 1, 1, 1), **f32), torch.zeros(128, **f32),
                                dw=torch.zeros((128, 256), **f32), db=torch.zeros(128, **f32))
        self.all_convs = [self.stem] + body + self.lat + [c for c in self.fpn_out if c is not None] + self.hconv

    def repack(self, head_only: bool = False):
        """fp32 master weights -> 16-bit GEMM operands (after every optimiser step / checkpoint load); head_only: the head's convs and the
        fused predictor, when no backbone weight has changed (a frozen backbone's operands are packed once)."""
        self._packed_ver = tuple(p._version for p in self._params)
        if head_only:
            _replay_static(self._graphs, "repack_head", [self._repack_head])
        else:
            _replay_static(self._graphs, "repack", [self._repack_launches])

    def _repack_launches(self):
        for c in self.all_convs[:-len(self.hconv)]:
            c.repack()
        self._repack_head()

    def _repack_head(self):
        for c in self.hconv:
            c.repack()
        hd, A, pr = self.head, self.A, self.predictor
        pr.weight[:A].copy_(hd.cls_logits.weight.data)
        pr.weight[A:self.n_pred].copy_(hd.bbox_pred.weight.data)
        pr.bias[:A].copy_(hd.cls_logits.bias.data); pr.bias[A:self.n_pred].copy_(hd.bbox_pred.bias.data)
        pr.repack()

    # ------------------------------------------------------------------------------------------------ plan
    def plan(self, n, dims):
        key = (n, tuple(int(d) for d in dims), self.freeze_backbone)
        p = self._plans.get(key)
        if p is not None:
            self._plans.move_to_end(key)
            return p
        p = _TrainPlan(self, n, key[1], key[2])
        self._plans[key] = p
        while len(self._plans) > PLAN_CACHE:
            _, old = self._plans.popitem(last=False)
            if any(st["graph"] is not None for st in old._graphs.values()):
                torch.cuda.current_stream().synchronize()          # its graphs may still be in flight
            old.release()
        return p

    def plan_for(self, grids):
        """The plan of a stacked (N,4,X,Y,Z) batch, or of a list of (4,X_i,Y_i,Z_i) scenes padded to their element-wise maximum."""
        if isinstance(grids, (list, tuple)):
            return self.plan(len(grids), ops.padded_extent(grids))
        n, c, X, Y, Z = grids.shape
        return self.plan(n, (X, Y, Z))

    def cache_stats(self):
        """Plans and captured CUDA graphs alive, pool slots and their bytes (the training step's activation / gradient memory), the shared scratch
        and the cached plans' materialised anchors."""
        return {"plans": len(self._plans), "graphs": sum(st["graph"] is not None for p in self._plans.values() for st in p._graphs.values()),
                "pool_slots": len(self._pool), "pool_bytes": sum(t.numel() for t in self._pool), "pool_growths": self.pool_growths,
                "scratch_bytes": sum(t.numel() * t.element_size() for t in self._scratch.values()), "scratch_growths": self.scratch_growths,
                "anchor_bytes": sum(p.anchors.numel() * 4 for p in self._plans.values() if p.anchors is not None)}

    def _drop_graphs(self):
        """A scratch buffer of the backward pass is about to be replaced by a larger one: the launch lists fetch scratch when they run, so the plans
        stay, but every captured graph holds the old pointer and goes (its plan runs eagerly twice and captures again)."""
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("nerf_rpn_b200: training buffers must not grow during graph capture")
        self.scratch_growths += 1
        if any(st["graph"] is not None for p in self._plans.values() for st in p._graphs.values()):
            torch.cuda.current_stream().synchronize()
            for p in self._plans.values():
                p._graphs.clear()

    def _drop_cached(self, keep=None):
        """A pool slot or scratch buffer is about to be replaced by a larger one: every cached plan but `keep` (and every graph) points at the old
        memory, so they go; `keep` runs eagerly again until its launch lists are re-captured."""
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("nerf_rpn_b200: training buffers must not grow during graph capture")
        torch.cuda.current_stream().synchronize()
        for key in [k for k, p in self._plans.items() if p is not keep]:
            self._plans.pop(key).release()
        if keep is not None:
            keep._graphs.clear()
        self.pool_growths += 1

    def _pool_view(self, k, shape, dtype, plan):
        """Request k of a plan under construction: the first numel elements of pool slot k, as `shape`."""
        numel = math.prod(shape)
        nbytes = max(numel * torch.empty((), dtype=dtype).element_size(), 1)
        if k >= len(self._pool) or self._pool[k].numel() < nbytes:
            if k < len(self._pool):
                if not plan._grew:                      # once per plan: after that no other plan is left to drop
                    self._drop_cached(keep=plan)
                    plan._grew = True
                self._pool[k] = None                    # nothing else refers to the old slot now: freed before the larger one is allocated
            slot = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            if k < len(self._pool):
                self._pool[k] = slot
            else:
                self._pool.append(slot)
        return self._pool[k][:nbytes].view(dtype)[:numel].view(shape)

    def density_to_alpha(self) -> bool:
        """The model's density_to_alpha_on_device: raw densities in, datasets.py:165-167 applied by the stem packing (training and evaluation alike)."""
        return bool(getattr(self.model, "density_to_alpha_on_device", False))

    # ------------------------------------------------------------------------------------------------ step
    def forward_backward(self, grids, targets: Sequence[torch.Tensor]):
        """grids: (N,4,X,Y,Z) fp32 CUDA, or a list of N (4,X_i,Y_i,Z_i) fp32 CUDA scenes of different sizes (each contiguous or the dataset's
        channels-last view), trained as the batch zero-padded to their element-wise maximum like the reference does (nerf_rpn.py:129-146,
        anchors in the padding labelled -1); targets: N tensors (G,6|7).  Runs forward, losses, backward (+ the overlapped gradient
        all-reduce when a process group is active).  Returns the loss tensor (2,) = [loss_objectness, loss_rpn_box_reg] (device).
        One step at a time: every shape shares the engine's buffers."""
        plan = self.plan_for(grids)
        plan.run(grids, targets)
        return self.losses

    def optimizer_step(self, lr: Optional[float] = None):
        """clip_grad_norm_(clip) + AdamW on the flat buffers (after the all-reduce has drained), then re-pack the 16-bit operands.  With a
        frozen backbone, norm, update and re-packing cover the head alone, as torch's skip parameters whose .grad is None."""
        torch.cuda.current_stream().wait_stream(self.comm_stream)
        self.step_count += 1
        inv = 1.0 / (self.loss_scale * self.world)
        L = lib()
        lo = self.head_lo if self.freeze_backbone else 0
        p, g, m, v = (ctypes.c_void_p(t.data_ptr() + 4 * lo) for t in (self.flat_p, self.flat_g, self.flat_m, self.flat_v))
        n = self.n_params - lo
        check(L.nrpn_grad_norm(g, n, inv, _p(self._norm), _p(self._norm_ws), self._norm_ws.numel(), _stream()), "grad_norm")
        check(L.nrpn_adamw_step(p, g, m, v, n, _p(self._norm), float(self.clip),
                                inv, float(self.lr if lr is None else lr), self.betas[0], self.betas[1], self.eps, self.wd, self.step_count, _stream()),
              "adamw_step")
        self.repack(head_only=self.freeze_backbone)

    def train_step(self, grids, targets, lr: Optional[float] = None):
        losses = self.forward_backward(grids, targets)
        self.optimizer_step(lr)
        return losses


class _TrainPlan:
    """Buffers and the launch lists (forward, backward) for n scenes of one size.  frozen: the backbone gets no gradient, so the backward list
    is the head's alone and every backbone activation that only its backward would read lives in a few reused slots.
    Built in four parts: the stem, the backbone body (ResNet blocks or VGG stages), the FPN and the head."""

    def __init__(self, eng: RPNTrainEngine, n: int, dims, frozen: bool = False):
        self.eng, self.n, self.dims, self.frozen = eng, n, dims, frozen
        self.fwd: List = []
        self.bwd: List = []                      # built in forward order, executed reversed
        self.bwd_lo: List[int] = []              # lowest flat-parameter offset whose gradient is final once bwd[i] has run
        self.f16 = eng.f16
        self._scratch = eng._scratch             # shared by every plan (engine-level, grows to the largest batch)
        self._graphs = {}
        self._grew = False
        self._n_req = 0
        self.input = None
        d1 = _down(dims)
        d2 = _down(d1)
        geo = self._resnet_geometry(d2) if eng.vgg_stages is None else self._vgg_geometry(d2)
        self.packed = self._req((n, d1[0], d1[1], d1[2] + 1, 64))
        self.fwd.append(self._pack_input)
        if frozen:
            self._act = self._frozen_slots(*(self._resnet_slot_uses(geo, d1, d2) if eng.vgg_stages is None else self._vgg_slot_uses(geo, d1, d2)))
        else:
            self._act = lambda slot, d, c: self._buf(d, c)
        p0, dp0 = self._build_stem(d1, d2)
        c_out = self._build_resnet_body(geo, p0, dp0) if eng.vgg_stages is None else self._build_vgg_body(geo, p0, dp0)
        self._build_head(*self._build_fpn(c_out))
        self._src = None
        self._sizes = None
        self._alpha = False
        self.valid = None
        self.anchors = None
        if self._grew:
            torch.cuda.empty_cache()            # hand the replaced (smaller) slots back instead of keeping them cached next to the new ones

    # ------------------------------------------------------------------------------------------------ buffers of the plan
    def _req(self, shape, dtype=None):
        """The next buffer of the plan: every plan requests its buffers in the same order (see RPNTrainEngine._pool_view)."""
        t = self.eng._pool_view(self._n_req, tuple(shape), self.eng.act_dtype if dtype is None else dtype, self)
        self._n_req += 1
        return t

    def _buf(self, d, c, dtype=None):
        return self._req((self.n, *d, c), dtype)

    def _frozen_slots(self, use, names):
        """Slots of a frozen plan's forward-only activations: use[k] = [(dims, channels)] of every activation placed in slot kind k; names =
        [(slot, kind)] in request order, each slot sized for its kind's largest use.  Returns act(slot, dims, channels)."""
        n = self.n
        size = {k: max([n * math.prod(d) * c for d, c in u] + [1]) for k, u in use.items()}
        slots = {s: self._req((size[k],)) for s, k in names}

        def act(slot, d, c):
            return slots[slot][:n * math.prod(d) * c].view(n, *d, c)
        return act

    # ------------------------------------------------------------------------------------------------ stem
    def _build_stem(self, d1, d2):
        """Stem conv (+ its bias, VGG) + BN + ReLU + max-pool (3, 2, 1).  Returns the pooled map and the buffer receiving its gradient."""
        eng, n, L = self.eng, self.n, lib()
        y0 = self._act("y", d1, 64); a0 = self._act("a", d1, 64)
        self._conv_fwd(eng.stem, [self.packed], [(d1[0], d1[1], d1[2] + 1)], [y0], [d1])
        self._bn_fwd(eng.stem_bn, y0, None, a0, True)
        p0 = self._act("x0", d2, 64)
        if self.frozen:
            self.fwd.append(lambda: check(L.nrpn_maxpool3d_k3s2(_p(a0), n, d1[0], d1[1], d1[2], 64, _p(p0), self.f16, _stream()), "maxpool"))
            return p0, None
        self.pool_idx = self._buf(d2, 64, torch.uint8)
        self.fwd.append(lambda: check(L.nrpn_maxpool3d_k3s2_argmax(_p(a0), n, d1[0], d1[1], d1[2], 64, _p(p0), _p(self.pool_idx), self.f16, _stream()),
                                      "maxpool_argmax"))
        dp0 = self._buf(d2, 64)                          # gradient w.r.t. the pooled map
        da0 = self._buf(d1, 64); dy0 = self._buf(d1, 64)

        # backward of the stem (runs LAST): pool backward -> BN backward -> stem wgrad (on the packed input) and bias gradient
        def stem_bwd():
            check(L.nrpn_maxpool3d_k3s2_backward(_p(dp0), _p(self.pool_idx), n, d1[0], d1[1], d1[2], 64, _p(da0), self.f16, _stream()), "maxpool_backward")
            self._bn_bwd(eng.stem_bn, da0, a0, y0, dy0, None, True)
            self._wgrad_stem(dy0)
            if eng.stem.db is not None:                 # VGG's stem conv has a bias, ResNet's has none
                self._bias_grad(eng.stem, [dy0])
        self.bwd.append(stem_bwd)
        self.bwd_lo.append(0)
        return p0, dp0

    # ------------------------------------------------------------------------------------------------ ResNet body
    def _resnet_geometry(self, d2):
        """The blocks in order: (stage, block, its input dims, its output dims, is the stage's first / last block)."""
        geo, xd = [], d2
        for si, stage in enumerate(self.eng.bb.layers):
            for j in range(len(stage)):
                e = self.eng.blocks[len(geo)]
                od = _down(xd) if e["stride"] == 2 else xd
                geo.append((si, e, xd, od, j == 0, j == len(stage) - 1))
                xd = od
        return geo

    def _resnet_slot_uses(self, geo, d1, d2):
        # activations read only by the forward: the stem's y0 / a0 share slots "y" / "a" with the blocks' y3 / yd, every block's y1, y2
        # share "y1" and a1, a2 share "a1", and the max-pool output and the outputs that are not a stage's last alternate between "x0"
        # and "x1" (sized alike).  Each slot is requested once, at its largest use.
        use = {"y": [(d1, 64)], "a": [(d1, 64)], "r": [], "y1": [], "a1": [], "x": [(d2, 64)]}
        for si, e, xd_, od, first, last in geo:
            use["y1"].append((od, e["c1"].cout)); use["a1"].append((od, e["c1"].cout)); use["y"].append((od, e["c3"].cout))
            if e["ds"] is not None:
                use["a"].append((od, e["c3"].cout)); use["r"].append((od, e["c3"].cout))
            if not last:
                use["x"].append((od, e["c3"].cout))
        return use, [("y", "y"), ("a", "a"), ("r", "r"), ("y1", "y1"), ("a1", "a1"), ("x0", "x"), ("x1", "x")]

    def _build_resnet_body(self, geo, p0, dp0):
        """Bottleneck blocks.  Returns the four stage outputs [(tensor, dims, gradient buffer)], finest first."""
        eng, frozen, act, buf = self.eng, self.frozen, self._act, self._buf
        x, dx, xs = p0, dp0, "x0"     # block input, the buffer that receives its gradient, and its slot (frozen)
        c_out = []
        for si, e, xd, od, first, last in geo:
            # a stage's first block -- and only it -- has a downsample, strided in every stage but the first (ResNet_FPN_256._make_layer):
            # the backward of the first block of stages 1..3 adds its zero-stuffed data gradient to the lateral part fpn_bwd wrote
            assert (e["ds"] is not None) == first and (e["stride"] == 2) == (first and si > 0), "unexpected ResNet stage layout"
            s = e["stride"]
            planes, outc = e["c1"].cout, e["c3"].cout
            y1, a1 = act("y1", od, planes), act("a1", od, planes)
            y2, a2 = act("y1", od, planes), act("a1", od, planes)
            y3 = act("y", od, outc)
            if frozen and not last:
                xs = "x1" if xs == "x0" else "x0"
                out = act(xs, od, outc)
            else:
                out = buf(od, outc)                # a stage output (read by its FPN lateral) persists
            self._conv_fwd(e["c1"], [x], [xd], [y1], [od])
            self._bn_fwd(e["bn1"], y1, None, a1, True)
            self._conv_fwd(e["c2"], [a1], [od], [y2], [od])
            self._bn_fwd(e["bn2"], y2, None, a2, True)
            self._conv_fwd(e["c3"], [a2], [od], [y3], [od])
            if e["ds"] is not None:
                yd, r = act("a", od, outc), act("r", od, outc)
                self._conv_fwd(e["ds"], [x], [xd], [yd], [od])
                self._bn_fwd(e["bnd"], yd, None, r, False)
            else:
                yd, r = None, x
            self._bn_fwd(e["bn3"], y3, r, out, True)
            dout = None
            if not frozen:
                dout = buf(od, outc)               # gradient w.r.t. the block output (filled by the consumer's backward)
                self.bwd.append(self._make_block_bwd(e, x, xd, dx, od, y1, a1, y2, a2, y3, out, yd, dout, s))
                self.bwd_lo.append(min(eng.offsets[id(p_)][0] for k_ in ("c1", "c2", "c3", "ds") if e[k_] is not None for p_ in [e[k_].weight]))
            x, dx = out, dout
            if last:
                c_out.append((x, od, dx))
        return c_out

    # ------------------------------------------------------------------------------------------------ VGG body
    def _vgg_geometry(self, d2):
        """Per stage: [(item, its input dims, its output dims, its output channels)]; a ceil-mode pool halves the extent rounding up."""
        geo, xd, c = [], d2, 64
        for items in self.eng.vgg_stages:
            st = []
            for it in items:
                od = _down(xd) if it[0] == "pool" else xd
                c = it[1].cout if it[0] == "conv" else c
                st.append((it, xd, od, c))
                xd = od
            geo.append(st)
        return geo

    def _vgg_slot_uses(self, geo, d1, d2):
        # activations read only by the forward: every conv's raw output shares slot "y" with the stem's y0, the stem's a0 has slot "a", and
        # the max-pool output and the activations that are not a stage's output alternate between "x0" and "x1"
        use = {"y": [(d1, 64)], "a": [(d1, 64)], "x": [(d2, 64)]}
        for st in geo:
            for j, (it, xd, od, c) in enumerate(st):
                if it[0] == "conv":
                    use["y"].append((xd, c))
                if j < len(st) - 1:
                    use["x"].append((od, c))
        return use, [("y", "y"), ("a", "a"), ("x0", "x"), ("x1", "x")]

    def _build_vgg_body(self, geo, p0, dp0):
        """Stages of conv (+ bias) -> batch statistics -> BN + ReLU, a stage of cfg AF / DF / EF ending in MaxPool3d(2, 2, ceil_mode=True)
        from the second on (feature_extractor.py:343-357).  Returns the four stage outputs [(tensor, dims, gradient buffer)], finest first."""
        eng, n, L, frozen = self.eng, self.n, lib(), self.frozen
        x, dx, xs = p0, dp0, "x0"
        c_out = []
        for si, st in enumerate(geo):
            recs = []                             # what the stage's backward reads, in forward order
            for j, (it, xd, od, c) in enumerate(st):
                if frozen and j < len(st) - 1:
                    xs = "x1" if xs == "x0" else "x0"
                    out = self._act(xs, od, c)
                else:
                    out = self._buf(od, c)        # a stage output (read by its FPN lateral) persists
                if it[0] == "conv":
                    _, conv, bn = it
                    y = self._act("y", xd, c)     # raw conv output, conv bias included (_TConv.shift)
                    self._conv_fwd(conv, [x], [xd], [y], [xd])
                    self._bn_fwd(bn, y, None, out, True)
                    recs.append(("conv", conv, bn, x, xd, y, out))
                elif frozen:
                    self.fwd.append(lambda a=x, o=out, d=xd, ch=c: check(L.nrpn_maxpool3d_k2s2_ceil(_p(a), n, d[0], d[1], d[2], ch, _p(o), self.f16, _stream()),
                                                                        "maxpool_k2s2"))
                else:
                    idx = self._buf(od, c, torch.uint8)
                    self.fwd.append(lambda a=x, o=out, i=idx, d=xd, ch=c: check(
                        L.nrpn_maxpool3d_k2s2_ceil_argmax(_p(a), n, d[0], d[1], d[2], ch, _p(o), _p(i), self.f16, _stream()), "maxpool_k2s2_argmax"))
                    recs.append(("pool", x, xd, idx))
                x = out
            dout = None
            if not frozen:
                dout = self._buf(st[-1][2], st[-1][3])  # gradient w.r.t. the stage output: fpn_bwd writes the lateral part first
                self.bwd.append(self._make_vgg_stage_bwd(recs, dx, dout, accumulate=si > 0))
                self.bwd_lo.append(min(eng.offsets[id(r[1].weight)][0] for r in recs if r[0] == "conv"))
            c_out.append((x, st[-1][2], dout))
            dx = dout
        return c_out

    def _make_vgg_stage_bwd(self, recs, dx, dout, accumulate):
        """Backward of one VGG stage, items in reverse: pool backward; BN backward (ReLU masked), weight and bias gradients, data gradient.
        dx receives the gradient of the stage input.  accumulate: dx is the previous stage's output gradient, which already holds the lateral
        part fpn_bwd wrote, and the first conv's data gradient is added to it."""
        L, n, dt = lib(), self.n, self.eng.act_dtype

        def f():
            g = dout                                                            # gradient w.r.t. the current item's output
            for k in range(len(recs) - 1, -1, -1):
                r = recs[k]
                if r[0] == "pool":
                    _, a, ad, idx = r
                    da = self._scratch_buf("vgg_g", a.numel(), dt).view_as(a)
                    check(L.nrpn_maxpool3d_k2s2_ceil_backward(_p(g), _p(idx), n, ad[0], ad[1], ad[2], a.shape[-1], _p(da), self.f16, _stream()),
                          "maxpool_k2s2_backward")
                    g = da
                    continue
                _, conv, bn, x, xd, y, a = r
                dy = self._scratch_buf("vgg_dy", y.numel(), dt).view_as(y)
                self._bn_bwd(bn, g, a, y, dy, None, True)
                self._param_grad(conv, [dy], [x])
                dst = dx if k == 0 and not accumulate else self._scratch_buf("vgg_g", x.numel(), dt).view_as(x)
                self._dgrad(conv, [dy], [dst], [xd])
                g = dst
            if accumulate:
                check(L.nrpn_add_inplace(_p(dx), _p(g), dx.numel(), self.f16, _stream()), "add_inplace")
        return f

    # ------------------------------------------------------------------------------------------------ FPN
    def _build_fpn(self, c_out):
        """Top-down FPN of either neck (feature_extractor.py:224-235, fpn.py:134-161) on the stage outputs c_out (finest first): level i,
        coarsest first, is eng.lat[i] on its stage output plus the nearest up-sampled level i - 1, then eng.fpn_out[i] on it (None: the
        level itself is the feature map).  Returns ([P2..P5], their gradient buffers, their dims)."""
        eng, n, L, frozen, buf = self.eng, self.n, lib(), self.frozen, self._buf
        grad = (lambda d, c: None) if frozen else buf      # the FPN's gradient buffers (none when the backbone is frozen)
        lvl = c_out[::-1]
        q, dq, qd = [], [], []
        for i, ((c, cd, _), lat) in enumerate(zip(lvl, eng.lat)):
            q.append(buf(cd, 256)); dq.append(grad(cd, 256)); qd.append(cd)
            if i == 0:
                self._conv_fwd(lat, [c], [cd], [q[0]], [cd])
            else:
                self._conv_fwd(lat, [c], [cd], [q[i]], [cd], res=q[i - 1], res_dims=qd[i - 1])
        feats, dfeats = [], []
        for i, oc in enumerate(eng.fpn_out):
            if oc is None:                                  # the level's gradient accumulates in dq[i]
                feats.append(q[i]); dfeats.append(dq[i])
                continue
            f = buf(qd[i], 256); df = grad(qd[i], 256)
            self._conv_fwd(oc, [q[i]], [qd[i]], [f], [qd[i]])
            feats.append(f); dfeats.append(df)

        # FPN backward (executed after the head's backward): output convs and the top-down merge from the finest level, then the laterals
        def fpn_bwd():
            for i in range(len(q) - 1, -1, -1):
                oc = eng.fpn_out[i]
                if oc is not None:
                    self._param_grad(oc, [dfeats[i]], [q[i]])
                    self._dgrad(oc, [dfeats[i]], [dq[i]], [qd[i]])
                if i + 1 < len(q):                          # the finer level's merged map took up(q[i]) as its residual
                    fd, cd_ = qd[i + 1], qd[i]
                    check(L.nrpn_upsample_nearest_backward(_p(dq[i + 1]), n, fd[0], fd[1], fd[2], cd_[0], cd_[1], cd_[2], 256, _p(dq[i]), self.f16, _stream()),
                          "upsample_backward")
            for i, ((c, cd, dc), lat) in enumerate(zip(lvl, eng.lat)):
                self._param_grad(lat, [dq[i]], [c])
                self._dgrad(lat, [dq[i]], [dc], [cd])      # dc = gradient of the stage output from the lateral branch
        # NOTE: the stage outputs c2..c4 also receive the next stage's data gradient: the body's backward ADDS it into dc, because fpn_bwd
        # (which runs earlier) has already written the lateral part.
        if not frozen:
            self.bwd.append(fpn_bwd)
            self.bwd_lo.append(min(eng.offsets[id(c.weight)][0] for c in eng.lat + [o for o in eng.fpn_out if o is not None]))
        self.dbg = dict(q=q, dq=dq, c_out=c_out)           # tools/debug_train.py
        self.features, self.feat_dims = feats[::-1], qd[::-1]   # [P2, P3, P4, P5]; fpn_bwd keeps reading dfeats coarsest level first
        return self.features, dfeats[::-1], self.feat_dims

    # ------------------------------------------------------------------------------------------------ head
    def _build_head(self, feats, dfeats, fdims):
        """All levels in one launch per layer, activations of all levels in ONE buffer (bias gradients are one reduction)."""
        eng, n, L, frozen, req = self.eng, self.n, lib(), self.frozen, self._req
        dims = self.dims
        vox = [d[0] * d[1] * d[2] for d in fdims]
        self.total_vox = n * sum(vox)

        def level_views(t):
            out, o = [], 0
            for d, v in zip(fdims, vox):
                out.append(t[o:o + n * v].view(n, *d, t.shape[-1])); o += n * v
            return out
        hs = [req((self.total_vox, 256)) for _ in eng.hconv]
        dhs = [req((self.total_vox, 256)) for _ in eng.hconv]
        self.pred = req((self.total_vox, 128), torch.float32)
        self.dpred = req((self.total_vox, 128))             # zeroed by every loss_grad
        self.pred_levels, self.dpred_levels = level_views(self.pred), level_views(self.dpred)
        h_lv, dh_lv = [level_views(h) for h in hs], [level_views(h) for h in dhs]
        cur = feats
        for layer, nxt in zip(eng.hconv, h_lv):
            self._conv_fwd(layer, cur, fdims, nxt, fdims, relu=True)
            cur = nxt
        self._conv_fwd(eng.predictor, cur, fdims, self.pred_levels, fdims, out_fp32=True)
        self.dbg.update(hs=h_lv, dhs=dh_lv, dfeats=dfeats)
        self.strides = [tuple(dims[k] // d[k] for k in range(3)) for d in fdims]
        # the head's layers with the input and the output of each, all levels, and their gradients
        layers, ins, dins, douts = eng.hconv + [eng.predictor], [feats] + h_lv, [dfeats] + dh_lv, dh_lv + [self.dpred_levels]

        def head_bwd():
            for k in range(len(layers) - 1, -1, -1):
                self._param_grad(layers[k], douts[k], ins[k])
                if k == 0 and frozen:
                    break                                       # nothing reads the gradient of a frozen backbone's feature maps
                self._dgrad(layers[k], douts[k], dins[k], fdims)
                if k > 0:                                       # the input of layer k is the ReLU output of layer k - 1
                    check(L.nrpn_relu_backward(_p(dhs[k - 1]), _p(hs[k - 1]), dhs[k - 1].numel(), self.f16, _stream()), "relu_backward")
            A, hd, pr = eng.A, eng.head, eng.predictor          # the fused predictor's gradients: cls and bbox rows are separate parameters
            eng.grad_of(hd.cls_logits.weight).copy_(pr.dw[:A].reshape(-1)); eng.grad_of(hd.bbox_pred.weight).copy_(pr.dw[A:eng.n_pred].reshape(-1))
            eng.grad_of(hd.cls_logits.bias).copy_(pr.db[:A]); eng.grad_of(hd.bbox_pred.bias).copy_(pr.db[A:eng.n_pred])
        self.bwd.append(head_bwd)
        self.bwd_lo.append(min(eng.offsets[id(p_)][0] for p_ in eng.head.parameters()))

    def release(self):
        """Drops everything this plan holds -- pool views, anchors, launch lists, CUDA graphs -- when the engine evicts it or replaces the pool
        slots it points at.  The launch lists are closures over the plan, so without this the memory would wait for Python's cyclic collector.
        A released plan cannot run again."""
        self.__dict__.clear()
        self.released = True

    def _check_live(self):
        if getattr(self, "released", False):
            raise RuntimeError("nerf_rpn_b200: this training plan was released (evicted, or its buffers were replaced by a larger batch)")

    # ------------------------------------------------------------------------------------------------ helpers
    def _workspace(self, nbytes):
        return self._scratch_buf("workspace", max(int(nbytes), 1 << 20), torch.uint8)

    def _scratch_buf(self, name, numel, dtype):
        t = self._scratch.get(name)
        if t is None or t.numel() < numel or t.dtype != dtype:
            if t is not None:
                self.eng._drop_graphs()                     # captured graphs hold the old pointer
            t = torch.empty(int(numel), dtype=dtype, device=self.eng.device)
            self._scratch[name] = t
        return t[:numel]

    def _conv_fwd(self, layer: _TConv, xs, xds, ys, yds, res=None, res_dims=None, relu=False, out_fp32=False):
        """Records one launch of `layer`'s forward over the levels xs[i] (dims xds[i]) -> ys[i] (dims yds[i]); res: one level's residual added
        in the epilogue, read at res_dims (up-sampled when coarser)."""
        args = [ops.ConvLevelArgs(x, y, self.n, xd, yd, y.shape[-1], res=res, res_dims=res_dims, ldr=0 if res is None else res.shape[-1])
                for x, xd, y, yd in zip(xs, xds, ys, yds)]
        cout = ys[0].shape[-1]
        self.fwd.append(lambda: ops.conv3d_fprop(args, layer.fwd, layer.shift, layer.cin, cout, layer.taps, stride=layer.stride, relu=relu,
                                                 out_fp32=out_fp32))

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

    def _wgrad(self, dys, xs, taps, cout, cin, dw, layout):
        """dW of a stride-1 'same' conv from per-level channels-last (dY, X) pairs, written to `dw` (fp32) in `layout`."""
        d = ops.wgrad_desc(dys, xs, taps, cout, cin, self.f16)
        d.dw_layout = int(layout)
        need = lib().nrpn_conv3d_wgrad_workspace_bytes(ctypes.byref(d))
        if need == 0:
            raise ValueError(f"conv3d_wgrad: unsupported shape cout={cout} cin={cin}")
        ws = self._workspace(need)
        d.dw, d.workspace, d.workspace_bytes = dw.data_ptr(), ws.data_ptr(), ws.numel()
        check(lib().nrpn_conv3d_wgrad(ctypes.byref(d), _stream()), "conv3d_wgrad")

    def _param_grad(self, layer: _TConv, dys, xs):
        """layer.dw (nn.Conv3d's layout) from per-level (dY, X) pairs, and layer.db when the layer has a bias.  The levels of dY are consecutive
        rows of one buffer."""
        self._wgrad(dys, xs, layer.taps, layer.cout, layer.cin_real, layer.dw, layout=1)
        if layer.db is not None:
            self._bias_grad(layer, dys)

    def _bias_grad(self, layer: _TConv, dys):
        L = lib()
        ws = self._workspace(L.nrpn_bias_grad_workspace_bytes(layer.cout))
        rows = sum(dy.numel() for dy in dys) // layer.cout
        check(L.nrpn_bias_grad(_p(dys[0]), rows, layer.cout, layer.cout, self.f16, _p(layer.db), _p(ws), ws.numel(), _stream()), "bias_grad")

    def _dgrad(self, layer: _TConv, dys, dxs, dims, res=None):
        """Data gradient of a stride-1 layer: its mirrored / transposed operand run forward over the levels dys[i] -> dxs[i] (both dims[i]),
        + res (one level) in the epilogue."""
        args = [ops.ConvLevelArgs(dy, dx, self.n, d, d, dx.shape[-1], res=res, ldr=0 if res is None else res.shape[-1]) for dy, dx, d in zip(dys, dxs, dims)]
        ops.conv3d_fprop(args, layer.bwd, layer.bwd_shift, layer.bwd_cols, dxs[0].shape[-1], layer.taps)

    def _wgrad_stem(self, dy0):
        st = self.eng.stem
        dwp = self._scratch_buf("stem_dw", len(st.taps) * 64 * 64, torch.float32)
        self._wgrad([dy0], [self.packed], st.taps, 64, 64, dwp, layout=0)
        check(lib().nrpn_gather_pack(_p(dwp), _p(st.scatter_idx), st.dw.numel(), None, _p(st.dw), self.f16, _stream()), "gather_pack(stem grad)")

    def _make_block_bwd(self, e, x, xd, dx, od, y1, a1, y2, a2, y3, out, yd, dout, s):
        eng, L, n = self.eng, lib(), self.n
        cin = e["c1"].cin_real
        dt = eng.act_dtype

        def f():
            g = self._scratch_buf("g_skip", out.numel(), dt).view_as(out)        # masked gradient of the block output = skip-branch gradient
            dy3 = self._scratch_buf("dy3", y3.numel(), dt).view_as(y3)
            self._bn_bwd(e["bn3"], dout, out, y3, dy3, g, True)
            da2 = self._scratch_buf("da2", a2.numel(), dt).view_as(a2)
            self._param_grad(e["c3"], [dy3], [a2])
            self._dgrad(e["c3"], [dy3], [da2], [od])
            dy2 = self._scratch_buf("dy2", y2.numel(), dt).view_as(y2)
            self._bn_bwd(e["bn2"], da2, a2, y2, dy2, None, True)
            da1 = self._scratch_buf("da1", a1.numel(), dt).view_as(a1)
            self._param_grad(e["c2"], [dy2], [a1])
            self._dgrad(e["c2"], [dy2], [da1], [od])
            dy1 = self._scratch_buf("dy1", y1.numel(), dt).view_as(y1)
            self._bn_bwd(e["bn1"], da1, a1, y1, dy1, None, True)
            if s == 1:
                xs = x
            else:                                                               # stride-2 1^3 convs read the even voxels of x
                xs = self._scratch_buf("x_s2", n * od[0] * od[1] * od[2] * cin, dt).view(n, *od, cin)
                check(L.nrpn_stride2(_p(x), _p(xs), n, xd[0], xd[1], xd[2], cin, 0, _stream()), "stride2 gather")
            if e["ds"] is None:                                                 # identity skip (not a stage's first block): dx = dgrad_c1(dy1) + g
                self._param_grad(e["c1"], [dy1], [xs])
                self._dgrad(e["c1"], [dy1], [dx], [od], res=g)
                return
            dyd = self._scratch_buf("dyd", yd.numel(), dt).view_as(yd)
            self._bn_bwd(e["bnd"], g, None, yd, dyd, None, False)
            self._param_grad(e["c1"], [dy1], [xs])
            self._param_grad(e["ds"], [dyd], [xs])
            t1 = self._scratch_buf("t1", n * od[0] * od[1] * od[2] * cin, dt).view(n, *od, cin)
            self._dgrad(e["c1"], [dy1], [t1], [od])
            if s == 1:                                                          # stage 0: dx = dgrad_ds(dyd) + dgrad_c1(dy1)
                self._dgrad(e["ds"], [dyd], [dx], [od], res=t1)
                return
            # stages 1..3: the sum, zero-stuffed to x's grid, is added to the lateral part fpn_bwd has already written into dx
            t2 = self._scratch_buf("t2", n * od[0] * od[1] * od[2] * cin, dt).view(n, *od, cin)
            self._dgrad(e["ds"], [dyd], [t2], [od], res=t1)
            full = self._scratch_buf("dx_tmp", dx.numel(), dt).view_as(dx)
            check(L.nrpn_stride2(_p(t2), _p(full), n, xd[0], xd[1], xd[2], cin, 1, _stream()), "stride2 scatter")
            check(L.nrpn_add_inplace(_p(dx), _p(full), dx.numel(), self.f16, _stream()), "add_inplace")
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

    def _pack_input(self):
        ops.pack_stem_input(self._src, self.packed, density_to_alpha=self._alpha)

    def _set_input(self, grids):
        """The caller's batch for the stem packing: a stacked (N,4,X,Y,Z) grid, or a list of scenes whose padded extent is this plan's dims.
        An fp32 grid in neither memory order the packing reads in place is packed from a contiguous copy."""
        self._alpha = self.eng.density_to_alpha()
        if isinstance(grids, (list, tuple)):
            if len(grids) != self.n or ops.padded_extent(grids) != tuple(self.dims):
                raise ValueError(f"nerf_rpn_b200: this plan trains {self.n} scenes padded to {self.dims}")
            self._src = [g if ops._stem_layout(g, stacked=False, copy_ok=True) is not None else g.contiguous() for g in grids]
            self._sizes = [tuple(int(v) for v in g.shape[-3:]) for g in grids]
            return
        self._src = grids if ops._stem_layout(grids, stacked=True, copy_ok=True) is not None else grids.contiguous()
        self._sizes = None

    def padding_masks(self):
        """(N, anchors) uint8 padding masks of the current batch (None when no scene is padded): AnchorGenerator3D.get_padding_masks."""
        if self._sizes is None or all(s == tuple(self.dims) for s in self._sizes):
            return None
        return ops.anchor_padding_mask(self._sizes, self.dims, self.feat_dims, self.eng.A, device=self.eng.device)

    def forward_loss(self, grids, targets, w_obj=1.0, w_reg=None, w_2d=None, eval_2d=False):
        """Forward launches, target assignment, sampling, losses; fills d(pred) for the weighted sum w_obj * L_obj + w_reg * L_reg (+ w_2d * L_2d).
        grids: the stacked batch or the list of differently sized scenes (see RPNTrainEngine.forward_backward)."""
        self._check_live()
        eng, n = self.eng, self.n
        eng.forward_count += 1
        self._set_input(grids)
        self.fwd[0]()                                               # stem packing reads the caller's grid: its pointer changes from step to step
        _replay_static(self._graphs, "fwd", self.fwd[1:])
        anchors = self._anchors()
        self.valid = valid = self.padding_masks()
        samples = []
        forced = getattr(self, "forced_samples", None)         # tests: (pos, neg) index tensors per mesh instead of the sampler's draw
        for i in range(n):
            gt = targets[i].to(device=eng.device, dtype=torch.float32).contiguous()
            vi = None if valid is None else valid[i]
            if gt.numel() == 0:                                     # background mesh (rpn.py:246-250): every anchor is a negative
                labels = torch.zeros(anchors.shape[0], dtype=torch.float32, device=eng.device)
                if vi is not None:                                  # ... except those in the padding (rpn.py:283-285): -1
                    labels = vi.to(torch.float32) - 1.0
                pos, neg = self._sample(labels)
                samples.append((pos, neg, torch.zeros((0, 7 if eng.rotated else 6), dtype=torch.float32, device=eng.device)))
                continue
            labels, idx = ops.assign_targets(anchors, gt, vi, eng.rpn.fg_iou_thresh, eng.rpn.bg_iou_thresh, True)
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

    def _put_dpred(self, i, level, vox, cols, g, add):
        """Writes the per-positive gradient rows g (n_pos, code) of mesh i to where _gather_deltas found the deltas in d(pred): assigned (g already
        in d(pred)'s dtype), or with add=True added to what is there in fp32 and rounded once."""
        for l, dp in enumerate(self.dpred_levels):
            m = level == l
            if m.any():
                view, rows = dp[i].reshape(-1, 128), vox[m].view(-1, 1)
                view[rows, cols[m]] = (view[rows, cols[m]].float() + g[m]).to(view.dtype) if add else g[m]

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
                self._put_dpred(i, level, vox, cols, g * (w_2d * eng.loss_scale), add=True)
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
        anchors = self._anchors()
        total = torch.zeros((), dtype=torch.float32, device=eng.device)
        for i, (pos, neg, gtp) in enumerate(self.last_samples):
            if pos.numel() == 0:
                continue
            deltas, level, vox, cols = self._gather_deltas(i, pos)
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
                self._put_dpred(i, level, vox, cols, (g * (w_reg * eng.loss_scale)).to(self.dpred.dtype), add=False)
        eng.losses[1] = total

    def backward(self):
        """Backward launches in reverse construction order.  Gradients become final from the END of the flat bucket (head, FPN) towards
        its start (stem): every time >= bucket_elems new elements are final their all-reduce is launched on the comm stream, overlapping
        the dgrad / wgrad of the layers below (run_rpn.py:235-236: DDP's bucketed all-reduce during loss.backward())."""
        self._check_live()
        eng = self.eng
        if not (eng.world > 1 and eng.overlap_allreduce):
            self.allreduce_calls = 0
            _replay_static(self._graphs, "bwd", list(reversed(self.bwd)))
            return
        sched = {k: (lo, hi) for k, lo, hi in bucket_schedule(self.bwd_lo, eng.n_params, eng.bucket_elems, lowest=self.bwd_lo[0])}
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
