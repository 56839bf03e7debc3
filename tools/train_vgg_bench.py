"""Training steps of VGG-EF and VGG-AF FPN + anchor head (one 160x256x256 scene, --rotated_bbox, 16 planted oriented boxes, bf16) on the CUDA
engine, and the unmodified reference's own autograd step (fp32 and under torch.autocast(bf16): forward, backward, clip_grad_norm_, AdamW) on the
same card, all timed alternately in one process after the engines have captured their CUDA graphs.

Prints one JSON line: per backbone the engine's step time from CUDA events (median of the rounds), the TFLOP the step executes (convolution
MACs x 2 from the layer shapes: forward, weight gradients and data gradients), the resulting TFLOP/s and the plan pool's bytes; the reference's
step times; and the card's name and power limit read in the same run.
Usage: python tools/train_vgg_bench.py [--steps 5] [--rounds 5] [--warmup 4] [--ref-steps 2]
"""
import argparse
import json
import math
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tools.train_frozen_bench import card  # noqa: E402

DIMS = (160, 256, 256)


def step_flop(model, dims, n_pred):
    """FLOP of one full training step on one scene: 2 x MACs of every convolution the step runs, at the layers' real channel counts."""
    from nerf_rpn_b200.engine import _down
    bb, head = model.backbone, model.rpn.head

    def conv(c, d, cout=None):
        co, ci, *k = c.weight.shape
        return 2 * math.prod(d) * (cout or co) * ci * math.prod(k)
    mods = list(bb.layers.children())
    d1 = _down(dims)
    stem = conv(mods[0], d1)
    backbone, xd, stage_dims = 0, _down(d1), []
    for grp in mods[-4:]:
        for m in grp:
            if isinstance(m, torch.nn.Conv3d):
                backbone += conv(m, xd)
            elif isinstance(m, torch.nn.MaxPool3d):
                xd = _down(xd)
        stage_dims.append(xd)
    neck = bb.fpn_neck
    fpn = sum(conv(m, d) for m, d in zip(neck.lateral_convs, stage_dims)) + sum(conv(m, d) for m, d in zip(neck.fpn_convs, stage_dims))
    hconv = sum(conv(c, d) for c in head.conv if isinstance(c, torch.nn.Conv3d) for d in stage_dims)
    pred = sum(conv(head.cls_logits, d, n_pred) for d in stage_dims)
    fwd = stem + backbone + fpn + hconv + pred
    return fwd + fwd + (fwd - stem)                                     # forward + wgrad of every conv + dgrad of all but the stem


def build(cfg, reference=False):
    from oracle import ref_gpu
    torch.manual_seed(0)
    if reference:
        ref = ref_gpu.load()
        bb = ref.feature_extractor.VGG_FPN(cfg, 4, True, 160)
        ag = ref.anchor.AnchorGenerator3D(ref_gpu.ANCHOR_SIZES, ref_gpu.ASPECT)
        head = ref.anchor.RPNHead(256, ag.num_anchors_per_location()[0], 4, rotate=True)
        return ref.nerf_rpn.NeRFRegionProposalNetwork(bb, ag, head, rotated_bbox=True).cuda().train()
    from nerf_rpn_b200.model.anchor import AnchorGenerator3D, RPNHead
    from nerf_rpn_b200.model.feature_extractor import VGG_FPN
    from nerf_rpn_b200.model.nerf_rpn import NeRFRegionProposalNetwork
    ag = AnchorGenerator3D(ref_gpu.ANCHOR_SIZES, ref_gpu.ASPECT)
    return NeRFRegionProposalNetwork(VGG_FPN(cfg, 4, True, 160), ag, RPNHead(256, ag.num_anchors_per_location()[0], 4, rotate=True),
                                     rotated_bbox=True).cuda().train()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--ref-steps", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_vgg_bench: needs a CUDA device")
    from oracle import ref_gpu
    from tests.test_gpu_train import _planted
    grid, gt = _planted(DIMS, 16, 11, True)
    grid, gt = grid.cuda(), gt.cuda()
    name, power = card()
    out = {"card": name, "power_limit": power, "dims": DIMS, "steps_per_round": args.steps, "rounds": args.rounds}
    runs = {}
    for cfg in ("EF", "AF"):
        model = build(cfg)
        eng = model.train_engine(precision="bf16", lr=1e-4, weight_decay=0.01, clip_grad_norm=0.1, reg_loss_weight=5.0, seed=0)
        for _ in range(args.warmup):                                  # two eager steps, then the captured graphs
            eng.train_step(grid[None], [gt])
        torch.cuda.synchronize()
        st = eng.cache_stats()
        tflop = step_flop(model, DIMS, eng.n_pred) / 1e12
        out[f"vgg_{cfg}"] = {"tflop_per_step": round(tflop, 3), "pool_gib": round(st["pool_bytes"] / 2**30, 2), "graphs": st["graphs"]}
        runs[f"vgg_{cfg}"] = (lambda e=eng: e.train_step(grid[None], [gt]), args.steps)
    if ref_gpu.available():
        for dt in (None, torch.bfloat16):
            m = build("EF", reference=True)
            params = [p for p in m.parameters() if p.requires_grad]
            opt = torch.optim.AdamW(params, lr=1e-4, weight_decay=0.01)

            def ref_step(m=m, opt=opt, params=params, dt=dt):
                with torch.autocast("cuda", dtype=dt, enabled=dt is not None):
                    _, losses, _ = m([grid], [gt])
                    loss = losses["loss_objectness"] + 5.0 * losses["loss_rpn_box_reg"]
                loss.backward()
                torch.nn.utils.clip_grad_norm_(params, 0.1)
                opt.step()
                opt.zero_grad()
            ref_step()
            torch.cuda.synchronize()
            key = "reference_vgg_EF_" + ("fp32" if dt is None else "autocast_bf16")
            out[key] = {}
            runs[key] = (ref_step, args.ref_steps)
    else:
        out["reference"] = "oracle/_ref not staged: not measured"
    times = {k: [] for k in runs}
    for _ in range(args.rounds):
        for key, (fn, steps) in runs.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(steps):
                fn()
            b.record()
            b.synchronize()
            times[key].append(a.elapsed_time(b) / steps)
    for key in runs:
        ms = statistics.median(times[key])
        out[key].update(ms_per_step=round(ms, 2), ms_min=round(min(times[key]), 2), ms_max=round(max(times[key]), 2))
        if "tflop_per_step" in out[key]:
            out[key]["tflops"] = round(out[key]["tflop_per_step"] / ms * 1e3, 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
