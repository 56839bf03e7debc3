"""Training steps of ResNet50-FPN + anchor head (BASELINE config 4: one 160x256x256 scene, --rotated_bbox, 16 planted oriented boxes, bf16) with
the full backward pass and with a frozen backbone (RPNTrainEngine(freeze_backbone=True), run_rpn.py --freeze_backbone), timed alternately in one
process after both have captured their CUDA graphs.

Prints one JSON line: per mode the step time from CUDA events (median of the rounds), the TFLOP the step executes (convolution MACs x 2 from the
layer shapes: forward, weight gradients and data gradients it runs), the resulting TFLOP/s, the peak torch.cuda.max_memory_allocated() while the
mode's engine was built and warmed up (above what was allocated before it), the plan pool's bytes, and the card's name and power limit read in
the same run.  Usage: python tools/train_frozen_bench.py [--steps 10] [--rounds 5] [--warmup 4]
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

DIMS = (160, 256, 256)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except Exception as e:                                              # noqa: BLE001
        pl = f"unavailable ({type(e).__name__})"
    return name, pl


def step_flop(model, dims, n_pred):
    """(full, frozen) FLOP of one training step on one scene: 2 x MACs of every convolution the step runs, at the layers' real channel counts."""
    from nerf_rpn_b200.engine import _down
    bb, head = model.backbone, model.rpn.head

    def conv(c, d, cout=None):
        co, ci, *k = c.weight.shape
        return 2 * math.prod(d) * (cout or co) * ci * math.prod(k)
    d1 = _down(dims)
    stem = conv(bb.conv1, d1)
    backbone, xd, stage_dims = 0, _down(d1), []
    for stage in bb.layers:
        for blk in stage:
            od = _down(xd) if blk.stride == 2 else xd
            backbone += sum(conv(c, od) for c in (blk.conv1, blk.conv2, blk.conv3)) + (conv(blk.downsample[0], od) if blk.downsample is not None else 0)
            xd = od
        stage_dims.append(xd)
    fpn = sum(conv(m, d) for m, d in zip(bb.latlayers, reversed(stage_dims))) + sum(conv(m, d) for m, d in zip(bb.smooths, reversed(stage_dims[:3])))
    convs = [m for m in head.conv if isinstance(m, torch.nn.Conv3d)]
    hconv = sum(conv(c, d) for c in convs for d in stage_dims)
    pred = sum(conv(head.cls_logits, d, n_pred) for d in stage_dims)              # the fused cls | bbox predictor: one 1^3 GEMM
    fwd = stem + backbone + fpn + hconv + pred
    full = fwd + fwd + (fwd - stem)                                               # forward + wgrad of every conv + dgrad of all but the stem
    first = sum(conv(convs[0], d) for d in stage_dims)
    frozen = fwd + (hconv + pred) + (hconv - first + pred)                        # forward + the head's wgrad + its dgrad above the first conv
    return full, frozen


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_frozen_bench: needs a CUDA device")
    from bench import build_model
    from tests.test_gpu_train import _planted
    grid, gt = _planted(DIMS, 16, 11, True)
    grid, gt = grid.cuda()[None], [gt.cuda()]
    name, power = card()
    engines, out = {}, {"card": name, "power_limit": power, "dims": DIMS, "steps_per_round": args.steps, "rounds": args.rounds}
    for mode in ("frozen", "full"):
        torch.manual_seed(0)
        model = build_model(rotated=True, spread=0.0).cuda().train()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        eng = model.train_engine(precision="bf16", lr=1e-4, weight_decay=0.01, clip_grad_norm=0.1, reg_loss_weight=5.0, seed=0,
                                 freeze_backbone=(mode == "frozen"))
        for _ in range(args.warmup):                                  # two eager steps, then the captured graphs
            eng.train_step(grid, gt)
        torch.cuda.synchronize()
        st = eng.cache_stats()
        full_f, frozen_f = step_flop(model, DIMS, eng.n_pred)
        engines[mode] = eng
        out[mode] = {"tflop_per_step": round((frozen_f if mode == "frozen" else full_f) / 1e12, 3),
                     "peak_allocated_gib": round((torch.cuda.max_memory_allocated() - base) / 2**30, 2),
                     "pool_gib": round(st["pool_bytes"] / 2**30, 2), "graphs": st["graphs"]}
    times = {m: [] for m in engines}
    for _ in range(args.rounds):
        for mode, eng in engines.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.steps):
                eng.train_step(grid, gt)
            b.record()
            b.synchronize()
            times[mode].append(a.elapsed_time(b) / args.steps)
    for mode in engines:
        ms = statistics.median(times[mode])
        out[mode].update(ms_per_step=round(ms, 2), ms_min=round(min(times[mode]), 2), ms_max=round(max(times[mode]), 2),
                         tflops=round(out[mode]["tflop_per_step"] / ms * 1e3, 1))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
