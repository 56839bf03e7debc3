"""Training steps of ResNet50-FPN + anchor head (--rotated_bbox, bf16) on batches of two differently sized scenes, as the reference's datasets
produce them (--resolution 160 caps the longest side only), against the same number of steps on equal-size batches at the padded maximum.

Prints ms/step, peak torch.cuda.max_memory_reserved() of each leg (reset between the two), the plans and CUDA graphs alive, and the card's name and power limit read in the
same run.  Usage: python tools/train_ragged_bench.py [--steps 24] [--warmup 4] [--seed 0]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

SHAPES = [(160, 128, 96), (128, 160, 112), (144, 112, 160), (160, 144, 128), (112, 136, 120), (96, 160, 144)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except Exception as e:                                              # noqa: BLE001
        pl = f"unavailable ({type(e).__name__})"
    return name, pl


def scene(dims, gen):
    """A (4,X,Y,Z) scene in the dataset's channels-last memory order, and 12 planted oriented boxes."""
    g = torch.rand(*dims, 4, generator=gen).cuda().permute(3, 0, 1, 2)
    d = torch.tensor(dims, dtype=torch.float32)
    size = torch.rand(12, 3, generator=gen) * 40.0 + 8.0
    ctr = torch.rand(12, 3, generator=gen) * (d - 16.0) + 8.0
    return g, torch.cat([ctr, size, (torch.rand(12, 1, generator=gen) - 0.5) * 3.14159], 1).cuda()


def run(eng, batches, steps, warmup):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()                            # the peak of this leg only (warm-up and plan builds included)
    for i in range(warmup):
        eng.train_step(*batches[i % len(batches)])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        losses = eng.train_step(*batches[(warmup + i) % len(batches)])
        losses.tolist()                                             # the losses are read back every step, like a training loop logs them
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    return ms, torch.cuda.max_memory_reserved()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_ragged_bench: needs a CUDA device")
    from bench import build_model
    from nerf_rpn_b200 import train as T

    rng = random.Random(args.seed)
    gen = torch.Generator().manual_seed(args.seed)
    pool = {s: scene(s, gen) for s in SHAPES}
    pairs = [(rng.choice(SHAPES), rng.choice(SHAPES)) for _ in range(args.steps + args.warmup)]
    ragged = [([pool[a][0], pool[b][0]], [pool[a][1], pool[b][1]]) for a, b in pairs]
    pmax = tuple(max(s[k] for s in SHAPES) for k in range(3))
    eq_grid = torch.stack([scene(pmax, gen)[0].contiguous() for _ in range(2)])
    eq = [(eq_grid, [pool[SHAPES[0]][1], pool[SHAPES[1]][1]])]

    model = build_model(rotated=True, spread=0.0).cuda().train()
    eng = model.train_engine(precision="bf16", lr=1e-4, weight_decay=0.01, clip_grad_norm=0.1, reg_loss_weight=5.0)
    name, power = card()
    ms_r, mem_r = run(eng, ragged, args.steps, args.warmup)
    st = eng.cache_stats()
    padded = sorted({tuple(max(a[k], b[k]) for k in range(3)) for a, b in pairs})
    ms_e, mem_e = run(eng, eq, args.steps, args.warmup)
    out = {
        "card": name, "power_limit": power, "steps": args.steps, "warmup": args.warmup, "seed": args.seed,
        "ragged": {"ms_per_step": round(ms_r, 2), "max_memory_reserved_gib": round(mem_r / 2**30, 2), "distinct_padded_shapes": len(padded),
                   "plans_alive": st["plans"], "graphs_alive": st["graphs"], "pool_gib": round(st["pool_bytes"] / 2**30, 2),
                   "pool_growths": st["pool_growths"], "scratch_growths": st["scratch_growths"], "plan_cache": T.PLAN_CACHE},
        "equal_size_at_padded_max": {"dims": pmax, "ms_per_step": round(ms_e, 2), "max_memory_reserved_gib": round(mem_e / 2**30, 2),
                                     "plans_alive": eng.cache_stats()["plans"], "graphs_alive": eng.cache_stats()["graphs"]},
        "scene_shapes": SHAPES, "batch": 2,
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
