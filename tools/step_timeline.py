#!/usr/bin/env python
"""Timeline of one steady-state headline step: where the step's wall time goes between the main-stream kernels.

Builds bench.py's headline model (build_model, 4 scenes of 160x256x256 per step, default precision), runs it through the
engine's captured graphs, times K steps with CUDA events (profiler off), then traces a few more steps with torch.profiler
(CUDA activity only) and takes one step from the trace: from one input-packing kernel (the first launch of every step) on the
main stream to the next.  Writes under the directory OUT:
  launches.csv   every kernel that starts inside the step: name, stream, start / end (us from the step's start), and for
                 main-stream kernels the idle time before it and the side-stream kernel time overlapping it;
  summary.json   step wall time (events and trace), main-stream kernel sum, main-stream idle, side-stream overlap of the
                 convolutions, and the largest idle gaps;
  trace.pt.trace.json  the raw trace.
Usage: python tools/step_timeline.py OUT [--steps K]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402


def _gpu_desc():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return torch.cuda.get_device_name()


def _union(intervals):
    out = []
    for a, b in sorted(intervals):
        if out and a <= out[-1][1]:
            out[-1][1] = max(out[-1][1], b)
        else:
            out.append([a, b])
    return out


def _overlap(a, b, union):
    return sum(max(0.0, min(b, y) - max(a, x)) for x, y in union)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", help="output directory")
    ap.add_argument("--steps", type=int, default=20, help="steps timed with CUDA events")
    ap.add_argument("--batch", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("step_timeline: needs a CUDA device")
    os.makedirs(args.out, exist_ok=True)
    torch.cuda.set_device(0)

    from nerf_rpn_b200 import precision as nprec
    model = bench.build_model(precision=nprec.resolve(None)).cuda().eval()
    eng = model.engine()
    grids = [bench.synth_scene(i, "dataset").permute(1, 2, 3, 0).contiguous().cuda() for i in range(4)]
    batches = [torch.stack([grids[(i + k) % 4] for k in range(args.batch)], 0).permute(0, 4, 1, 2, 3) for i in range(4)]

    with torch.no_grad():
        for i in range(6):
            plan = eng.forward_device(batches[i % 4])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.steps):
            plan = eng.forward_device(batches[i % 4])
        torch.cuda.current_stream().wait_event(plan.done)
        e1.record()
        torch.cuda.synchronize()
        event_ms = e0.elapsed_time(e1) / args.steps

        prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA])
        with prof:
            for i in range(5):
                plan = eng.forward_device(batches[i % 4])
            torch.cuda.synchronize()
    trace = os.path.join(args.out, "trace.pt.trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        ev = json.load(f)
    ev = ev["traceEvents"] if isinstance(ev, dict) else ev
    kernels = [dict(name=e["name"], stream=e.get("args", {}).get("stream"), t0=float(e["ts"]), t1=float(e["ts"]) + float(e["dur"]))
               for e in ev if e.get("cat") == "kernel"]
    kernels.sort(key=lambda k: k["t0"])
    packs = [k for k in kernels if "pack_stem" in k["name"]]
    if len(packs) < 4:
        raise SystemExit(f"step_timeline: found {len(packs)} input-packing kernels in the trace, need at least 4")
    main_stream = packs[2]["stream"]
    s0, s1 = packs[2]["t0"], packs[3]["t0"]                  # the third traced step: graphs and both buffer parities warm
    step = [k for k in kernels if s0 <= k["t0"] < s1]
    main = [k for k in step if k["stream"] == main_stream]
    side_union = _union([(k["t0"], k["t1"]) for k in kernels if k["stream"] != main_stream])

    rows, idle, gaps, conv_overlap, conv_time = [], 0.0, [], 0.0, 0.0
    prev_end = s0
    for k in step:
        on_main = k["stream"] == main_stream
        gap = side = None
        if on_main:
            gap = max(0.0, k["t0"] - prev_end)
            idle += gap
            gaps.append((gap, k["name"][:80]))
            prev_end = max(prev_end, k["t1"])
            side = _overlap(k["t0"], k["t1"], side_union)
            if "conv3d" in k["name"]:
                conv_overlap += side
                conv_time += k["t1"] - k["t0"]
        rows.append((k["name"], k["stream"], k["t0"] - s0, k["t1"] - s0, gap, side))
    idle += max(0.0, s1 - prev_end)

    with open(os.path.join(args.out, "launches.csv"), "w") as f:
        f.write("name,stream,start_us,end_us,idle_before_us,side_overlap_us\n")
        for name, stream, a, b, gap, side in rows:
            f.write(f"\"{name}\",{stream},{a:.1f},{b:.1f},{'' if gap is None else f'{gap:.1f}'},{'' if side is None else f'{side:.1f}'}\n")
    wall_us = s1 - s0
    main_sum = sum(k["t1"] - k["t0"] for k in main)
    summary = {
        "gpu": _gpu_desc(), "batch": args.batch,
        "step_ms_events": round(event_ms, 3), "step_ms_trace": round(wall_us / 1e3, 3),
        "main_stream_kernels": len(main), "main_stream_kernel_sum_ms": round(main_sum / 1e3, 3),
        "main_stream_idle_ms": round(idle / 1e3, 3), "main_stream_busy_share": round(main_sum / wall_us, 4),
        "side_stream_kernels": len(step) - len(main),
        "conv_ms": round(conv_time / 1e3, 3), "side_overlap_of_convs_ms": round(conv_overlap / 1e3, 3),
        "largest_idle_gaps_us": [(round(g, 1), n) for g, n in sorted(gaps, reverse=True)[:12]],
    }
    with open(os.path.join(args.out, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps(summary, indent=1))


if __name__ == "__main__":
    main()
