"""Timing of the INCUMBENT: the unmodified reference (oracle/_ref) on the same GPU -- cuDNN fp32 / TF32 convolutions, ATen
pointwise kernels, the Python NMS loop and its own K1 extension (SURVEY.md 8(d): "also report the reference GPU path on the same
H100 since that is the real incumbent").  TEST / BENCH INFRASTRUCTURE: only bench.py's `reference_gpu` leg and tools/ call this.

Method = the reference's own benchmark() (run_rpn.py:594-617): eval mode, warm-up forwards, then `reps` forwards of
`model([grid])` each bracketed by CUDA events + synchronize, mean / std in ms.  The reference uses 10 + 300 repetitions on a
randn(4,200,200,130) grid; here the grid is the bench workload (U[0,1) 160x256x256) and the repetition count is bounded
(the Python NMS loop costs seconds per scene), both stated in the result.
"""
import time

import torch

from . import ref_gpu


def time_reference_gpu(dims=(160, 256, 256), rotated=False, spread=0.0, tf32=True, warmup=2, reps=5, seed=0, budget_s=60.0):
    """-> dict(ms_per_scene, std_ms, backbone_head_ms, proposals, reps, ...) or {"unavailable": reason}."""
    if not ref_gpu.available():
        return {"unavailable": "oracle/_ref not staged (python oracle/build_ref.py in the build container)"}
    if not torch.cuda.is_available():
        return {"unavailable": "no CUDA device"}
    model = ref_gpu.build_reference_model(rotated=rotated, seed=seed, spread=spread).cuda().eval()
    g = torch.Generator().manual_seed(1000)
    x = torch.rand(*dims, 4, generator=g).permute(3, 0, 1, 2).contiguous().cuda()
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.benchmark)
    torch.backends.cudnn.allow_tf32 = tf32
    torch.backends.cuda.matmul.allow_tf32 = tf32
    out = {}
    try:
        with torch.no_grad():
            t_start = time.perf_counter()
            for _ in range(warmup):
                res = model([x])
            torch.cuda.synchronize()
            per = (time.perf_counter() - t_start) / max(warmup, 1)
            reps = max(1, min(reps, int(budget_s / max(per, 1e-3))))
            times = []
            for _ in range(reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                res = model([x])
                b.record()
                torch.cuda.synchronize()
                times.append(a.elapsed_time(b))
            # network only (backbone + FPN + head: the cuDNN part), same methodology
            net = []
            for _ in range(max(3, reps)):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                feats = model.backbone(x[None])
                model.rpn.head(feats)
                b.record()
                torch.cuda.synchronize()
                net.append(a.elapsed_time(b))
        t = torch.tensor(times)
        out = {"ms_per_scene": float(t.mean()), "std_ms": float(t.std()) if len(times) > 1 else 0.0, "scenes_per_s": 1000.0 / float(t.mean()),
               "network_only_ms": float(torch.tensor(net[1:]).mean()), "proposals": int(res[0][1][0].shape[0]), "reps": reps, "warmup": warmup,
               "math": "cuDNN TF32 (PyTorch default: torch.backends.cudnn.allow_tf32=True)" if tf32 else "cuDNN fp32 (allow_tf32=False)",
               "method": "run_rpn.py:594-617 (CUDA events around model([grid]), eval mode), bounded repetitions",
               "workload": f"{'x'.join(map(str, dims))}x4 U[0,1) grid, ResNet50-FPN + anchor head ({'OBB' if rotated else 'AABB'}), seed-{seed} init"
                           + (f", cls_logits.weight x{spread:g}" if spread else ""),
               "torch": torch.__version__, "cudnn": torch.backends.cudnn.version()}
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.benchmark = old
        del model
        torch.cuda.empty_cache()
    return out


if __name__ == "__main__":
    import json
    import sys
    rot = "--rotated" in sys.argv
    for tf32 in (True, False):
        print(json.dumps(time_reference_gpu(rotated=rot, tf32=tf32, spread=30.0 if "--spread" in sys.argv else 0.0)), flush=True)
