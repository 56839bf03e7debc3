#!/usr/bin/env python
"""BASELINE config 5: oriented 3-D IoU + NMS throughput sweep, 1k .. 1M proposals per scene, 1 x H100.
Inputs per SURVEY.md 8(d): centres U[0,256)^3*(1,1,0.625), sizes U[4,48], theta U[-pi/2,pi/2), scores U[0,1), seed 0,
threshold 0.3, 1 and 4 level groups; cull mode 0 (exact-zero culls only: provably the reference's keep set) and 3 (+ geometric ratio culls).  Algorithmic bytes: 32 B per input box + 8 B per kept index."""
import json
import math
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nerf_rpn_b200 import ops  # noqa: E402


def main():
    rows = []
    for mode, groups in ((0, 1), (0, 4), (3, 1), (3, 4)):
        ops.set_nms_cull_mode(mode)
        for n in ((1000, 4000, 16000, 64000, 256000, 1000000) if mode == 0 else (64000, 256000, 1000000)):
            g = torch.Generator().manual_seed(0)
            c = torch.rand(n, 3, generator=g) * torch.tensor([256.0, 256.0, 160.0])
            s = torch.rand(n, 3, generator=g) * 44 + 4
            th = (torch.rand(n, 1, generator=g) - 0.5) * math.pi
            boxes = torch.cat([c, s, th], 1).cuda().contiguous()
            scores = torch.rand(n, generator=g).cuda()
            grp = torch.randint(0, groups, (n,), generator=g).int().cuda() if groups > 1 else None
            for _ in range(2):
                keep, nk = ops.nms_device(boxes, scores, grp, 0.3)
            torch.cuda.synchronize()
            ts = []
            for _ in range(3):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); keep, nk = ops.nms_device(boxes, scores, grp, 0.3); b.record(); torch.cuda.synchronize()
                ts.append(a.elapsed_time(b))
            ms = sorted(ts)[1]
            k = int(nk.item())
            rows.append(dict(cull_mode=mode, n=n, groups=groups, kept=k, ms=ms, boxes_per_s=n / (ms * 1e-3), gb_per_s=(32 * n + 8 * k) / (ms * 1e-3) / 1e9))
            print(rows[-1], flush=True)
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump(rows, open("gpurun_out/nms_sweep.json", "w"), indent=1)


if __name__ == "__main__":
    main()
