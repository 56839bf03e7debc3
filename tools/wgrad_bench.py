#!/usr/bin/env python
"""Time the weight-gradient GEMM at the RPN head layer's size (3^3 256->256 over P2..P5 of one 160x256x256 scene)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nerf_rpn_b200 import ops  # noqa: E402

dims = [(40, 64, 64), (20, 32, 32), (10, 16, 16), (5, 8, 8)]
g = torch.Generator(device="cuda").manual_seed(0)
xs = [torch.randn((1, *d, 256), device="cuda", generator=g).to(torch.bfloat16) for d in dims]
dys = [torch.randn((1, *d, 256), device="cuda", generator=g).to(torch.bfloat16) for d in dims]
taps = [(a - 1, b - 1, c - 1) for a in range(3) for b in range(3) for c in range(3)]
vox = sum(d[0] * d[1] * d[2] for d in dims)
fl = 2.0 * vox * 256 * 256 * 27
for _ in range(2):
    dw = ops.conv3d_wgrad(dys, xs, taps)
torch.cuda.synchronize()
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
a.record()
for _ in range(5):
    dw = ops.conv3d_wgrad(dys, xs, taps)
b.record(); torch.cuda.synchronize()
ms = a.elapsed_time(b) / 5
print(f"wgrad head layer: {ms:.3f} ms, {fl / ms / 1e9:.1f} TFLOP/s algorithmic")
