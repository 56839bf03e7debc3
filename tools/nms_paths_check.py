#!/usr/bin/env python
"""Diagnostic: the keep list of one config-5 input (n boxes) from both NMS paths for large inputs (cell lists / plain chunked kept-list scan)
with the cull modes 0 / 1 / 3, each in its own process (the switches are read once per process)."""
import json
import os
import subprocess
import sys
import textwrap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
n = int(sys.argv[1]) if len(sys.argv) > 1 else 256000
groups = int(sys.argv[2]) if len(sys.argv) > 2 else 1
code = textwrap.dedent(f"""
    import sys, math, numpy as np, torch
    sys.path.insert(0, {ROOT!r})
    from nerf_rpn_b200 import ops
    n, groups = {n}, {groups}
    g = torch.Generator().manual_seed(0)
    c = torch.rand(n, 3, generator=g) * torch.tensor([256.0, 256.0, 160.0])
    s = torch.rand(n, 3, generator=g) * 44 + 4
    th = (torch.rand(n, 1, generator=g) - 0.5) * math.pi
    boxes = torch.cat([c, s, th], 1).cuda().contiguous()
    scores = torch.rand(n, generator=g).cuda()
    grp = torch.randint(0, groups, (n,), generator=g).int().cuda() if groups > 1 else None
    k, nk = ops.nms_device(boxes, scores, grp, 0.3)
    np.save(sys.argv[1], k[: int(nk.item())].cpu().numpy())
""")
import numpy as np
res = {}
os.makedirs("gpurun_out", exist_ok=True)
for name, env in (("cells", {}), ("plain", {"NRPN_NMS_CELLS": "0"})):
    for lens in ("0", "1", "3"):
        key = f"{name}_mode{lens}"
        out = f"gpurun_out/_paths_{key}.npy"
        r = subprocess.run([sys.executable, "-c", code, out], capture_output=True, text=True, env={**os.environ, **env, "NRPN_NMS_CULL_MODE": lens})
        if r.returncode != 0:
            print(key, "FAILED", r.stderr[-500:]); continue
        res[key] = np.load(out)
        print(key, res[key].shape[0], flush=True)
base = res.get("plain_mode0")
for k, v in res.items():
    same = v.shape == base.shape and bool((v == base).all())
    plain = res.get("plain_" + k.split("_")[1])
    same_mode = plain is not None and v.shape == plain.shape and bool((v == plain).all())
    print(f"{k}: kept {v.shape[0]}  == plain_mode0: {same}  == plain, same mode: {same_mode}  only_here {np.setdiff1d(v, base)[:8].tolist()}  "
          f"missing {np.setdiff1d(base, v)[:8].tolist()}")
