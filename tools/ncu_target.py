#!/usr/bin/env python
"""Target for `ncu --nvtx --nvtx-include "target/"`: one full-size scene (eager), then the kernels we want captured,
each inside the NVTX range "target": the RPN-head conv layer (wgmma implicit GEMM over P2..P5), the stem conv,
pack_stem_input, maxpool and the whole post-processing (top-k, decode, NMS)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from nerf_rpn_b200.model.nerf_rpn import NeRFRegionProposalNetwork  # noqa: E402

backbone, ag, head = bench.build_modules()
model = NeRFRegionProposalNetwork(backbone, ag, head, rpn_pre_nms_top_n_test=2500, rpn_post_nms_top_n_test=2500,
                                  rpn_nms_thresh=0.3).cuda().eval()
eng = model.engine()
eng.use_graph = False
x = bench.synth_scene(0).cuda()[None]
plan = eng.forward_device(x)
torch.cuda.synchronize()
which = os.environ.get("NCU_TARGET", "head")
torch.cuda.nvtx.range_push("target")
if which == "head":
    plan.head_launches[1]()
elif which == "stem":
    plan.launches[1]()                                                    # stem conv (halo-slab kernel)
elif which == "l0c2":
    [f for f in plan.launches if "L0.c2" in plan.names.get(id(f), ("",))[0]][0]()
elif which in ("l0c3", "l0c1", "l1c3", "lat3"):
    key = {"l0c3": "L0.c3+res", "l0c1": "L0.c1", "l1c3": "L1.c3+res", "lat3": "lat3+up"}[which]
    [f for f in plan.launches if key in plan.names.get(id(f), ("",))[0]][-1]()
elif which == "misc":
    plan.launches[0](); plan.launches[1](); plan.launches[2]()          # pack, stem conv, maxpool
    for f in plan._post[0]:
        f()
torch.cuda.synchronize()
torch.cuda.nvtx.range_pop()
