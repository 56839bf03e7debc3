"""Access to the staged, UNMODIFIED reference (oracle/_ref/nerf_rpn, see oracle/build_ref.py) -- TEST INFRASTRUCTURE.

Only tests/, __graft_entry__.smoke() and bench.py's reference/incumbent legs may import this; the product package
(nerf_rpn_b200/) never does.

`load()` imports the reference's own modules (`model.*`, `eval`, `datasets`) from the staged copy with its real native op
`sort_vertices` (K1, built by its own setup.py for sm_90) when a GPU is present, and returns them in a namespace.  The
reference imports by bare module name (`from model.utils import ...`, run_rpn.py:14-22), so the staged directory is put on
sys.path for the duration of the import and the bare names are removed from sys.modules afterwards: the loaded classes keep
working (they hold their module objects) and nothing leaks into later imports (e.g. dropin/model.py in the same process).
"""
import importlib
import os
import sys
import types

from .build_ref import CUDA_OP, k1_path, ref_root

_BARE = ("model", "eval", "datasets", "sort_vertices", "run_rpn", "run_fcos")
_cached = None


def available() -> bool:
    return ref_root() is not None


def load(need_k1: bool = True):
    """-> SimpleNamespace with the reference's modules; raises RuntimeError when the staged copy is absent."""
    global _cached
    if _cached is not None:
        return _cached
    root = ref_root()
    if root is None:
        raise RuntimeError("oracle/_ref is not staged: run `python oracle/build_ref.py` in the build container")
    import torch
    stash = {k: v for k, v in sys.modules.items() if k.split(".")[0] in _BARE}
    for k in stash:
        del sys.modules[k]
    paths = [root]
    if torch.cuda.is_available() and k1_path() is not None:
        paths.insert(0, CUDA_OP)                       # the real K1 extension
    elif need_k1:
        raise RuntimeError("the reference's sort_vertices extension needs a CUDA device (and oracle/_ref built)")
    sys.path[:0] = paths
    try:
        if "wandb" not in sys.modules:
            try:
                importlib.import_module("wandb")
            except Exception:                          # optional logger of run_rpn.py, never used by the tests
                sys.modules["wandb"] = types.ModuleType("wandb")
        ns = types.SimpleNamespace(root=root)
        ns.utils = importlib.import_module("model.utils")
        ns.anchor = importlib.import_module("model.anchor")
        ns.feature_extractor = importlib.import_module("model.feature_extractor")
        ns.nerf_rpn = importlib.import_module("model.nerf_rpn")
        ns.rpn = importlib.import_module("model.rpn")
        ns.oriented_iou_loss = importlib.import_module("model.rotated_iou.oriented_iou_loss")
        ns.box_intersection_2d = importlib.import_module("model.rotated_iou.box_intersection_2d")
        ns.fcos = importlib.import_module("model.fcos.fcos")
        ns.fpn = importlib.import_module("model.fpn")
        ns.eval = importlib.import_module("eval")
        ns.datasets = importlib.import_module("datasets")
        ns.sort_vertices = sys.modules.get("sort_vertices")
    finally:
        for p in paths:
            sys.path.remove(p)
        for k in [k for k in sys.modules if k.split(".")[0] in _BARE]:
            del sys.modules[k]
        sys.modules.update(stash)
    _cached = ns
    return ns


ANCHOR_SIZES = ((8,), (16,), (32,), (64,),)
ASPECT = (((1., 1., 1.), (1., 1., 2.), (1., 2., 2.), (1., 1., 3.), (1., 3., 3.)),) * 4


def build_reference_model(rotated=False, seed=0, spread=0.0, layers=(3, 4, 6, 3), **rpn_kw):
    """The reference's ResNet50-FPN + anchor head + wrapper, reference init under torch.manual_seed(seed) (run_rpn.py:171-216).
    spread > 0 multiplies cls_logits.weight so that objectness is not ~0.5 everywhere (SURVEY 8d's score-spread variant)."""
    import torch
    ref = load()
    torch.manual_seed(seed)
    bb = ref.feature_extractor.ResNet_FPN_256(ref.feature_extractor.Bottleneck, list(layers), input_dim=4, is_max_pool=True)
    ag = ref.anchor.AnchorGenerator3D(ANCHOR_SIZES, ASPECT)
    head = ref.anchor.RPNHead(256, ag.num_anchors_per_location()[0], 4, rotate=rotated)
    if spread:
        with torch.no_grad():
            head.cls_logits.weight.mul_(spread)
    kw = dict(rpn_pre_nms_top_n_test=2500, rpn_post_nms_top_n_test=2500, rpn_nms_thresh=0.3, rpn_score_thresh=0.0, rotated_bbox=rotated)
    kw.update(rpn_kw)
    return ref.nerf_rpn.NeRFRegionProposalNetwork(bb, ag, head, **kw)
