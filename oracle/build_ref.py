#!/usr/bin/env python
"""Recipe for oracle/_ref: the UNMODIFIED reference, staged so that it travels to the GPU box.

TEST INFRASTRUCTURE ONLY (the checker and the incumbent timing arm) -- nothing under nerf_rpn_b200/ imports this.

The reference (lyclyc52/NeRF_RPN) is a script directory (no setup.py / pyproject: `pip install --target baseline/_ref
/root/reference` fails, DESIGN.md section 5), so "installing" it is:
  1. copy /root/reference/nerf_rpn (Python sources, 660 KB) to oracle/_ref/nerf_rpn -- oracle/_ref/ is git-ignored
     (history stays free of reference sources) but NOT gpurun-ignored, so the copy ships with the snapshot;
  2. build the reference's ONE native op on the hot path, `sort_vertices` (model/rotated_iou/cuda_op/sort_vert.cpp,
     sort_vert_kernel.cu -- K1 of SURVEY.md 2.2) with its own setup.py, unmodified, TORCH_CUDA_ARCH_LIST=9.0, inside
     the copy (the reference tree is read-only).

On the GPU machine this gives the true GPU oracle (the reference's torch-CUDA IoU chain + K1 + Python NMS + cuDNN convs)
and the incumbent whose scenes/s bench.py reports next to ours.  `python oracle/build_ref.py` or build_ref() from
__graft_entry__.build(); a no-op when /root/reference is absent (the GPU box uses the staged files).
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = "/root/reference/nerf_rpn"
REF_DST = os.path.join(HERE, "_ref", "nerf_rpn")
CUDA_OP = os.path.join(REF_DST, "model", "rotated_iou", "cuda_op")


def ref_root():
    """Path of the staged reference (oracle/_ref/nerf_rpn) or None."""
    return REF_DST if os.path.isfile(os.path.join(REF_DST, "run_rpn.py")) else None


def k1_path():
    """Path of the built sort_vertices extension inside the staged copy, or None."""
    if not os.path.isdir(CUDA_OP):
        return None
    for f in os.listdir(CUDA_OP):
        if f.startswith("sort_vertices") and f.endswith(".so"):
            return os.path.join(CUDA_OP, f)
    return None


def build_ref(force: bool = False, verbose: bool = True):
    if not os.path.isdir(REF_SRC):
        if verbose:
            print(f"oracle/build_ref: {REF_SRC} absent; staged copy {'present' if ref_root() else 'ABSENT'}")
        return ref_root()
    if force and os.path.isdir(REF_DST):
        shutil.rmtree(REF_DST)
    if ref_root() is None:
        os.makedirs(os.path.dirname(REF_DST), exist_ok=True)
        shutil.copytree(REF_SRC, REF_DST, ignore=shutil.ignore_patterns("__pycache__", "*.pyc"), dirs_exist_ok=True)
    if k1_path() is None:
        env = dict(os.environ, TORCH_CUDA_ARCH_LIST="9.0", MAX_JOBS="4")
        log = os.path.join(HERE, "_ref", "k1_build.log")
        with open(log, "w") as f:
            rc = subprocess.call([sys.executable, "setup.py", "build_ext", "--inplace"], cwd=CUDA_OP, env=env, stdout=f, stderr=subprocess.STDOUT)
        if rc != 0 or k1_path() is None:
            raise RuntimeError(f"oracle/build_ref: building the reference's sort_vertices extension failed, see {log}")
        shutil.rmtree(os.path.join(CUDA_OP, "build"), ignore_errors=True)
    if verbose:
        print(f"oracle/build_ref: staged {REF_DST}; K1 = {os.path.basename(k1_path())}")
    return ref_root()


if __name__ == "__main__":
    build_ref(force="--force" in sys.argv)
