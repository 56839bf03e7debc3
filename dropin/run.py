#!/usr/bin/env python
"""Launch one of the reference's UNMODIFIED drivers (run_rpn.py / run_fcos.py) on this package's CUDA path:

    python dropin/run.py /path/to/NeRF_RPN/nerf_rpn/run_rpn.py --mode eval --backbone_type resnet ...

`python run_rpn.py` puts the script's own directory first on sys.path, so the reference's `model/` package would shadow the
shim; this launcher registers dropin/model.py as `model` (and `sort_vertices`) first, adds the driver's directory for its
`datasets` / `eval` modules, and executes the script file as __main__ with runpy -- not one line of it is changed.
"""
import os
import runpy
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def main():
    if len(sys.argv) < 2 or not os.path.isfile(sys.argv[1]):
        sys.exit("usage: python dropin/run.py /path/to/nerf_rpn/run_rpn.py [driver arguments ...]")
    script = os.path.abspath(sys.argv[1])
    # the driver's own directory comes right after the shim (ahead of site-packages: its `datasets` / `eval` modules would otherwise
    # lose to installed packages of the same name); its `model/` package is never imported because `model` is already registered
    sys.path[:0] = [HERE, ROOT, os.path.dirname(script)]
    import model  # noqa: F401  (dropin/model.py: registers nerf_rpn_b200.model as the top-level package `model`)
    sys.argv = [script] + sys.argv[2:]
    runpy.run_path(script, run_name="__main__")


if __name__ == "__main__":
    main()
