"""Drop-in for the reference's pybind module `sort_vertices` (nerf_rpn/model/rotated_iou/cuda_op/sort_vert.cpp:32-34):
put this directory on PYTHONPATH and the reference's own cuda_ext.py:4 (`import sort_vertices`) binds to this package's kernel."""
from nerf_rpn_b200.ops import sort_vertices_forward  # noqa: F401
