"""nerf_rpn_b200 -- CUDA implementation of the NeRF-RPN voxel RPN hot path for the H100 (sm_90a).

Python here is host-side glue mirroring the reference's module interface; all computation happens in
libnerf_rpn_b200.so (hand-written CUDA, see nerf_rpn_b200/csrc).  There is no CPU or eager-PyTorch fallback.
"""
__version__ = "0.1.0"
