"""tensoir_b200 — H100-native (sm_90a) implementation of TensoIR's volume-rendering hot path.

Python/PyTorch host code owns tensors and autograd and mirrors the reference's public surface
(TensorVMSplit, relight_utils, Renderer_TensoIR_train); per-sample work runs in hand-written CUDA kernels
behind the C ABI of include/tensoir_b200.h (csrc/, loaded with ctypes — no CPU fallback).
"""
from .tensorf import TensorVMSplit, AlphaGridMask, raw2alpha            # noqa: F401
from .tensorf_init import TensorVMSplit as TensorVMSplitInit            # noqa: F401
from .renderer import Renderer_TensoIR_train, OctreeRender_trilinear_fast  # noqa: F401
from . import relight_utils                                              # noqa: F401
from .evaluation import (compute_rescale_ratio, evaluation_iter_TensoIR, evaluation_iter_TensoIR_simple,  # noqa: F401
                         evaluation_iter_TensoIR_general_multi_lights)
from .mesh import convert_sdf_samples_to_ply, export_mesh, marching_cubes                   # noqa: F401

__version__ = "0.1.0"
