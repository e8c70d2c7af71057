"""compute_engine_b200 -- an H100-native (sm_90a) implementation of the one hot
path of larq/compute-engine: LceQuantize -> LceBconv2d (-> LceBMaxPool2d /
LceDequantize), behind the reference's TFLite custom-op surface.

Layout
  csrc/lce_b200_kernels.cuh   hand-written CUDA kernels
  csrc/lce_b200.cu            C-ABI (include/lce_b200.h)
  csrc/host/                  C++ TFLite custom-op shell + graph host
  capi.py                     ctypes binding of the C-ABI (torch tensors in/out)
There is no CPU compute path in this package: every op fails loudly when the CUDA
library or a CUDA device is missing.
"""
from . import capi  # noqa: F401

__all__ = ["capi"]
__version__ = "0.1.0"
