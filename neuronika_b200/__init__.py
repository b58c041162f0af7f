"""neuronika_b200 -- H100-native dense forward/backward hot path of neuronika.

Device tensors live in HBM; every operator is a hand-written sm_90a CUDA kernel reached through
the C ABI in include/nk_b200.h (libnk_b200.so).  Importing this package without the built library
raises ImportError: there is no CPU fallback."""
from . import _lib
from ._lib import NkError
from .device import BF16, F32, CuArray, Device
from . import ops
from . import variable, nn, optim
from .variable import (Reduction, Status, Var, VarDiff, cat, from_ndarray, full, ones, rand, set_fusion, stack, zeros)
from .nn import (AdaptiveAvgPool1d, AdaptiveAvgPool2d, AdaptiveAvgPool3d, AvgPool1d, AvgPool2d, AvgPool3d, BatchNorm1d,
                 BatchNorm2d, BatchNorm3d, Embedding, LayerNorm, MaxPool1d, MaxPool2d, MaxPool3d)

__all__ = ["Device", "CuArray", "F32", "BF16", "NkError", "ops", "variable", "nn", "optim", "Var", "VarDiff",
           "Reduction", "Status", "zeros", "ones", "full", "rand", "from_ndarray", "set_fusion", "cat", "stack",
           "MaxPool1d", "MaxPool2d", "MaxPool3d", "AvgPool1d", "AvgPool2d", "AvgPool3d", "AdaptiveAvgPool1d",
           "AdaptiveAvgPool2d", "AdaptiveAvgPool3d", "BatchNorm1d", "BatchNorm2d", "BatchNorm3d", "LayerNorm",
           "Embedding"]
