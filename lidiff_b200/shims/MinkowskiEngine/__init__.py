"""`import MinkowskiEngine as ME` -> lidiff_b200.me (H100-native operator surface)."""
from lidiff_b200.me import *  # noqa: F401,F403
from lidiff_b200.me import (CoordinateManager, MinkowskiAlgorithm, MinkowskiBatchNorm, MinkowskiConvolution,  # noqa: F401
                            MinkowskiConvolutionTranspose, MinkowskiReLU, MinkowskiSyncBatchNorm, SparseTensor,
                            SparseTensorQuantizationMode, TensorField, cat, utils)

__version__ = "0.5.4+lidiff_b200"
