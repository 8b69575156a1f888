"""surfelmeshing_b200 — Hopper-native (sm_90a, H100) per-frame surfel reconstruction.

Drop-in for the hot path of puzzlepaint/surfelmeshing: depth pre-processing and
CUDASurfelReconstruction::Integrate()/Regularize() as hand-written CUDA kernels behind a
C ABI (include/surfel_b200.h, libsurfel_b200.so). This package holds the kernels (csrc/),
the build recipe, the ctypes bindings and a Python mirror of the reference interface used
by the tests and the benchmark. There is no CPU fallback.
"""
from ._lib import (IntegrateParams, PreprocessParams, StreamDesc, StreamStats, SurfelError, load_product,
                   EXPORTED_SYMBOLS, LIB_PATH)
from .reconstruction import (CUDASurfelReconstruction, BilateralFilteringAndDepthCutoffCUDA,
                             OutlierDepthMapFusionCUDA, ErodeDepthMapCUDA, CopyWithoutBorderCUDA,
                             ComputeNormalsAndDropBadPixelsCUDA, ComputePointRadiiAndRemoveIsolatedPixelsCUDA,
                             invert_rigid)

__all__ = [
    "IntegrateParams", "PreprocessParams", "StreamDesc", "StreamStats", "SurfelError", "load_product",
    "EXPORTED_SYMBOLS", "LIB_PATH", "CUDASurfelReconstruction", "BilateralFilteringAndDepthCutoffCUDA",
    "OutlierDepthMapFusionCUDA", "ErodeDepthMapCUDA", "CopyWithoutBorderCUDA",
    "ComputeNormalsAndDropBadPixelsCUDA", "ComputePointRadiiAndRemoveIsolatedPixelsCUDA", "invert_rigid",
]
