"""moleculekit_b200 -- H100-native voxel-descriptor and trajectory-distance engine.

Drop-in for ONE hot path of Acellera/moleculekit (SURVEY.md section 8):

    moleculekit.tools.voxeldescriptors.getVoxelDescriptors / getCenters
    moleculekit.projections.metricdistance.MetricDistance / MetricSelfDistance (.project)
    moleculekit.occupancy_utils / moleculekit.distance_utils (the Cython kernels underneath)

Python host code -> ctypes C-ABI (include/mkb200.h) -> hand-written CUDA kernels for sm_90a (H100).
PyTorch tensors are the device container only.  There is no CPU fallback.
"""
__version__ = "0.1.0"

from . import _lib  # noqa: F401  (does not dlopen until first use)


def library_path() -> str:
    return _lib.LIB_PATH
