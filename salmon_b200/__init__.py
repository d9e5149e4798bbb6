"""salmon_b200 -- H100-native (sm_90a) hot path of Salmon quantification.

Only what the path needs: csrc/ (CUDA kernels + the C ABI in include/salmon_b200.h),
the ctypes binding (_capi), the host-side mirror of the reference's optimiser
interface (inference) and the synthetic workload generators (synth).
"""
from . import _capi  # noqa: F401
from ._capi import EMContext, EqClasses, SalmonB200Error, default_params  # noqa: F401

__all__ = ["EMContext", "EqClasses", "SalmonB200Error", "default_params"]
