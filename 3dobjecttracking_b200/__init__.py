"""3dobjecttracking_b200 — H100-native (sm_90a) implementation of M3T's per-frame pose-optimisation
hot path behind a C ABI (include/m3t_b200.h), plus the host-side mirrors of the reference interface.

The package name starts with a digit, so import it with
    importlib.import_module("3dobjecttracking_b200")

    .capi   ctypes binding of libm3t_b200.so (the CUDA path; fails loudly when it cannot be loaded)
    .synth  seeded synthetic workloads (BASELINE.json configs)
    ._build in-tree nvcc / g++ builds
"""
from . import _build, model_io, roofline, sharding, synth  # noqa: F401


def __getattr__(name):
    if name == "capi":
        import importlib
        return importlib.import_module(__name__ + ".capi")
    raise AttributeError(name)
