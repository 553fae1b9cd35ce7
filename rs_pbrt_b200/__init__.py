"""rs_pbrt_b200 -- H100-native PathIntegrator hot path for rs_pbrt behind a C ABI (the package keeps its original name).

The product is rs_pbrt_b200/librs_pbrt_b200.so (hand-written CUDA for sm_90a + the C++ host mirror);
this package only holds the ctypes bindings and the synthetic scene generators used by tests/bench.
Importing the package does not load the library; the first call does, and fails loudly if it is missing.
"""
from . import _abi  # noqa: F401
from .host import GpuScene, HostScene, PbrtError, bvh_build, create_multi, pin_description, render_multi, unpin_description  # noqa: F401

__all__ = ["GpuScene", "HostScene", "PbrtError", "bvh_build", "create_multi", "render_multi", "pin_description", "unpin_description"]
