"""superlu_dist_b200 -- an H100-native (sm_90a) `pdgstrf3d` for SuperLU_DIST.

The product is the C-ABI shared library ``lib/libslu_b200.so`` (hand-written CUDA kernels + host
orchestration, ``include/slu_b200.h``).  This Python package is only the thin host-side mirror
used by the tests and the benchmark: ctypes bindings (``capi``), the producers of the hot path's
input in the reference's block layout (``hostlib``, ``problem``) and readers for the golden
fixtures dumped from the reference (``dumpio``).  Nothing here computes a factorization.
"""
from .problem import LUProblem  # noqa: F401

__all__ = ["LUProblem", "autograd"]


def __getattr__(name):
    # superlu_dist_b200.autograd imports torch: loaded on first use
    if name == "autograd":
        import importlib
        return importlib.import_module(".autograd", __name__)
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
