"""acsfit: H100-native decision engine behind the acs-engine autoscaler's per-tick hot path.

Host-side mirror of the reference's `autoscaler` package for that path (same class and
function names), with the arithmetic done by hand-written sm_90a kernels in libacsfit.so.
Importing the package does not load CUDA; constructing an engine does, and fails loudly
when the extension or a GPU is missing (there is no CPU fallback).
"""
__all__ = ["KubePodStatus", "KubePod", "KubeNode", "KubeResource"]


def __getattr__(name):  # lazy re-exports, like reference autoscaler/__init__.py:1-5
    if name in __all__:
        from . import kube
        return getattr(kube, name)
    raise AttributeError(name)
