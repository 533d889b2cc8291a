"""bundlefusion_b200 -- H100-native (sm_90a) implementation of BundleFusion's per-frame hot path.

The product is the C-ABI shared library ``libbundlefusion_b200.so`` (include/*.h); this package is
its Python host-side mirror of the reference's class surface.  There is no CPU fallback.
"""
from . import _capi  # noqa: F401

__all__ = ["_capi"]
