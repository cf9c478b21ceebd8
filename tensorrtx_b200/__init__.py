"""tensorrtx_b200 -- H100-native (sm_90a) detection decode / NMS / pre-process hot path.

Product = libtrtx_hot.so (C ABI, include/trtx_hot.h) + this thin host-side mirror of the
reference's plugin interface.  Importing `tensorrtx_b200.plugins` requires the built library
(python -m tensorrtx_b200.build); there is no CPU or PyTorch fallback.
"""
__version__ = "0.1.0"
