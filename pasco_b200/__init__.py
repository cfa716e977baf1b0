"""pasco_b200 — H100-native (sm_90a) sparse-voxel engine behind PaSCo's operator surface.

    pasco_b200.me       MinkowskiEngine-compatible API (the drop-in boundary; compat/MinkowskiEngine re-exports it)
    pasco_b200.ops      tensor-level wrappers / autograd Functions over the C-ABI
    pasco_b200._lib     ctypes binding of libpasco_sm100.so (include/pasco_sm100.h)
    pasco_b200.build    nvcc build of the in-tree shared library

No CPU fallback exists: ops raise if the library is missing or no CUDA device is present.
"""
__version__ = "0.1.0"
