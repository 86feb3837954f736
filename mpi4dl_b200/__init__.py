"""mpi4dl_b200 -- H100-native (sm_90a) spatial-parallel convolution engine behind the torchgems API.

Layout (only what the hot path needs):
    csrc/            hand-written sm_90a CUDA kernels + the C ABI (include/spconv.h)
    libspconv.so     built in-tree by build.py (nvcc -gencode arch=compute_90a,code=sm_90a)
    _lib.py          ctypes binding (no fallback: raises when the library is missing)
    torchgems/       host-side mirror of the reference's torchgems package for this path
"""
__version__ = "0.1.0"
