"""gpujpeg_b200 -- H100-native JPEG encode/decode hot path behind the libgpujpeg C API.

The product is the C-ABI shared library ``gpujpeg_b200/lib/libgpujpeg.so.0`` (host C + hand-written
sm_90a CUDA kernels, see ``include/gpujpeg_b200.h``).  This Python package is a thin ctypes mirror of
that API for tests, benchmarks and multi-GPU drivers; it never computes anything itself and raises
if the library cannot be built/loaded (there is no CPU fallback).
"""
from .api import (  # noqa: F401
    Decoder,
    Encoder,
    GpuJpegError,
    ImageParameters,
    Parameters,
    Transcoder,
    lib,
    library_path,
    version,
)
