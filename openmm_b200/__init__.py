"""openmm_b200 -- host-side Python binding of the CUDA-native (sm_90a) OpenMM hot path.

The product is native code: `libb200md.so` (C-ABI, include/b200md.h, CUDA kernels for sm_90a under csrc/) and the
OpenMM Platform plugin `libOpenMMB200.so` (plugin/).  This package only binds the C-ABI for tests and bench.py and
provides builders for the benchmark systems.  There is no CPU fallback.
"""
from .engine import Engine, EngineError          # noqa: F401
from .systems import SystemDesc                  # noqa: F401
from . import systems                            # noqa: F401
