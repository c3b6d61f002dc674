"""kubeai_b200 — H100-native in-process inference engine behind KubeAI's proxy/router seam.

Python here is a thin ctypes driver over the C-ABI library (kubeai_b200/lib/libb200engine.so,
declared in include/b200engine.h); all compute is hand-written sm_90a CUDA.
"""
from ._lib import B200Error, lib  # noqa: F401

__version__ = "0.1.0"
