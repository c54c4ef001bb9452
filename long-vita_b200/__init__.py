"""long-vita_b200: H100-native (sm_90a) implementation of Long-VITA's long-context hot path.

Python host code over a C-ABI CUDA library (``include/lvb200.h`` / ``lib/liblvb200.so``).  The
product path never falls back to PyTorch math: every operator in :mod:`long_vita_b200.ops` raises
``RuntimeError`` if the CUDA extension is missing or a call fails.
"""
__version__ = "0.1.0"
