"""gypsum_b200 -- H100-native GPS L1 C/A correlation engine behind gypsum's acquisition / tracking call surface.

Host code is Python over a C ABI (include/gypsum_b200.h, ctypes); the arithmetic runs in hand-written sm_90a
CUDA (gypsum_b200/csrc).  There is no CPU fallback: importing the compute modules without the built shared
library, or using them without a GPU, raises.
"""
__version__ = "0.1.0"
