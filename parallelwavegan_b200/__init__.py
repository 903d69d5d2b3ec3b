"""parallelwavegan_b200 -- H100-native (sm_90a) vocoder hot path behind the
``parallel_wavegan`` model/loss API.

``models`` / ``layers`` / ``losses`` mirror the reference namespaces (classes are
looked up by name from the yaml configs, train.py:1364-1381) and dispatch every
forward to hand-written CUDA kernels in ``libpwgb.so`` through the C ABI declared
in ``include/pwgb.h``.  There is no CPU or PyTorch fallback: if the library is
missing or a tensor is not on a CUDA device, the call raises.
"""

__version__ = "0.1.0"
