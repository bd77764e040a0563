"""gen6d_b200 -- H100-native (sm_90a) implementation of the Gen6D inference hot path.

Host side: Python classes that mirror the reference's `network.{detector,selector,refiner}` and
`estimator.Gen6DEstimator` interfaces (same names, arguments, checkpoint format).
Device side: hand-written CUDA kernels behind a C-ABI shared library (include/gen6d_b200.h,
gen6d_b200/csrc/), loaded with ctypes.  There is no CPU fallback: importing
`gen6d_b200.network` works everywhere (parameter containers only), but any compute call raises
if libgen6d_b200.so is missing or no CUDA device is present.
"""
__version__ = '0.1.0'
