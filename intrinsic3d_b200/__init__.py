"""intrinsic3d_b200 — H100-native engine for Intrinsic3D's joint refinement hot path.

The compute path lives in csrc/ (sm_90a CUDA behind the C-ABI of include/i3d_c_api.h);
`engine.Engine` is the Python host-side mirror used by tests and bench.py.
"""
__version__ = "0.1.0"
