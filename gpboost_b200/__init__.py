"""gpboost_b200 — CUDA-native (H100, sm_90a) GP + tree hot path behind GPBoost's own C API.

`GPModel` mirrors the reference's Python class for the hot-path configurations and binds
`lib_gpboost_b200.so` (built in-tree by `gpboost_b200.build`) through ctypes. No CPU fallback exists.
"""
from .basic import GPModel, GPBoostError  # noqa: F401
from .libpath import load_lib, find_lib_path  # noqa: F401
from .engine import train  # noqa: F401

__version__ = "0.1.0"
