"""mad_icp_b200 -- H100 (sm_90a) implementation of MAD-ICP's per-scan registration hot path.

Layout: csrc/ (CUDA kernels + C ABI + host flat-tree builder + device tree build/ingest), csrc/facade/ (C++
classes and pybind modules with the reference's names: pymadtree, pymadicp, pypeline, pyvector -> pybind/),
csrc/adapter/ (backend TU the reference's own Pipeline links against), engine.py (ctypes handles used by the
tests and bench.py), distributed.py (multi-GPU plumbing), synth.py (synthetic inputs).
"""
from .engine import DeskewPlan, DeviceTree, FlatTree, Registrar, MadIcpError, VoxelMap  # noqa: F401

__version__ = "0.1.0"
