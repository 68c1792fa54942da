"""rav1e_b200 — CUDA backend (sm_90a, H100) for rav1e's RDO inner loop.

The product is the C-ABI shared library `libb200rdo.so` (include/b200rdo.h) built from
rav1e_b200/csrc/*.cu.  This Python package is plumbing for tests, bench.py and
torch.distributed sharding: a ctypes binding (`backend`) and tile/shard helpers (`shard`).
There is no CPU fallback anywhere in this package: a missing library or a missing GPU
raises immediately.
"""
from . import backend  # noqa: F401

__all__ = ["backend"]
