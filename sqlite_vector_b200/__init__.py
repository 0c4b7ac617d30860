"""sqlite_vector_b200 — H100-native brute-force distance scan behind sqlite-vector's SQL surface.

The product is the pair of shared libraries built from csrc/ (see include/vsb200.h):
  lib/libvsb200.so  C-ABI scan engine (hand-written sm_90a CUDA)
  lib/vector.so     SQLite loadable extension (entry point sqlite3_vector_init) + the engine
This package is the thin host-side mirror used by tests and bench.py: ctypes bindings (api.py) and the
torch.distributed row-shard driver (shard.py: one process per GPU; the heads travel over NVLink peer memory).
There is no CPU fallback anywhere in this package.
"""
from .api import Engine, Group, Index, VsbError, load_engine  # noqa: F401

__all__ = ["Engine", "Group", "Index", "VsbError", "load_engine"]
