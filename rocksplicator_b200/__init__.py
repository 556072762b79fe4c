"""rocksplicator_b200 — H100-native engine for Rocksplicator's sharded-replica hot path.

Package contents: csrc/ (CUDA kernels + the C ABI of include/rsp_b200.h), host/ (C++ mirror of the
reference's rocksdb:: / replicator:: / admin:: interfaces), engine.py (ctypes binding),
write_batch.py (WriteBatch wire format helper).
"""
from .write_batch import WriteBatch  # noqa: F401
