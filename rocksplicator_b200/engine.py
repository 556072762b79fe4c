"""ctypes binding of librsp_b200.so (include/rsp_b200.h): the product's Python face.

There is no CPU path behind these classes: if the CUDA library is missing or no GPU is visible the
constructors raise.  Method names on `Shard` follow the reference's rocksdb::DB / DbWrapper usage
(rocksdb_replicator/rocksdb_wrapper.cpp, rocksdb_admin/application_db.cpp).
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(HERE, "librsp_b200.so")

OK, NOT_FOUND, CORRUPTION, NOT_SUPPORTED, INVALID_ARGUMENT, IO_ERROR = 0, 1, 2, 3, 4, 5
INCOMPLETE = 7
MERGE_NONE, MERGE_COUNTER, MERGE_UINT64ADD, MERGE_APPEND, MERGE_CALLBACK, MERGE_STRING_APPEND = 0, 1, 2, 3, 4, 5
SHARD_ALLOW_INGEST_BEHIND = 1  # rsp_shard_open_ex flags
COMPACT_CHANGE_LEVEL = 1       # rsp_compact_ex flags

MERGE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                       C.c_size_t, C.c_void_p, C.c_void_p)


class EngineCfg(C.Structure):
    _fields_ = [("abi_version", C.c_uint32), ("max_shards", C.c_uint32), ("arena_bytes", C.c_uint64),
                ("staging_bytes", C.c_uint64), ("l0_compaction_trigger", C.c_uint32), ("reserved", C.c_uint32)]


class ShardOpts(C.Structure):
    _fields_ = [("merge_op", C.c_uint32), ("merge_delim", C.c_uint32), ("write_buffer_bytes", C.c_uint64),
                ("merge_fn", C.c_void_p), ("merge_state", C.c_void_p)]


class Stats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "latest_seq", "memtable_entries", "memtable_bytes", "n_runs", "run_entries", "run_bytes", "flushes",
        "compactions", "compaction_bytes_read", "compaction_bytes_written", "flush_comparison_sorts")]


EXPORTS = {
    # name: (restype, argtypes)
    "rsp_version": (C.c_char_p, []),
    "rsp_engine_create": (C.c_int, [C.c_int, C.POINTER(EngineCfg), C.POINTER(C.c_void_p)]),
    "rsp_engine_destroy": (None, [C.c_void_p]),
    "rsp_engine_device": (C.c_int, [C.c_void_p]),
    "rsp_engine_stream": (C.c_void_p, [C.c_void_p]),
    "rsp_shard_open": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(ShardOpts), C.POINTER(C.c_void_p)]),
    "rsp_shard_close": (C.c_int, [C.c_void_p]),
    "rsp_shard_index": (C.c_uint32, [C.c_void_p]),
    "rsp_shard_name": (C.c_char_p, [C.c_void_p]),
    "rsp_apply": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.c_uint64, C.POINTER(C.c_uint64)]),
    "rsp_write": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.POINTER(C.c_uint64)]),
    "rsp_apply_many": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p]),
    "rsp_apply_updates": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.POINTER(C.c_size_t)]),
    "rsp_multi_get_slices": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    "rsp_router_create": (C.c_int, [C.c_size_t, C.c_void_p, C.POINTER(C.c_void_p)]),
    "rsp_router_destroy": (None, [C.c_void_p]),
    "rsp_router_add_shard": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p]),
    "rsp_router_remove_shard": (C.c_int, [C.c_void_p, C.c_uint32]),
    "rsp_router_multi_get": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_size_t, C.c_void_p, C.c_void_p]),
    "rsp_router_multi_get_fixed": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                             C.c_size_t, C.c_void_p, C.c_void_p]),
    "rsp_router_apply_many": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p]),
    "rsp_latest_seq": (C.c_uint64, [C.c_void_p]),
    "rsp_set_latest_seq": (C.c_int, [C.c_void_p, C.c_uint64]),
    "rsp_last_error": (C.c_size_t, [C.c_void_p, C.c_char_p, C.c_size_t]),
    "rsp_get": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "rsp_multi_get": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_size_t, C.c_void_p, C.c_void_p]),
    "rsp_multi_get_fixed": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                      C.c_size_t, C.c_void_p, C.c_void_p]),
    "rsp_iter_create": (C.c_void_p, [C.c_void_p]),
    "rsp_iter_destroy": (None, [C.c_void_p]),
    "rsp_iter_seek_to_first": (None, [C.c_void_p]),
    "rsp_iter_seek_to_last": (None, [C.c_void_p]),
    "rsp_iter_seek": (None, [C.c_void_p, C.c_char_p, C.c_size_t]),
    "rsp_iter_next": (None, [C.c_void_p]),
    "rsp_iter_prev": (None, [C.c_void_p]),
    "rsp_iter_valid": (C.c_int, [C.c_void_p]),
    "rsp_iter_key": (C.c_void_p, [C.c_void_p, C.POINTER(C.c_size_t)]),
    "rsp_iter_value": (C.c_void_p, [C.c_void_p, C.POINTER(C.c_size_t)]),
    "rsp_iter_status": (C.c_int, [C.c_void_p]),
    "rsp_iter_set_upper_bound": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t]),
    "rsp_iter_seek_for_prev": (None, [C.c_void_p, C.c_char_p, C.c_size_t]),
    "rsp_snapshot_create": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "rsp_snapshot_release": (None, [C.c_void_p]),
    "rsp_snapshot_seq": (C.c_uint64, [C.c_void_p]),
    "rsp_snapshot_slot": (C.c_uint32, [C.c_void_p]),
    "rsp_get_at": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "rsp_multi_get_at": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_size_t, C.c_void_p, C.c_void_p]),
    "rsp_multi_get_at_device": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                          C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rsp_iter_create_at": (C.c_void_p, [C.c_void_p]),
    "rsp_multi_scan": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                 C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    "rsp_multi_scan_bounded": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    "rsp_multi_scan_reverse": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                         C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p,
                                         C.c_void_p]),
    "rsp_multi_scan_at": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                    C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    "rsp_multi_scan_reverse_at": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                            C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p,
                                            C.c_void_p]),
    "rsp_flush": (C.c_int, [C.c_void_p]),
    "rsp_compact": (C.c_int, [C.c_void_p]),
    "rsp_flush_all": (C.c_int, [C.c_void_p]),
    "rsp_compact_all": (C.c_int, [C.c_void_p]),
    "rsp_get_stats": (C.c_int, [C.c_void_p, C.POINTER(Stats)]),
    "rsp_ingest_sorted": (C.c_int, [C.c_void_p, C.c_size_t, C.c_char_p, C.c_void_p, C.c_char_p, C.c_void_p, C.c_int,
                                    C.POINTER(C.c_uint64)]),
    "rsp_ingest_sorted_behind": (C.c_int, [C.c_void_p, C.c_size_t, C.c_char_p, C.c_void_p, C.c_char_p, C.c_void_p]),
    "rsp_shard_behind_bytes": (C.c_uint64, [C.c_void_p]),
    "rsp_shard_open_ex": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(ShardOpts), C.c_uint32, C.POINTER(C.c_void_p)]),
    "rsp_compact_ex": (C.c_int, [C.c_void_p, C.c_uint32]),
    "rsp_multi_get_device": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                       C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rsp_multi_scan_device": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32,
                                        C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rsp_multi_scan_bounded_device": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                                C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                                C.c_void_p]),
    "rsp_multi_scan_reverse_device": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int,
                                                C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p,
                                                C.c_void_p, C.c_void_p]),
    "rsp_multi_scan_at_device": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int,
                                           C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p,
                                           C.c_void_p, C.c_void_p]),
    "rsp_multi_scan_reverse_at_device": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint32,
                                                   C.c_int, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64,
                                                   C.c_void_p, C.c_void_p, C.c_void_p]),
    "rsp_stage_build": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.POINTER(C.c_void_p)]),
    "rsp_stage_free": (None, [C.c_void_p]),
    "rsp_reserve": (C.c_int, [C.c_void_p, C.c_void_p]),
    "rsp_apply_staged_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "rsp_apply_staged_finish": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "rsp_last_kernel_ms": (C.c_float, [C.c_void_p, C.c_char_p]),
    "rsp_kernel_launches": (C.c_uint64, [C.c_void_p]),
    "rsp_debug_last_pending": (C.c_uint32, [C.c_void_p, C.c_void_p, C.c_uint32]),
    "rsp_debug_combiner_stats": (None, [C.c_void_p, C.c_int, C.c_void_p]),
    "rsp_debug_arena": (None, [C.c_void_p, C.c_void_p]),
}

_lib = None


def load_library():
    """dlopen librsp_b200.so and bind every symbol include/rsp_b200.h declares.  No compute."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise RuntimeError(
            f"{SO_PATH} is missing: build it with `python -m rocksplicator_b200.build` "
            "(the engine has no CPU fallback)")
    lib = C.CDLL(SO_PATH)
    for name, (res, args) in EXPORTS.items():
        fn = getattr(lib, name)  # AttributeError == a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _pack_keys(keys):
    """byte strings -> (blob, offsets): key i is blob[off[i] .. off[i+1])"""
    off = np.zeros(len(keys) + 1, dtype=np.uint64)
    np.cumsum(np.fromiter((len(k) for k in keys), dtype=np.uint64, count=len(keys)), out=off[1:])
    return np.frombuffer(b"".join(keys) + b"\0", dtype=np.uint8), off


def _handles(snapshots):
    """Snapshots (or None) -> the C array of their handles"""
    return (C.c_void_p * max(len(snapshots), 1))(*[s.h if s is not None else None for s in snapshots])


def _scan_records(out, n_out, st, n, stride):
    """the [u32 klen][u32 vlen][key][value] records of n scans at out + i * stride -> [(status, [(key, value)])].  A key
    that needs a host-side merge operator (RSP_MERGE_APPEND or RSP_MERGE_CALLBACK: vlen 0xffffffff, no value bytes; the
    scan's status is NotSupported in the host forms, 100 in the device forms) comes back as (key, None).  Device-folded
    operators (counter, uint64add, string append) always come back with their value."""
    res = []
    for i in range(n):
        recs, at = [], i * stride
        for _ in range(int(n_out[i])):
            kl = int(out[at:at + 4].view(np.uint32)[0])
            vl = int(out[at + 4:at + 8].view(np.uint32)[0])
            if vl == 0xffffffff:
                recs.append((out[at + 8:at + 8 + kl].tobytes(), None))
                at += 8 + kl
                continue
            recs.append((out[at + 8:at + 8 + kl].tobytes(), out[at + 8 + kl:at + 8 + kl + vl].tobytes()))
            at += 8 + kl + vl
        res.append((int(st[i]), recs))
    return res


class Iterator:
    """upper_bound: ReadOptions::iterate_upper_bound (exclusive; None = no bound)"""

    def __init__(self, shard, snapshot=None, upper_bound=None):
        self.lib = shard.lib
        self.h = self.lib.rsp_iter_create(shard.h) if snapshot is None else self.lib.rsp_iter_create_at(snapshot.h)
        self._shard = shard
        if upper_bound is not None:
            self.set_upper_bound(upper_bound)

    def set_upper_bound(self, key):
        rc = self.lib.rsp_iter_set_upper_bound(self.h, key, 0 if key is None else len(key))
        if rc != OK:
            raise RuntimeError(f"rsp_iter_set_upper_bound -> {rc}")

    def close(self):
        if self.h:
            self.lib.rsp_iter_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def seek_to_first(self): self.lib.rsp_iter_seek_to_first(self.h)
    def seek_to_last(self): self.lib.rsp_iter_seek_to_last(self.h)
    def seek(self, k): self.lib.rsp_iter_seek(self.h, k, len(k))
    def seek_for_prev(self, k): self.lib.rsp_iter_seek_for_prev(self.h, k, len(k))
    def next(self): self.lib.rsp_iter_next(self.h)
    def prev(self): self.lib.rsp_iter_prev(self.h)
    def valid(self): return bool(self.lib.rsp_iter_valid(self.h))
    def status(self): return self.lib.rsp_iter_status(self.h)

    def key(self):
        n = C.c_size_t()
        p = self.lib.rsp_iter_key(self.h, C.byref(n))
        return C.string_at(p, n.value) if n.value else b""

    def value(self):
        n = C.c_size_t()
        p = self.lib.rsp_iter_value(self.h, C.byref(n))
        return C.string_at(p, n.value) if n.value else b""


class Snapshot:
    """DB::GetSnapshot on one shard: reads through it see the shard as it was at `seq`.  Release it (or leave the
    `with` block) to let go of the HBM it pins; iterators created from it keep their own pins."""

    def __init__(self, shard):
        self.shard = shard
        self.lib = shard.lib
        h = C.c_void_p()
        rc = self.lib.rsp_snapshot_create(shard.h, C.byref(h))
        if rc != OK:
            raise RuntimeError(f"rsp_snapshot_create({shard.name}) -> {rc}")
        self.h = h
        self.seq = self.lib.rsp_snapshot_seq(h)
        self.slot = self.lib.rsp_snapshot_slot(h)

    def release(self):
        if self.h:
            self.lib.rsp_snapshot_release(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.release()

    def get(self, key: bytes, cap: int = 256):
        while True:
            buf = C.create_string_buffer(max(cap, 1))
            n = C.c_size_t()
            rc = self.lib.rsp_get_at(self.h, key, len(key), buf, cap, C.byref(n))
            if rc == INCOMPLETE:
                cap = n.value
                continue
            return (rc, buf.raw[:n.value]) if rc == OK else (rc, None)

    def multi_get(self, keys, stride=256):
        return self.shard.engine.multi_get_at([self] * len(keys), keys, stride)

    def iterator(self, upper_bound=None):
        return Iterator(self.shard, self, upper_bound)

    def scan(self, start=None, limit=None, end=None):
        """up to `limit` live entries from `start` (None: the first key) to `end` (exclusive; None: the last key)"""
        it = self.iterator(upper_bound=end)
        if start is None:
            it.seek_to_first()
        else:
            it.seek(start)
        out = []
        while it.valid() and (limit is None or len(out) < limit):
            out.append((it.key(), it.value()))
            it.next()
        it.close()
        return out


class Shard:
    """One DB ("segment%05d"): apply == DbWrapper::HandleReplicateResponse, write == WriteToLeader,
    latest_seq == LatestSequenceNumber, get/multi_get/iterator == the ApplicationDB read surface."""

    def __init__(self, engine, name, merge_op=MERGE_NONE, write_buffer_bytes=0, merge_fn=None, merge_delim=None,
                 allow_ingest_behind=False):
        """merge_delim: MERGE_STRING_APPEND's delimiter, one byte (b"," / b"\\0") or None for plain concatenation;
        allow_ingest_behind: DBOptions::allow_ingest_behind (ingest(..., behind=True); no compaction is bottom-most)"""
        self.engine = engine
        self.lib = engine.lib
        self.kind = "b200"
        delim = 0
        if merge_delim is not None:
            if len(merge_delim) != 1:
                raise ValueError("merge_delim is one byte or None")
            delim = 0x100 | bytes(merge_delim)[0]
        opts = ShardOpts(merge_op=merge_op, merge_delim=delim, write_buffer_bytes=write_buffer_bytes)
        self._merge_fn = None
        if merge_fn is not None:
            self._merge_fn = MERGE_FN(merge_fn)
            opts.merge_fn = C.cast(self._merge_fn, C.c_void_p)
        h = C.c_void_p()
        flags = SHARD_ALLOW_INGEST_BEHIND if allow_ingest_behind else 0
        rc = self.lib.rsp_shard_open_ex(engine.h, name.encode(), C.byref(opts), flags, C.byref(h))
        if rc != OK:
            raise RuntimeError(f"rsp_shard_open({name}) -> {rc}")
        self.h = h
        self.name = name
        self.index = self.lib.rsp_shard_index(h)

    def close(self):
        if self.h:
            self.lib.rsp_shard_close(self.h)
            self.h = None

    @property
    def last_error(self):
        buf = C.create_string_buffer(256)
        self.lib.rsp_last_error(self.h, buf, 256)
        return buf.value.decode()

    def apply(self, batch: bytes, ts_ms: int = 0) -> int:
        return self.lib.rsp_apply(self.h, batch, len(batch), ts_ms, None)

    def write(self, batch: bytes) -> int:
        return self.lib.rsp_write(self.h, batch, len(batch), None)

    def latest_seq(self) -> int:
        return self.lib.rsp_latest_seq(self.h)

    def get(self, key: bytes, cap: int = 256):
        while True:
            buf = C.create_string_buffer(max(cap, 1))
            n = C.c_size_t()
            rc = self.lib.rsp_get(self.h, key, len(key), buf, cap, C.byref(n))
            if rc == INCOMPLETE:
                cap = n.value
                continue
            return (rc, buf.raw[:n.value]) if rc == OK else (rc, None)

    def multi_get(self, keys, stride=256):
        res = self.engine.multi_get([self.index] * len(keys), keys, stride)
        return res

    def iterator(self, upper_bound=None):
        return Iterator(self, upper_bound=upper_bound)

    def snapshot(self):
        return Snapshot(self)

    def scan(self, start=None, limit=None, end=None):
        """up to `limit` live entries from `start` (None: the first key) to `end` (exclusive; None: the last key)"""
        it = self.iterator(upper_bound=end)
        if start is None:
            it.seek_to_first()
        else:
            it.seek(start)
        out = []
        while it.valid() and (limit is None or len(out) < limit):
            out.append((it.key(), it.value()))
            it.next()
        it.close()
        return out

    def flush(self): return self.lib.rsp_flush(self.h)
    def compact(self, change_level=False):
        """CompactRange(nullptr, nullptr); change_level=True also folds the ingested-behind tier in"""
        return self.lib.rsp_compact_ex(self.h, COMPACT_CHANGE_LEVEL if change_level else 0)

    def behind_bytes(self) -> int:
        """bytes held by the ingested-behind tier (0: empty)"""
        return self.lib.rsp_shard_behind_bytes(self.h)

    def ingest(self, sorted_kv, allow_global_seqno=True, behind=False) -> int:
        """DB::IngestExternalFile for sorted (key, value) pairs (see rocksplicator_b200/sst.py for SST files);
        behind=True: IngestExternalFileOptions::ingest_behind (allow_global_seqno plays no part)"""
        n = len(sorted_kv)
        koff = np.zeros(n + 1, dtype=np.uint64)
        voff = np.zeros(n + 1, dtype=np.uint64)
        np.cumsum(np.fromiter((len(k) for k, _ in sorted_kv), dtype=np.uint64, count=n), out=koff[1:])
        np.cumsum(np.fromiter((len(v) for _, v in sorted_kv), dtype=np.uint64, count=n), out=voff[1:])
        keys = b"".join(k for k, _ in sorted_kv) + b"\0"
        vals = b"".join(v for _, v in sorted_kv) + b"\0"
        if behind:
            return self.lib.rsp_ingest_sorted_behind(self.h, n, keys, koff.ctypes.data, vals, voff.ctypes.data)
        return self.lib.rsp_ingest_sorted(self.h, n, keys, koff.ctypes.data, vals, voff.ctypes.data,
                                          1 if allow_global_seqno else 0, None)

    def stats(self):
        st = Stats()
        self.lib.rsp_get_stats(self.h, C.byref(st))
        return {n: getattr(st, n) for n, _ in Stats._fields_}


class Engine:
    """One engine per GPU (shard_id -> GPU partitioning happens above, SURVEY §8e)."""

    def __init__(self, device=0, max_shards=0, arena_bytes=0, l0_compaction_trigger=0):
        self.lib = load_library()
        cfg = EngineCfg(abi_version=1, max_shards=max_shards, arena_bytes=arena_bytes,
                        l0_compaction_trigger=l0_compaction_trigger)
        h = C.c_void_p()
        rc = self.lib.rsp_engine_create(device, C.byref(cfg), C.byref(h))
        if rc != OK:
            raise RuntimeError(f"rsp_engine_create(device={device}) -> {rc}: no usable CUDA device "
                               "(the engine has no CPU fallback)")
        self.h = h
        self.device = device
        self.shards = {}

    def close(self):
        if self.h:
            for s in list(self.shards.values()):
                s.h = None
            self.lib.rsp_engine_destroy(self.h)
            self.h = None

    def open_shard(self, name, **kw):
        s = Shard(self, name, **kw)
        self.shards[name] = s
        return s

    # ---- batched calls (numpy in / numpy out; host memory) ----
    def apply_many(self, shard_ix, batches, ts_ms=None):
        """batches: list of bytes.  Returns int32 status per batch."""
        n = len(batches)
        six = np.ascontiguousarray(shard_ix, dtype=np.uint32)
        lens = np.fromiter((len(b) for b in batches), dtype=np.uint64, count=n)
        off = np.zeros(n + 1, dtype=np.uint64)
        np.cumsum(lens, out=off[1:])
        blob = np.frombuffer(b"".join(batches) + b"\0", dtype=np.uint8)
        return self.apply_packed(six, blob, off, ts_ms)

    def apply_packed(self, six, blob, off, ts_ms=None):
        n = len(six)
        st = np.zeros(n, dtype=np.int32)
        ts = None if ts_ms is None else np.ascontiguousarray(ts_ms, dtype=np.uint64)
        rc = self.lib.rsp_apply_many(self.h, n, _ptr(six), _ptr(blob), _ptr(off), _ptr(ts), _ptr(st))
        self.last_rc = rc  # (the call's own status: the first failing batch's, or an engine failure)
        return st

    def multi_get(self, shard_ix, keys, stride=256):
        """keys: list of bytes -> [(status, value|None)] with RocksDB MultiGet semantics."""
        n = len(keys)
        six = np.ascontiguousarray(shard_ix, dtype=np.uint32)
        off = np.zeros(n + 1, dtype=np.uint64)
        np.cumsum(np.fromiter((len(k) for k in keys), dtype=np.uint64, count=n), out=off[1:])
        blob = np.frombuffer(b"".join(keys) + b"\0", dtype=np.uint8)
        while True:
            vals = np.zeros(max(n * stride, 1), dtype=np.uint8)
            vlen = np.zeros(max(n, 1), dtype=np.uint32)
            st = np.zeros(max(n, 1), dtype=np.int32)
            rc = self.lib.rsp_multi_get(self.h, n, _ptr(six), _ptr(blob), _ptr(off), _ptr(vals), stride,
                                        _ptr(vlen), _ptr(st))
            if rc != OK:
                raise RuntimeError(f"rsp_multi_get -> {rc}")
            if n and (st[:n] == INCOMPLETE).any():
                stride = int(vlen[:n][st[:n] == INCOMPLETE].max())
                continue
            out = []
            for i in range(n):
                out.append((int(st[i]), vals[i * stride:i * stride + vlen[i]].tobytes() if st[i] == OK else None))
            return out

    def multi_get_at(self, snapshots, keys, stride=256):
        """lookup i at snapshots[i] (a Snapshot, or None: InvalidArgument) -> [(status, value|None)]"""
        n = len(keys)
        handles = (C.c_void_p * max(n, 1))(*[s.h if s is not None else None for s in snapshots])
        off = np.zeros(n + 1, dtype=np.uint64)
        np.cumsum(np.fromiter((len(k) for k in keys), dtype=np.uint64, count=n), out=off[1:])
        blob = np.frombuffer(b"".join(keys) + b"\0", dtype=np.uint8)
        while True:
            vals = np.zeros(max(n * stride, 1), dtype=np.uint8)
            vlen = np.zeros(max(n, 1), dtype=np.uint32)
            st = np.zeros(max(n, 1), dtype=np.int32)
            rc = self.lib.rsp_multi_get_at(self.h, n, handles, _ptr(blob), _ptr(off), _ptr(vals), stride,
                                           _ptr(vlen), _ptr(st))
            if rc != OK:
                raise RuntimeError(f"rsp_multi_get_at -> {rc}")
            if n and (st[:n] == INCOMPLETE).any():
                stride = int(vlen[:n][st[:n] == INCOMPLETE].max())
                continue
            return [(int(st[i]), vals[i * stride:i * stride + vlen[i]].tobytes() if st[i] == OK else None)
                    for i in range(n)]

    def multi_get_fixed(self, six, keys, klen, vals, stride, vlen, st):
        """numpy arrays in place (pinned or pageable host memory)."""
        return self.lib.rsp_multi_get_fixed(self.h, len(six), _ptr(six), _ptr(keys), klen, _ptr(vals), stride,
                                            _ptr(vlen), _ptr(st))

    def _scan(self, fn, n, first, keys, ends, max_entries, stride, exclusive=None, ends_are="end"):
        """one call of the host-form scan entry point `fn`: `first` is the shard indices or the snapshot handles, keys
        and ends are byte strings (None: none) -> [(status, [(key, value)])].  exclusive=None: `fn` takes no exclusive
        flag (rsp_multi_scan, rsp_multi_scan_bounded); rsp_multi_scan alone takes no end keys."""
        if keys is not None and len(keys) != n:
            raise ValueError("one start key per scan")
        if ends is not None and len(ends) != n:
            raise ValueError(f"one {ends_are} key per scan")
        blob, off = _pack_keys(keys) if keys is not None else (None, None)
        eblob, eoff = _pack_keys(ends) if ends is not None else (None, None)
        out = np.zeros(max(n * stride, 1), dtype=np.uint8)
        n_out = np.zeros(max(n, 1), dtype=np.uint32)
        st = np.zeros(max(n, 1), dtype=np.int32)
        args = [self.h, n, first, _ptr(blob), _ptr(off)]
        if exclusive is not None:
            args.append(1 if exclusive else 0)
        if fn != "rsp_multi_scan":
            args += [_ptr(eblob), _ptr(eoff)]
        rc = getattr(self.lib, fn)(*args, max_entries, _ptr(out), stride, _ptr(n_out), _ptr(st))
        if rc != OK:
            raise RuntimeError(f"{fn} -> {rc}")
        return _scan_records(out, n_out, st, n, stride)

    def multi_scan(self, shard_ix, keys, max_entries, stride, ends=None):
        """scan i: up to max_entries live entries from keys[i], before ends[i] (exclusive) when ends is given ->
        [(status, [(key, value)])]"""
        six = np.ascontiguousarray(shard_ix, dtype=np.uint32)
        fn = "rsp_multi_scan" if ends is None else "rsp_multi_scan_bounded"
        return self._scan(fn, len(keys), _ptr(six), keys, ends, max_entries, stride)

    def multi_scan_reverse(self, shard_ix, keys, max_entries, stride, lows=None, exclusive=False):
        """reverse scan i (SeekForPrev + Prev): up to max_entries live entries in descending key order from the last key
        <= keys[i] (< keys[i] when exclusive; keys=None: from the shard's last key), down to lows[i] (inclusive) when
        lows is given -> [(status, [(key, value)])].  [a, b) newest-first: keys=[b], lows=[a], exclusive=True."""
        six = np.ascontiguousarray(shard_ix, dtype=np.uint32)
        return self._scan("rsp_multi_scan_reverse", len(six), _ptr(six), keys, lows, max_entries, stride, exclusive,
                          ends_are="low")

    def multi_scan_at(self, snapshots, keys, max_entries, stride, ends=None, exclusive=False):
        """scan i at snapshots[i] (a Snapshot, or None: InvalidArgument): up to max_entries live entries from keys[i]
        (after it when exclusive; keys=None: from the snapshot's first key), before ends[i] (exclusive) when ends is
        given -> [(status, [(key, value)])].  Flushes nothing."""
        return self._scan("rsp_multi_scan_at", len(snapshots), _handles(snapshots), keys, ends, max_entries, stride,
                          exclusive)

    def multi_scan_reverse_at(self, snapshots, keys, max_entries, stride, lows=None, exclusive=False):
        """multi_scan_reverse at snapshots[i] (keys=None: from the snapshot's last key) -> [(status, [(key, value)])].
        Flushes nothing."""
        return self._scan("rsp_multi_scan_reverse_at", len(snapshots), _handles(snapshots), keys, lows, max_entries,
                          stride, exclusive)

    def flush_all(self): return self.lib.rsp_flush_all(self.h)
    def compact_all(self): return self.lib.rsp_compact_all(self.h)
    def last_kernel_ms(self, what): return self.lib.rsp_last_kernel_ms(self.h, what.encode())
    def kernel_launches(self): return self.lib.rsp_kernel_launches(self.h)

    def debug_last_pending(self, out=None):
        """lookups of the last multi_get_fixed / rsp_multi_get_device call (not the read combiner's) that the 16-byte-key
        kernel deferred to the generic path: returns their number and writes their positions (in no particular order)
        into `out`, a uint32 array, up to its length"""
        cap = 0 if out is None else len(out)
        return self.lib.rsp_debug_last_pending(self.h, _ptr(out) if cap else None, cap)


class Router:
    """Several engines (one per GPU) behind one handle: shard_id -> engine fan-out of cross-shard batches
    (examples/counter_service/counter_router.cpp:36-66 inside one box)."""

    def __init__(self, engines):
        self.lib = load_library()
        self.engines = list(engines)
        arr = (C.c_void_p * len(self.engines))(*[e.h for e in self.engines])
        h = C.c_void_p()
        rc = self.lib.rsp_router_create(len(self.engines), arr, C.byref(h))
        if rc != OK:
            raise RuntimeError(f"rsp_router_create -> {rc}")
        self.h = h

    def close(self):
        if self.h:
            self.lib.rsp_router_destroy(self.h)
            self.h = None

    def add_shard(self, shard_id, shard):
        rc = self.lib.rsp_router_add_shard(self.h, shard_id, shard.h)
        if rc != OK:
            raise RuntimeError(f"rsp_router_add_shard({shard_id}) -> {rc}")

    def apply_many(self, shard_ids, batches, ts_ms=None):
        n = len(batches)
        ids = np.ascontiguousarray(shard_ids, dtype=np.uint32)
        off = np.zeros(n + 1, dtype=np.uint64)
        np.cumsum(np.fromiter((len(b) for b in batches), dtype=np.uint64, count=n), out=off[1:])
        blob = np.frombuffer(b"".join(batches) + b"\0", dtype=np.uint8)
        st = np.zeros(max(n, 1), dtype=np.int32)
        ts = None if ts_ms is None else np.ascontiguousarray(ts_ms, dtype=np.uint64)
        self.lib.rsp_router_apply_many(self.h, n, _ptr(ids), _ptr(blob), _ptr(off), _ptr(ts), _ptr(st))
        return st[:n]

    def multi_get(self, shard_ids, keys, stride=256):
        n = len(keys)
        ids = np.ascontiguousarray(shard_ids, dtype=np.uint32)
        off = np.zeros(n + 1, dtype=np.uint64)
        np.cumsum(np.fromiter((len(k) for k in keys), dtype=np.uint64, count=n), out=off[1:])
        blob = np.frombuffer(b"".join(keys) + b"\0", dtype=np.uint8)
        while True:
            vals = np.zeros(max(n * stride, 1), dtype=np.uint8)
            vlen = np.zeros(max(n, 1), dtype=np.uint32)
            st = np.zeros(max(n, 1), dtype=np.int32)
            rc = self.lib.rsp_router_multi_get(self.h, n, _ptr(ids), _ptr(blob), _ptr(off), _ptr(vals), stride, _ptr(vlen), _ptr(st))
            if n and (st[:n] == INCOMPLETE).any():
                stride = int(vlen[:n][st[:n] == INCOMPLETE].max())
                continue
            return [(int(st[i]), vals[i * stride:i * stride + vlen[i]].tobytes() if st[i] == OK else None) for i in range(n)], rc

    def multi_get_fixed(self, shard_ids, keys, klen, vals, stride, vlen, st):
        return self.lib.rsp_router_multi_get_fixed(self.h, len(shard_ids), _ptr(shard_ids), _ptr(keys), klen, _ptr(vals), stride,
                                                   _ptr(vlen), _ptr(st))
