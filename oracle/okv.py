"""ctypes binding for the oracle interface in oracle/okv.h (TEST INFRASTRUCTURE ONLY).

Two libraries export the same symbols:
  libokv_port.so      — CPU restatement (oracle/kv_oracle.c)
  _ref/libokv_ref.so  — driver over the reference's own RocksDB binary (oracle/ref_driver.c)
"""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
PORT_SO = os.path.join(HERE, "libokv_port.so")
REF_SO = os.path.join(HERE, "_ref", "libokv_ref.so")

OK, NOT_FOUND, CORRUPTION, NOT_SUPPORTED, INVALID_ARGUMENT, IO_ERROR = 0, 1, 2, 3, 4, 5
MERGE_NONE, MERGE_COUNTER, MERGE_UINT64ADD, MERGE_APPEND = 0, 1, 2, 3


def build(ref=True):
    """Compile the checkers (gcc).  `ref` also (re)builds oracle/_ref when the reference's source tree is present."""
    subprocess.check_call(["make", "-s", "-C", HERE, "port", "bench"] + (["ref"] if ref else []),
                          stdout=subprocess.DEVNULL)


def _bind(path):
    lib = C.CDLL(path)
    vp, cp, sz, u64, i32 = C.c_void_p, C.c_char_p, C.c_size_t, C.c_uint64, C.c_int
    sig = {
        "okv_kind": (cp, []),
        "okv_open": (vp, [cp, i32, i32, cp, sz]),
        "okv_close": (None, [vp]),
        "okv_apply": (i32, [vp, cp, sz, u64, cp, sz]),
        "okv_latest_seq": (u64, [vp]),
        "okv_get": (i32, [vp, cp, sz, C.POINTER(vp), C.POINTER(sz), cp, sz]),
        "okv_multi_get": (i32, [vp, sz, cp, C.POINTER(u64), C.POINTER(C.c_int32), C.POINTER(vp),
                                C.POINTER(u64)]),
        "okv_iter_create": (vp, [vp]),
        "okv_iter_destroy": (None, [vp]),
        "okv_iter_seek_to_first": (None, [vp]),
        "okv_iter_seek_to_last": (None, [vp]),
        "okv_iter_seek": (None, [vp, cp, sz]),
        "okv_iter_next": (None, [vp]),
        "okv_iter_prev": (None, [vp]),
        "okv_iter_valid": (i32, [vp]),
        "okv_iter_key": (vp, [vp, C.POINTER(sz)]),
        "okv_iter_value": (vp, [vp, C.POINTER(sz)]),
        "okv_iter_status": (i32, [vp]),
        "okv_flush": (i32, [vp]),
        "okv_compact": (i32, [vp]),
        "okv_free": (None, [vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


_libs = {}


def load_port():
    if "port" not in _libs:
        if not os.path.exists(PORT_SO):
            build(ref=False)
        _libs["port"] = _bind(PORT_SO)
    return _libs["port"]


def ref_available():
    return os.path.exists(REF_SO) and os.path.exists(os.path.join(HERE, "_ref", "librocksdb.so.5.4"))


def load_ref():
    if "ref" not in _libs:
        _libs["ref"] = _bind(REF_SO)
    return _libs["ref"]


class OkvIter:
    def __init__(self, lib, db):
        self.lib = lib
        self.h = lib.okv_iter_create(db.h)
        self._db = db

    def close(self):
        if self.h:
            self.lib.okv_iter_destroy(self.h)
            self.h = None

    def seek_to_first(self): self.lib.okv_iter_seek_to_first(self.h)
    def seek_to_last(self): self.lib.okv_iter_seek_to_last(self.h)
    def seek(self, k): self.lib.okv_iter_seek(self.h, k, len(k))
    def next(self): self.lib.okv_iter_next(self.h)
    def prev(self): self.lib.okv_iter_prev(self.h)
    def valid(self): return bool(self.lib.okv_iter_valid(self.h))
    def status(self): return self.lib.okv_iter_status(self.h)

    def key(self):
        n = C.c_size_t()
        p = self.lib.okv_iter_key(self.h, C.byref(n))
        return C.string_at(p, n.value) if n.value else b""

    def value(self):
        n = C.c_size_t()
        p = self.lib.okv_iter_value(self.h, C.byref(n))
        return C.string_at(p, n.value) if n.value else b""


class Okv:
    """One shard (one DB) of the oracle."""

    def __init__(self, lib=None, merge_op=MERGE_NONE, wal=True, path=None):
        self.lib = lib or load_port()
        self.kind = self.lib.okv_kind().decode()
        self._tmp = None
        if path is None:
            base = "/dev/shm" if os.path.isdir("/dev/shm") else None
            self._tmp = tempfile.mkdtemp(prefix="okv_", dir=base)
            path = os.path.join(self._tmp, "db")
        err = C.create_string_buffer(512)
        self.h = self.lib.okv_open(path.encode(), merge_op, 1 if wal else 0, err, 512)
        if not self.h:
            raise RuntimeError("okv_open failed: " + err.value.decode())
        self.last_error = ""

    def close(self):
        if self.h:
            self.lib.okv_close(self.h)
            self.h = None
        if self._tmp:
            shutil.rmtree(self._tmp, ignore_errors=True)
            self._tmp = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def apply(self, batch: bytes, ts_ms: int = 0) -> int:
        err = C.create_string_buffer(256)
        rc = self.lib.okv_apply(self.h, batch, len(batch), ts_ms, err, 256)
        self.last_error = err.value.decode()
        return rc

    def latest_seq(self) -> int:
        return self.lib.okv_latest_seq(self.h)

    def get(self, key: bytes):
        """-> (status, value or None)"""
        v = C.c_void_p()
        n = C.c_size_t()
        err = C.create_string_buffer(256)
        rc = self.lib.okv_get(self.h, key, len(key), C.byref(v), C.byref(n), err, 256)
        self.last_error = err.value.decode()
        if rc != OK:
            return rc, None
        out = C.string_at(v.value, n.value) if n.value else b""
        self.lib.okv_free(v)
        return rc, out

    def multi_get(self, keys):
        n = len(keys)
        blob = b"".join(keys)
        koff = (C.c_uint64 * (n + 1))()
        at = 0
        for i, k in enumerate(keys):
            koff[i] = at
            at += len(k)
        koff[n] = at
        st = (C.c_int32 * max(n, 1))()
        voff = (C.c_uint64 * (n + 1))()
        vals = C.c_void_p()
        self.lib.okv_multi_get(self.h, n, blob, koff, st, C.byref(vals), voff)
        raw = C.string_at(vals.value, voff[n]) if voff[n] else b""
        self.lib.okv_free(vals)
        out = []
        for i in range(n):
            out.append((st[i], raw[voff[i]:voff[i + 1]] if st[i] == OK else None))
        return out

    def iterator(self):
        return OkvIter(self.lib, self)

    def scan(self, start=None, limit=None):
        it = self.iterator()
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

    def flush(self): return self.lib.okv_flush(self.h)
    def compact(self): return self.lib.okv_compact(self.h)
