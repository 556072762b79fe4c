"""Snapshot reads on the oracle (TEST INFRASTRUCTURE ONLY): DB::GetSnapshot / ReleaseSnapshot and Get, MultiGet and
iterators with ReadOptions::snapshot, on the port and on the reference's own RocksDB binary.

The C side is tests/oracle_snapshots/snapshot_{port,ref}.c: each compiles the oracle's own source (oracle/kv_oracle.c,
oracle/ref_driver.c) as it is and adds the okv_snapshot_* / okv_*_at calls, so the library exports oracle/okv.h plus
these.  The port's library is built under tests/oracle_snapshots/build/; the binary's next to the binary in
oracle/_ref/ (only where the reference could be built).

    python tests/snapshot_oracle.py --generate    # tests/golden/snapshots.json from the binary
"""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import okv  # noqa: E402

SRC = os.path.join(HERE, "oracle_snapshots")
PORT_SO = os.path.join(SRC, "build", "libokv_snap_port.so")
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libokv_snap_ref.so")
GOLDEN = os.path.join(HERE, "golden", "snapshots.json")


def _compile(src, deps, out):
    if os.path.exists(out) and all(os.path.getmtime(d) <= os.path.getmtime(out) for d in [src] + deps):
        return
    os.makedirs(os.path.dirname(out), exist_ok=True)
    fd, tmp = tempfile.mkstemp(suffix=".so", dir=os.path.dirname(out))
    os.close(fd)
    subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-w", "-fPIC", "-shared", "-o", tmp, src, "-ldl", "-lpthread"])
    os.replace(tmp, out)  # (concurrent test processes may build it at the same time)


def _bind(path):
    lib = okv._bind(path)
    vp, cp, sz, u64, i32 = C.c_void_p, C.c_char_p, C.c_size_t, C.c_uint64, C.c_int
    sig = {
        "okv_snapshot_create": (vp, [vp]),
        "okv_snapshot_release": (None, [vp, vp]),
        "okv_snapshot_seq": (u64, [vp]),
        "okv_get_at": (i32, [vp, vp, cp, sz, C.POINTER(vp), C.POINTER(sz), cp, sz]),
        "okv_multi_get_at": (i32, [vp, vp, sz, cp, C.POINTER(u64), C.POINTER(C.c_int32), C.POINTER(vp), C.POINTER(u64)]),
        "okv_iter_create_at": (vp, [vp, vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


_libs = {}


def load_port():
    if "port" not in _libs:
        deps = [os.path.join(ROOT, "oracle", f) for f in ("kv_oracle.c", "okv.h")]
        _compile(os.path.join(SRC, "snapshot_port.c"), deps, PORT_SO)
        _libs["port"] = _bind(PORT_SO)
    return _libs["port"]


def load_ref():
    if "ref" not in _libs:
        if not okv.ref_available():
            raise RuntimeError("oracle/_ref not built: run `make -C oracle ref` with the reference's source tree at REF")
        deps = [os.path.join(ROOT, "oracle", f) for f in ("ref_driver.c", "okv.h")]
        _compile(os.path.join(SRC, "snapshot_ref.c"), deps, REF_SO)
        lib = _bind(REF_SO)
        lib.okv_ingest_sst_consistency.restype = C.c_int
        lib.okv_ingest_sst_consistency.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.c_char_p, C.c_size_t]
        _libs["ref"] = lib
    return _libs["ref"]


class OkvSnapshot:
    """DB::GetSnapshot on one oracle DB (release it before the DB is closed)"""

    def __init__(self, db):
        self.db = db
        self.h = db.lib.okv_snapshot_create(db.h)
        self.seq = db.lib.okv_snapshot_seq(self.h)

    def release(self):
        if self.h:
            self.db.lib.okv_snapshot_release(self.db.h, self.h)
            self.h = None


class _IterAt(okv.OkvIter):
    def __init__(self, lib, db, snapshot):  # noqa: super().__init__ would open an iterator at the latest state
        self.lib = lib
        self.h = lib.okv_iter_create_at(db.h, snapshot.h)
        self._db = db


class SnapOkv(okv.Okv):
    """okv.Okv whose reads take an optional snapshot (None = the latest state); lib = load_port() or load_ref()"""

    def __init__(self, lib=None, merge_op=okv.MERGE_NONE, wal=True, path=None):
        super().__init__(lib or load_port(), merge_op=merge_op, wal=wal, path=path)

    def snapshot(self):
        return OkvSnapshot(self)

    def get(self, key: bytes, snapshot=None):
        if snapshot is None:
            return super().get(key)
        v, n, err = C.c_void_p(), C.c_size_t(), C.create_string_buffer(256)
        rc = self.lib.okv_get_at(self.h, snapshot.h, key, len(key), C.byref(v), C.byref(n), err, 256)
        self.last_error = err.value.decode()
        if rc != okv.OK:
            return rc, None
        out = C.string_at(v.value, n.value) if n.value else b""
        self.lib.okv_free(v)
        return rc, out

    def multi_get(self, keys, snapshot=None):
        if snapshot is None:
            return super().multi_get(keys)
        n = len(keys)
        koff = (C.c_uint64 * (n + 1))()
        for i, k in enumerate(keys):
            koff[i + 1] = koff[i] + len(k)
        st = (C.c_int32 * max(n, 1))()
        voff = (C.c_uint64 * (n + 1))()
        vals = C.c_void_p()
        self.lib.okv_multi_get_at(self.h, snapshot.h, n, b"".join(keys), koff, st, C.byref(vals), voff)
        raw = C.string_at(vals.value, voff[n]) if voff[n] else b""
        self.lib.okv_free(vals)
        return [(st[i], raw[voff[i]:voff[i + 1]] if st[i] == okv.OK else None) for i in range(n)]

    def iterator(self, snapshot=None):
        return super().iterator() if snapshot is None else _IterAt(self.lib, self, snapshot)

    def scan(self, start=None, limit=None, snapshot=None):
        it = self.iterator(snapshot)
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


def generate():
    """tests/golden/snapshots.json: tests/snapshot_streams.py's scenarios on the binary (snapshot sequence numbers,
    fingerprints of every read at every live snapshot and at the latest state; ingestion with live snapshots)"""
    import golden_util as G
    import snapshot_streams as S
    from rocksplicator_b200 import sst
    ref = load_ref()
    out = {"streams": {}, "ingest": []}
    for merge, seed in S.STREAM_CASES:
        db = SnapOkv(ref, merge_op=S.MERGES[merge])
        out["streams"]["%s-%d" % (merge, seed)] = S.run_stream(S.OkvSide(db), merge, seed, G.digest)
        db.close()
    tmp = tempfile.mkdtemp()
    for name, rows, allow, with_snapshot in S.ingest_steps():
        db = SnapOkv(ref)

        def ingest(rows, allow):
            path = os.path.join(tmp, name + ".sst")
            open(path, "wb").write(sst.write_sst(rows))
            err = C.create_string_buffer(256)
            rc = ref.okv_ingest_sst_consistency(db.h, path.encode(), 1 if allow else 0, 1, err, 256)
            return rc, err.value.decode()
        out["ingest"].append(S.run_ingest(S.OkvSide(db), name, rows, allow, with_snapshot, ingest, G.digest))
        db.close()
    with open(GOLDEN, "w") as f:
        json.dump({"generator": "tests/snapshot_oracle.py --generate", "source": "rocksdb_admin/tests/librocksdb.so.5.4",
                   "cases": out}, f, separators=(",", ":"))
    print("snapshots.json", os.path.getsize(GOLDEN), "bytes")


if __name__ == "__main__":
    if "--generate" in sys.argv:
        generate()
    else:
        print(__doc__)
