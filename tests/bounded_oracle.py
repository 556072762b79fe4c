"""Bounded iterators on the oracle (TEST INFRASTRUCTURE ONLY): ReadOptions::iterate_upper_bound and
Iterator::SeekForPrev on the port and on the reference's own RocksDB binary, and the edge cases recorded from the binary
into tests/golden/bounded_scans.json.

The C side is tests/oracle_bounded/bounded_{port,ref}.c: each compiles tests/oracle_snapshots/snapshot_{port,ref}.c (the
oracle with snapshot reads) as it is and adds okv_iter_create_bounded / okv_iter_destroy_bounded, the bounded forward
moves okv_biter_* and okv_iter_seek_for_prev.  The port's library is built under tests/oracle_bounded/build/; the
binary's next to the binary in oracle/_ref/ (only where the reference could be built).

    python tests/bounded_oracle.py --generate    # tests/golden/bounded_scans.json from the binary
"""
import ctypes as C
import json
import os
import struct
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import snapshot_oracle as SO  # noqa: E402
from oracle import okv  # noqa: E402
from rocksplicator_b200.write_batch import WriteBatch  # noqa: E402

SRC = os.path.join(HERE, "oracle_bounded")
PORT_SO = os.path.join(SRC, "build", "libokv_bounded_port.so")
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libokv_bounded_ref.so")
GOLDEN = os.path.join(HERE, "golden", "bounded_scans.json")


def _bind(path, ref):
    lib = SO._bind(path)
    vp, cp, sz = C.c_void_p, C.c_char_p, C.c_size_t
    sig = {
        "okv_iter_create_bounded": (vp, [vp, vp, cp, sz]),
        "okv_iter_destroy_bounded": (None, [vp]),
        "okv_biter_seek_to_first": (None, [vp]),
        "okv_biter_seek_to_last": (None, [vp]),
        "okv_biter_seek": (None, [vp, cp, sz]),
        "okv_biter_next": (None, [vp]),
        "okv_iter_seek_for_prev": (None, [vp, cp, sz]),
    }
    if ref:
        sig["okv_ingest_sst_consistency"] = (C.c_int, [vp, cp, C.c_int, C.c_int, cp, sz])
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


_libs = {}


def load_port():
    if "port" not in _libs:
        deps = [os.path.join(ROOT, "oracle", f) for f in ("kv_oracle.c", "okv.h")] + \
               [os.path.join(HERE, "oracle_snapshots", "snapshot_port.c")]
        SO._compile(os.path.join(SRC, "bounded_port.c"), deps, PORT_SO)
        _libs["port"] = _bind(PORT_SO, False)
    return _libs["port"]


def load_ref():
    if "ref" not in _libs:
        if not okv.ref_available():
            raise RuntimeError("oracle/_ref not built: run `make -C oracle ref` with the reference's source tree at REF")
        deps = [os.path.join(ROOT, "oracle", f) for f in ("ref_driver.c", "okv.h")] + \
               [os.path.join(HERE, "oracle_snapshots", "snapshot_ref.c")]
        SO._compile(os.path.join(SRC, "bounded_ref.c"), deps, REF_SO)
        _libs["ref"] = _bind(REF_SO, True)
    return _libs["ref"]


class BIter(okv.OkvIter):
    """an oracle iterator with an optional upper bound (None: unbounded) at an optional snapshot"""

    def __init__(self, lib, db, upper_bound=None, snapshot=None):  # noqa: super().__init__ would open an unbounded one
        self.lib = lib
        self._db = db
        self.h = lib.okv_iter_create_bounded(db.h, snapshot.h if snapshot is not None else None, upper_bound,
                                             0 if upper_bound is None else len(upper_bound))

    def close(self):
        if self.h:
            self.lib.okv_iter_destroy_bounded(self.h)
            self.h = None

    def seek_to_first(self): self.lib.okv_biter_seek_to_first(self.h)
    def seek_to_last(self): self.lib.okv_biter_seek_to_last(self.h)
    def seek(self, k): self.lib.okv_biter_seek(self.h, k, len(k))
    def next(self): self.lib.okv_biter_next(self.h)
    def seek_for_prev(self, k): self.lib.okv_iter_seek_for_prev(self.h, k, len(k))


class BoundedOkv(SO.SnapOkv):
    """SnapOkv whose iterators take an upper bound; lib = load_port() or load_ref()"""

    def __init__(self, lib=None, merge_op=okv.MERGE_NONE, wal=True, path=None):
        super().__init__(lib or load_port(), merge_op=merge_op, wal=wal, path=path)

    def iterator(self, snapshot=None, upper_bound=None):
        return BIter(self.lib, self, upper_bound, snapshot)

    def scan(self, start=None, limit=None, snapshot=None, end=None):
        it = self.iterator(snapshot, end)
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


# ---- the recorded edge cases ------------------------------------------------------------------------------------------
def _op(n):
    return struct.pack("<q", n)


# Three write phases.  k30 ends deleted, k40 and k85 hold merge operands only, k60 gets an operand on a 3-byte Put (a
# counter merge that fails; uint64add counts it as 0; append appends), k70 and k90 end deleted.  The last phase always
# stays in the memtable, so that no flush or compaction merges k60 (RocksDB fails the flush that would).
PHASES = [
    [("put", b"k10", b"v10"), ("put", b"k20", b"v20"), ("put", b"k30", b"v30"), ("merge", b"k40", _op(1)),
     ("put", b"k50", b"v50"), ("put", b"k60", b"abc"), ("put", b"k70", b"v70"), ("put", b"k90", b"v90")],
    [("del", b"k30"), ("merge", b"k40", _op(2)), ("put", b"k20", b"v20b"), ("put", b"k80", b"v80")],
    [("merge", b"k60", _op(5)), ("del", b"k70"), ("put", b"k75", b"v75"), ("merge", b"k85", _op(3)), ("del", b"k90")],
]
# where the flushes and compactions fall between the phases ("S": a snapshot, read at the end besides the latest state)
LAYOUTS = {
    "mem": ["A", "B", "C"],
    "run+mem": ["A", "B", "flush", "C"],
    "runs+mem": ["A", "flush", "B", "flush", "S", "C"],
    "compacted+mem": ["A", "flush", "B", "flush", "compact", "C"],
}
MERGES = {"counter": okv.MERGE_COUNTER, "uint64add": okv.MERGE_UINT64ADD, "append": okv.MERGE_APPEND}
# a deleted key, a merge-only key, a live key, between keys, a proper prefix of k60, longer than k60, the failing merge
# key itself, below and above every key, the empty bound, none
BOUNDS = [b"k30", b"k40", b"k50", b"k55", b"k6", b"k600", b"k60", b"a", b"z", b"", None]
MOVES = [
    [("first",)] + [("next",)] * 9,
    [("seek", b"k00"), ("next",), ("next",)],
    [("seek", b"k40"), ("next",), ("next",)],
    [("seek", b"k50"), ("next",)],
    [("seek", b"k55"), ("next",)],
    [("seek", b"k6"), ("next",)],
    [("seek", b"k95")],
    [("last",)] + [("prev",)] * 9,
    [("sfp", b"k10"), ("prev",), ("next",)],
    [("sfp", b"k40"), ("prev",), ("next",), ("next",)],
    [("sfp", b"k50"), ("next",), ("prev",)],
    [("sfp", b"k55"), ("prev",), ("next",), ("next",)],
    [("sfp", b"k65"), ("prev",), ("next",)],
    [("sfp", b"k95"), ("prev",), ("prev",), ("next",)],
    [("sfp", b"a")],
    [("last",), ("next",), ("prev",)],
    [("last",), ("prev",), ("next",), ("next",), ("prev",)],
    [("seek", b"k10"), ("next",), ("prev",), ("next",), ("next",), ("next",)],
]


def _state(it):
    return [it.key().hex(), it.value().hex(), it.status()] if it.valid() else [None, None, it.status()]


def run_moves(make_iter):
    """every move list on a fresh iterator -> the iterator's state after each move, up to the first move that leaves
    it invalid (Next and Prev require a valid iterator)"""
    out = []
    for moves in MOVES:
        it = make_iter()
        got = []
        for m in moves:
            if got and got[-1][0] is None:
                break
            if m[0] == "first":
                it.seek_to_first()
            elif m[0] == "last":
                it.seek_to_last()
            elif m[0] == "seek":
                it.seek(m[1])
            elif m[0] == "sfp":
                it.seek_for_prev(m[1])
            elif m[0] == "next":
                it.next()
            else:
                it.prev()
            got.append(_state(it))
        it.close()
        out.append(got)
    return out


def run_case(side, layout):
    """side: apply(batch) -> rc, flush(), compact(), snapshot(), release(snap), iterator(upper_bound, snapshot)"""
    snap = None
    for step in LAYOUTS[layout]:
        if step in ("A", "B", "C"):
            for op in PHASES["ABC".index(step)]:
                wb = WriteBatch()
                if op[0] == "put":
                    wb.put(op[1], op[2])
                elif op[0] == "merge":
                    wb.merge(op[1], op[2])
                else:
                    wb.delete(op[1])
                assert side.apply(wb.data()) == 0, (layout, op)
        elif step == "flush":
            assert side.flush() == 0
        elif step == "compact":
            assert side.compact() == 0
        else:
            snap = side.snapshot()
    res = {}
    for b in BOUNDS:
        tag = "none" if b is None else b.hex()
        res[tag] = run_moves(lambda: side.iterator(b, None))
        if snap is not None:
            res["snap-" + tag] = run_moves(lambda: side.iterator(b, snap))
    if snap is not None:
        side.release(snap)
    return res


def case_names():
    return ["%s-%s" % (m, lay) for m in MERGES for lay in LAYOUTS]


class OkvSide:
    def __init__(self, db):
        self.db = db

    def apply(self, batch): return self.db.apply(batch, 0)
    def flush(self): return self.db.flush()
    def compact(self): return self.db.compact()
    def snapshot(self): return self.db.snapshot()
    def release(self, s): s.release()
    def iterator(self, upper_bound, snapshot): return self.db.iterator(snapshot, upper_bound)


def run_on_oracle(lib, name):
    merge, layout = name.split("-", 1)
    db = BoundedOkv(lib, merge_op=MERGES[merge])
    try:
        return run_case(OkvSide(db), layout)
    finally:
        db.close()


def generate():
    ref = load_ref()
    out = {name: run_on_oracle(ref, name) for name in case_names()}
    with open(GOLDEN, "w") as f:
        json.dump({"generator": "tests/bounded_oracle.py --generate", "source": "rocksdb_admin/tests/librocksdb.so.5.4",
                   "cases": out}, f, separators=(",", ":"), sort_keys=True)
        f.write("\n")
    print("bounded_scans.json", os.path.getsize(GOLDEN), "bytes")


if __name__ == "__main__":
    if "--generate" in sys.argv:
        generate()
    else:
        print(__doc__)
