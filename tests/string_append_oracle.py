"""RocksDB's StringAppendOperator on the reference's own RocksDB binary (TEST INFRASTRUCTURE ONLY), the recorded cases
of tests/golden/string_append.json, and one replay of those cases for every side that answers them: the binary
(tests/oracle_string_append/sa_ref.c), the port (tests/string_append_model.py) and the engine.

A case is a stream of WriteBatches with flushes, full compactions and snapshots at fixed points; at fixed checkpoints
every key is read with Get and MultiGet, the whole key range is iterated forward and backward, and Seek / SeekForPrev
land on a few keys, at the latest state and at every snapshot taken so far.  The streams cover delimiters ',', none and
'\\0', Put / Merge / Delete / SingleDelete, empty operands and empty bases, and flushes of several operands without a
base (RocksDB folds those with PartialMerge).

    python tests/string_append_oracle.py --generate    # tests/golden/string_append.json from the binary
"""
import ctypes as C
import json
import os
import random
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import bounded_oracle as BO  # noqa: E402
import snapshot_oracle as SO  # noqa: E402
import string_append_model as SA  # noqa: E402
from oracle import okv  # noqa: E402

SRC = os.path.join(HERE, "oracle_string_append")
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libokv_sa_ref.so")
GOLDEN = os.path.join(HERE, "golden", "string_append.json")
DELIMS = {"comma": b",", "none": None, "nul": b"\0"}
_libs = {}


def delim_word(delim):
    """rsp_shard_opts.merge_delim / okv_open_string_append's delimiter: 0 = none, 0x100 | c"""
    return 0 if delim is None else 0x100 | delim[0]


def ref_available():
    return okv.ref_available()


def load_ref():
    if "ref" not in _libs:
        if not okv.ref_available():
            raise RuntimeError("oracle/_ref not built: run `make -C oracle ref` with the reference's source tree at REF")
        deps = [os.path.join(ROOT, "oracle", f) for f in ("ref_driver.c", "okv.h")] + \
               [os.path.join(HERE, "oracle_snapshots", "snapshot_ref.c"), os.path.join(HERE, "oracle_bounded", "bounded_ref.c")]
        SO._compile(os.path.join(SRC, "sa_ref.c"), deps, REF_SO)
        lib = BO._bind(REF_SO, True)
        lib.okv_open_string_append.restype = C.c_void_p
        lib.okv_open_string_append.argtypes = [C.c_char_p, C.c_uint32, C.c_int, C.c_char_p, C.c_size_t]
        _libs["ref"] = lib
    return _libs["ref"]


class RefDB(BO.BoundedOkv):
    """the binary with a StringAppendOperator of the given delimiter (one byte or None)"""

    def __init__(self, delim):  # noqa: super().__init__ would open the DB with another operator
        self.lib = load_ref()
        self.kind = "ref"
        base = "/dev/shm" if os.path.isdir("/dev/shm") else None
        self._tmp = tempfile.mkdtemp(prefix="okv_sa_", dir=base)
        err = C.create_string_buffer(512)
        self.h = self.lib.okv_open_string_append(os.path.join(self._tmp, "db").encode(), delim_word(delim), 1, err, 512)
        if not self.h:
            raise RuntimeError("okv_open_string_append failed: " + err.value.decode())
        self.last_error = ""


# ---- sides: write(ops), flush(), compact(), snapshot() -> handle, get(key, snap), multi_get(keys, snap),
# iterator(snap) -----------------------------------------------------------------------------------------------------
class RefSide:
    def __init__(self, delim):
        self.db = RefDB(delim)
        self.snaps = []

    def write(self, ops): assert self.db.apply(SA.batch_of(ops), 0) == 0
    def flush(self): assert self.db.flush() == 0
    def compact(self): assert self.db.compact() == 0

    def snapshot(self):
        s = self.db.snapshot()
        self.snaps.append(s)
        return s

    def get(self, k, snap):
        rc, v = self.db.get(k, snapshot=snap)
        return v if rc == 0 else None

    def multi_get(self, keys, snap):
        if snap is None:
            return [v if rc == 0 else None for rc, v in self.db.multi_get(keys)]
        return [self.get(k, snap) for k in keys]

    def iterator(self, snap): return self.db.iterator(snap)

    def close(self):
        for s in self.snaps:
            s.release()
        self.db.close()


class ModelIter:
    def __init__(self, items):
        self.items, self.pos = items, -1

    def seek_to_first(self): self.pos = 0 if self.items else -1
    def seek_to_last(self): self.pos = len(self.items) - 1

    def seek(self, k):
        self.pos = next((i for i, (x, _) in enumerate(self.items) if x >= k), -1)

    def seek_for_prev(self, k):
        self.pos = max((i for i, (x, _) in enumerate(self.items) if x <= k), default=-1)

    def next(self): self.pos = self.pos + 1 if 0 <= self.pos < len(self.items) - 1 else -1
    def prev(self): self.pos = self.pos - 1 if self.pos > 0 else -1
    def valid(self): return self.pos >= 0
    def key(self): return self.items[self.pos][0]
    def value(self): return self.items[self.pos][1]
    def status(self): return 0
    def close(self): pass


class ModelSide:
    """the port: tests/string_append_model.py"""

    def __init__(self, delim):
        self.m = SA.Model(delim)

    def write(self, ops): self.m.apply(ops)
    def flush(self): pass
    def compact(self): pass
    def snapshot(self): return self.m.seq
    def get(self, k, snap): return self.m.get(k, snap)
    def multi_get(self, keys, snap): return [self.m.get(k, snap) for k in keys]
    def iterator(self, snap): return ModelIter(self.m.items(snap))
    def close(self): pass


class EngineSide:
    """a shard of a rocksplicator_b200 engine (the caller owns the engine)"""

    def __init__(self, eng, name, delim):
        from rocksplicator_b200 import engine
        self.s = eng.open_shard(name, merge_op=engine.MERGE_STRING_APPEND, merge_delim=delim)
        self.snaps = []

    def write(self, ops): assert self.s.apply(SA.batch_of(ops), 0) == 0
    def flush(self): assert self.s.flush() == 0
    def compact(self): assert self.s.compact() == 0

    def snapshot(self):
        s = self.s.snapshot()
        self.snaps.append(s)
        return s

    def get(self, k, snap):
        rc, v = (snap or self.s).get(k, cap=8)
        return v if rc == 0 else None

    def multi_get(self, keys, snap):
        return [v if rc == 0 else None for rc, v in (snap or self.s).multi_get(keys, stride=8)]

    def iterator(self, snap): return (snap or self.s).iterator()

    def close(self):
        for s in self.snaps:
            s.release()
        self.s.close()


# ---- the cases -------------------------------------------------------------------------------------------------------
def _key(i):
    return b"k%02d" % i


def _stream(seed):
    """a seeded stream: [("write", ops) | ("flush",) | ("compact",) | ("snapshot",) | ("read",)].  Keys k00 .. k11.
    SingleDelete only on keys whose whole history is nothing or one Put: RocksDB leaves every other use undefined (a
    SingleDelete that meets a Delete in a compaction, for one, drops it and uncovers the older versions)."""
    rng = random.Random(seed)
    steps, hist = [], {}
    for r in range(14):
        ops = []
        for _ in range(rng.randrange(2, 9)):
            k = _key(rng.randrange(12))
            x = rng.random()
            h = hist.setdefault(k, [])
            if x < 0.55:
                ops.append((SA.MERGE, k, b"" if rng.random() < 0.15 else bytes(rng.choice(b"abcxyz,\0") for _ in range(rng.randrange(1, 4)))))
            elif x < 0.75:
                ops.append((SA.PUT, k, b"" if rng.random() < 0.3 else b"P%d" % r))
            elif x < 0.9 or h not in ([], [SA.PUT]):
                ops.append((SA.DEL, k, b""))
            else:
                ops.append((SA.SDEL, k, b""))
            h.append(ops[-1][0])
        steps.append(("write", ops))
        if r in (2, 5, 9, 12):
            steps.append(("flush",))
        if r == 10:
            steps.append(("compact",))
        if r in (3, 8):
            steps.append(("snapshot",))
        if r in (4, 7, 11, 13):
            steps.append(("read",))
    steps.append(("compact",))
    steps.append(("read",))
    return steps


def _fixed_stream():
    """the edge cases by hand: empty base against no base, Delete / SingleDelete under operands, operand-only flushes"""
    M, P, D, S = SA.MERGE, SA.PUT, SA.DEL, SA.SDEL
    return [
        ("write", [(P, b"a", b""), (M, b"a", b"x"), (M, b"b", b"x"), (M, b"b", b""), (M, b"b", b"")]),
        ("write", [(P, b"c", b"base"), (D, b"c", b""), (M, b"c", b"1"), (M, b"c", b"2")]),
        ("write", [(P, b"d", b"v"), (S, b"d", b""), (M, b"d", b"y")]),
        ("read",),
        ("flush",),
        ("snapshot",),
        ("write", [(M, b"e", b"1"), (M, b"e", b"2"), (M, b"e", b"3"), (M, b"a", b""), (M, b"c", b"3")]),
        ("flush",),  # operands without a base: RocksDB's flush folds them with PartialMerge
        ("write", [(M, b"e", b"4"), (M, b"f", b"only")]),
        ("flush",),
        ("read",),
        ("write", [(P, b"e", b""), (M, b"e", b"5"), (D, b"f", b"")]),
        ("compact",),
        ("read",),
    ]


def cases():
    out = {}
    for dn, delim in DELIMS.items():
        out["fixed_" + dn] = (delim, _fixed_stream())
        for seed in range(2):
            out["random%d_%s" % (seed, dn)] = (delim, _stream(1000 * seed + len(dn)))
    return out


def _hex(v):
    return None if v is None else v.hex()


def _walk(it, fwd, n=None):
    out = []
    while it.valid() and (n is None or len(out) < n):
        out.append([it.key().hex(), it.value().hex()])
        it.next() if fwd else it.prev()
    return out


def run_case(side, steps):
    """replay on a side -> the list of what each read checkpoint answered (JSON-able)"""
    snaps, reads, keys = [], [], set()
    for st in steps:
        if st[0] == "write":
            side.write(st[1])
            keys.update(k for _, k, _ in st[1])
        elif st[0] == "flush":
            side.flush()
        elif st[0] == "compact":
            side.compact()
        elif st[0] == "snapshot":
            snaps.append(side.snapshot())
        else:
            ks = sorted(keys) + [b"zz"]
            cp = []
            for snap in [None] + snaps:
                r = {"get": [_hex(side.get(k, snap)) for k in ks], "multi_get": [_hex(v) for v in side.multi_get(ks, snap)]}
                it = side.iterator(snap)
                it.seek_to_first()
                r["forward"] = _walk(it, True)
                it.seek_to_last()
                r["backward"] = _walk(it, False)
                r["seek"], r["seek_for_prev"] = [], []
                for t in (ks[0], ks[len(ks) // 2] + b"0", b"z"):
                    it.seek(t)
                    r["seek"].append(_walk(it, True, 3))
                    it.seek_for_prev(t)
                    r["seek_for_prev"].append(_walk(it, False, 3))
                assert it.status() == 0
                it.close()
                cp.append(r)
            reads.append(cp)
    return reads


def load_cases():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


def generate():
    out = {}
    for name, (delim, steps) in cases().items():
        side = RefSide(delim)
        try:
            out[name] = run_case(side, steps)
        finally:
            side.close()
            shutil.rmtree(side.db._tmp, ignore_errors=True)
    with open(GOLDEN, "w") as f:
        json.dump({"generator": "tests/string_append_oracle.py --generate", "source": "rocksdb_admin/tests/librocksdb.so.5.4",
                   "operator": "StringAppendOperator (C-API merge operator, tests/oracle_string_append/sa_ref.c)",
                   "cases": out}, f, separators=(",", ":"))
    print("string_append.json", os.path.getsize(GOLDEN), "bytes")


if __name__ == "__main__":
    if "--generate" in sys.argv:
        generate()
