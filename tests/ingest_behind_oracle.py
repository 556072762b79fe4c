"""Scripted ingest-behind cases and their answers from the reference's own RocksDB (librocksdb.so.5.4, through
oracle/ref_driver.c), recorded in tests/golden/ingest_behind.json; tests/test_ingest_behind_gpu.py replays them on the
engine.

RocksDB 5.4 predates ingest_behind, but pins its visible results exactly: a file F ingested behind a history H reads
like F ingested into an empty DB first (the file takes no sequence number there, as rocksdb_assumption_test.cpp:248-283
and tests/golden/reference_runs.json show), then H.  So at every checkpoint of a case the reference DB is rebuilt: every
behind file seen so far ingested first as an SST file, then every write so far.  A checkpoint records the latest sequence
number and fingerprints of the forward scan, of MultiGet of the case's probe keys (statuses included), and of bounded
forward and reverse scans over the seams between the files and the writes.

    python tests/ingest_behind_oracle.py --generate     (needs oracle/_ref, which build() makes)
"""
import ctypes as C
import json
import os
import random
import struct
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from rocksplicator_b200.write_batch import WriteBatch  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "ingest_behind.json")
MERGES = {"none": 0, "counter": 1, "uint64add": 2}


def key(i):
    return b"k%015d" % i


def _val(op, rnd):
    return struct.pack("<q", rnd.randrange(-1000, 1000)) if op != "none" else rnd.randbytes(rnd.randrange(0, 30))


def _file(op, rnd, ks, bad=()):
    return [(key(i), b"bad" if i in bad else _val(op, rnd)) for i in ks]


def cases():
    """name -> (merge operator, steps, probe keys, seams, scans checked).  Steps: ("w", [batch]), ("flush",),
    ("compact",), ("behind", rows), ("check",)"""
    out = {}
    for op in MERGES:
        rnd = random.Random("history-" + op)
        w1 = [WriteBatch().put(key(i), _val(op, rnd)).data() for i in range(0, 200, 2)]
        w1 += [WriteBatch().delete(key(i)).data() for i in range(0, 200, 10)]
        w1 += [WriteBatch().single_delete(key(i)).data() for i in range(1000, 1010)]
        if op != "none":
            w1 += [WriteBatch().merge(key(i), _val(op, rnd)).data() for i in range(0, 200, 3)]
        w2 = [WriteBatch().delete(key(i)).data() for i in range(201, 260, 4)]
        w3 = [WriteBatch().put(key(i), _val(op, rnd)).data() for i in range(100, 140, 3)]
        if op != "none":  # merges whose base arrives behind them later
            w3 += [WriteBatch().merge(key(i), _val(op, rnd)).data() for i in range(3000, 3010)]
        steps = [("w", w1), ("flush",), ("w", w2), ("compact",), ("check",),
                 ("behind", _file(op, rnd, range(0, 300))), ("check",), ("w", w3), ("check",),
                 ("behind", _file(op, rnd, range(3000, 3020))), ("check",), ("compact",), ("check",)]
        out["history_then_behind-" + op] = (op, steps, [key(i) for i in list(range(0, 320, 7)) + list(range(2995, 3025))],
                                            [(key(0), key(40)), (key(190), key(310)), (key(2990), key(3030))], True)
    rnd = random.Random("disjoint")
    steps = [("behind", _file("none", rnd, range(0, 100, 3))), ("w", [WriteBatch().put(key(i), b"w%d" % i).data()
                                                                     for i in range(50, 250, 5)]),
             ("check",), ("behind", _file("none", rnd, range(200, 300, 2))), ("flush",), ("check",),
             ("behind", _file("none", rnd, range(100, 200, 4))), ("compact",), ("check",)]
    out["several_disjoint_files"] = ("none", steps, [key(i) for i in range(0, 310, 3)],
                                     [(key(90), key(110)), (key(195), key(205)), (key(0), key(400))], True)
    rnd = random.Random("delete")
    steps = [("w", [WriteBatch().put(key(5), b"x").data(), WriteBatch().delete(key(5)).data(),
                    WriteBatch().delete(key(6)).data()]), ("flush",), ("compact",),
             ("behind", _file("none", rnd, range(0, 10))), ("check",), ("compact",), ("check",)]
    out["delete_compact_then_behind"] = ("none", steps, [key(i) for i in range(12)], [(key(0), key(10))], True)
    rnd = random.Random("failing")
    steps = [("w", [WriteBatch().merge(key(i), struct.pack("<q", i)).data() for i in range(20)]
              + [WriteBatch().merge(key(7), b"abc").data()]), ("flush",), ("compact",),
             ("behind", _file("counter", rnd, range(20), bad=range(0, 20, 4))), ("check",),
             ("w", [WriteBatch().merge(key(i), struct.pack("<q", 1)).data() for i in range(0, 20, 3)]), ("check",)]
    out["failing_counter_merges"] = ("counter", steps, [key(i) for i in range(22)], [], False)
    return out


def record(side, probes, seams, scans):
    """one checkpoint on a side with latest_seq / scan / multi_get / fwd(start, end) / rev(start, end)"""
    r = [side.latest_seq(), side.multi_get(probes)]
    if scans:
        r.append(side.scan())
        for lo, hi in seams:
            r.append(side.fwd(lo, hi))
            r.append(side.rev(lo, hi))
    return r


class RefSide:
    def __init__(self, db):
        self.db = db

    def latest_seq(self):
        return self.db.latest_seq()

    def multi_get(self, keys):
        return [tuple(x) for x in self.db.multi_get(keys)]

    def scan(self):
        return self.db.scan()

    def fwd(self, lo, hi):
        it, out = self.db.iterator(), []
        it.seek(lo)
        while it.valid() and it.key() < hi:
            out.append((it.key(), it.value()))
            it.next()
        it.close()
        return out

    def rev(self, lo, hi):
        it, out = self.db.iterator(), []
        it.seek(hi)
        if it.valid():
            it.prev()
        else:
            it.seek_to_last()
        while it.valid() and it.key() >= lo:
            out.append((it.key(), it.value()))
            it.prev()
        it.close()
        return out


def generate():
    import golden_util as G
    from rocksplicator_b200 import sst
    from snapshot_oracle import SnapOkv, load_ref
    ref = load_ref()
    tmp = tempfile.mkdtemp()
    out = {}
    for name, (op, steps, probes, seams, scans) in cases().items():
        recs = []
        for c, st in enumerate(steps):
            if st[0] != "check":
                continue
            db = SnapOkv(ref, merge_op=MERGES[op])
            for j, s in enumerate(steps[:c]):  # the files first
                if s[0] == "behind":
                    path = os.path.join(tmp, "%s-%d.sst" % (name, j))
                    open(path, "wb").write(sst.write_sst(s[1]))
                    err = C.create_string_buffer(256)
                    assert ref.okv_ingest_sst_consistency(db.h, path.encode(), 1, 1, err, 256) == 0, err.value
            assert db.latest_seq() == 0
            for s in steps[:c]:  # then the writes (flushes and compactions change no visible contents: a compaction
                if s[0] == "w":  # that folds a failing merge would latch the DB's background error instead)
                    for b in s[1]:
                        assert db.apply(b, 7) == 0, (name, db.last_error)
            r = record(RefSide(db), probes, seams, scans)
            recs.append([c, r[0]] + [G.digest(x) for x in r[1:]])
            db.close()
        out[name] = recs
    with open(GOLDEN, "w") as f:
        json.dump({"generator": "tests/ingest_behind_oracle.py --generate",
                   "source": "rocksdb_admin/tests/librocksdb.so.5.4", "cases": out}, f, indent=0, separators=(",", ":"))
    print("ingest_behind.json", os.path.getsize(GOLDEN), "bytes")


if __name__ == "__main__":
    if "--generate" in sys.argv:
        generate()
    else:
        print(__doc__)
