"""Batched range scans at snapshots on the oracle (TEST INFRASTRUCTURE ONLY): rsp_multi_scan_at and
rsp_multi_scan_reverse_at stated as the iterator walks they stand for, on iterators created at a snapshot -- forward,
Seek(key) (SeekToFirst without a key), one Next past the start key when the scan is exclusive and the iterator landed on
it, then Next until max_entries or the upper bound; reverse, the walk of tests/reverse_oracle.py -- on the port and on
the reference's own RocksDB binary, and the edge cases recorded from the binary into tests/golden/snapshot_scans.json.

Every snapshot of a case is read at the end of the case, after all of its writes, flushes, merges of runs and
ingestion, so each recorded walk is what that snapshot held however the shard changed since.  It uses the oracle
libraries of tests/bounded_oracle.py as they are.

    python tests/snapshot_scan_oracle.py --generate    # tests/golden/snapshot_scans.json from the binary
"""
import ctypes as C
import json
import os
import shutil
import struct
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import bounded_oracle as BO  # noqa: E402
import reverse_oracle as RO  # noqa: E402
from rocksplicator_b200.write_batch import WriteBatch  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "snapshot_scans.json")
load_port, load_ref, MERGES = BO.load_port, BO.load_ref, BO.MERGES
reverse_walk, expected_scan = RO.reverse_walk, RO.expected_scan


def forward_walk(it, key, exclusive, max_entries):
    """the walk a forward scan stands for, on an iterator that carries the scan's end as its upper bound -> {"pre": the
    status raised on an excluded start key, "taken": [[key hex, value hex, status on landing]], "stop": [key hex or
    None, status] where the walk stopped (None when it stopped at max_entries)}; expected_scan reads it as it reads a
    reverse walk"""
    pre = 0
    if key is None:
        it.seek_to_first()
    else:
        it.seek(key)
        if exclusive and it.valid() and it.key() == key:
            pre = it.status()
            it.next()
    taken, stop = [], None
    while True:
        if len(taken) == max_entries:
            break
        if not it.valid():
            stop = [None, it.status()]
            break
        taken.append([it.key().hex(), it.value().hex(), it.status()])
        it.next()
    return {"pre": pre, "taken": taken, "stop": stop}


# ---- the recorded edge cases ------------------------------------------------------------------------------------------
def _op(n):
    return struct.pack("<q", n)


PHASES = BO.PHASES  # A, B, C: see tests/bounded_oracle.py (C holds the failing counter merge on k60: never flushed)
# six small phases between flushes: a view of up to RSP_MAX_RUNS = 8 runs (seven runs and the memtable's)
UPDATES = [[("put", b"k20", b"v20-%d" % i), ("merge", b"k40", _op(10 + i)), ("put", b"k5%d" % i, b"u5%d" % i),
            ("del", b"k5%d" % (i - 1)) if i else ("put", b"k15", b"v15")] for i in range(6)]
# ingested behind a live snapshot: a global sequence number; k10 overlaps a run, k05 and k15 fall between its keys
INGEST = [(b"k05", b"i05"), (b"k10", b"i10"), (b"k15", b"i15")]
# fixed-size Puts (16-byte keys, 8-byte values, two blocks of 32 entries); overwritten after the snapshot
FIXED, FIXED_DEL = RO.FIXED, RO.FIXED_DEL
FIXED_OVER = [("put", b"key-%012d" % (3 * i), b"w%07d" % i) for i in range(0, 40, 2)] + \
             [("put", b"key-%012d" % (3 * i + 1), b"n%07d" % i) for i in range(30, 34)]
# a layout is a list of steps: "A" "B" "C" (phases), "U0".."U5" (updates), "F" "D" "O" (fixed Puts, deletes, overwrite),
# "flush", "compact", "ingest", and "S<name>" (a snapshot, read at the end)
LAYOUTS = {
    # snapshots before overwrites, deletes and merges (s1), a flush (s2), a merge of runs (s3), an ingest (s4), and
    # with the memtable holding the failing merge (s5)
    # (once C is written nothing is flushed: RocksDB fails the flush that would merge k60)
    "timing": ["A", "flush", "Ss1", "B", "Ss2", "flush", "Ss3", "compact", "Ss4", "ingest", "C", "Ss5", "U0"],
    "compacted": ["A", "flush", "B", "compact", "Ss", "C"],        # one compacted run, written to afterwards
    "two-run": ["A", "B", "flush", "C", "Ss", "U0"],                 # a run and the memtable's
    "runs8": ["A", "flush"] + sum([["U%d" % i, "flush"] for i in range(6)], []) + ["C", "Ss", "U0"],
    "fixed": ["F", "D", "compact", "Ss", "O", "flush", "compact"],  # the fast path, overwritten afterwards
}
STARTS = RO.STARTS  # live, deleted, merge-only, failing merge, between keys, outside the range, empty, none
FIXED_STARTS = RO.FIXED_STARTS + [b"key-000000000093", b"key-000000000096"]  # the last of block 0, the first of block 1


def _fk(i):
    return b"key-%012d" % (3 * i)


def walks(layout):
    """(direction, start, exclusive, end or low, max_entries) of every recorded walk on a layout"""
    fixed = layout == "fixed"
    out = []
    for d in ("f", "r"):
        out += [(d, s, x, None, 3) for s in (FIXED_STARTS if fixed else STARTS) for x in (0, 1)]
    # ends (exclusive) from one start: at a key, between keys, equal to the start, a prefix of longer keys, just past
    # the failing merge key k60; fixed: on and around the block edge
    if fixed:
        s, ends = _fk(10), [_fk(31), _fk(32), _fk(31) + b"\0", _fk(10), b"key-00000000009", _fk(39) + b"\0"]
    else:
        s, ends = b"k10", [b"k50", b"k55", b"k10", b"k6", b"k600", b"k61"]
    out += [("f", s, x, e, 100) for e in ends for x in (0, 1)]
    # lows (inclusive) from one start: at a key, between keys, equal to the start, a prefix, the empty key, just above
    # the failing merge key
    if fixed:
        s, lows = _fk(33), [_fk(32), _fk(31), _fk(31) + b"\0", _fk(33), b"key-00000000009", b""]
    else:
        s, lows = b"k80", [b"k50", b"k55", b"k80", b"k6", b"", b"k65"]
    out += [("r", s, x, lo, 100) for lo in lows for x in (0, 1)]
    # limits: 1, 2, more than exist (the starts above take 3); and everything from either end, whose length is the
    # exact count that the engine's tests ask for as a limit
    fs, rs = (_fk(6), _fk(8)) if fixed else (b"k40", b"k50")
    out += [("f", fs, 0, None, m) for m in (1, 2, 100)] + [("r", rs, 0, None, m) for m in (1, 2, 100)]
    out += [("f", None, 0, None, 100), ("r", None, 0, None, 100)]
    return out


def walk_tag(w):
    d, s, x, e, m = w
    return "%s|%s|%d|%s|%d" % (d, "-" if s is None else s.hex(), x, "-" if e is None else e.hex(), m)


def run_walk(make_iter, w):
    """make_iter(upper_bound) -> an iterator at the snapshot"""
    d, s, x, e, m = w
    if d == "f":
        it = make_iter(e)
        out = forward_walk(it, s, x, m)
    else:
        it = make_iter(None)
        out = reverse_walk(it, s, x, e, m)
    it.close()
    return out


def _batch(op):
    wb = WriteBatch()
    if op[0] == "put":
        wb.put(op[1], op[2])
    elif op[0] == "merge":
        wb.merge(op[1], op[2])
    else:
        wb.delete(op[1])
    return wb.data()


def build_layout(side, layout):
    """side: apply(batch) -> rc, flush(), compact(), snapshot(), ingest(sorted rows).  Returns {name: snapshot} in the
    order taken."""
    snaps = {}
    for step in LAYOUTS[layout]:
        if step[0] == "S":
            snaps[step[1:]] = side.snapshot()
        elif step == "flush":
            assert side.flush() == 0
        elif step == "compact":
            assert side.compact() == 0
        elif step == "ingest":
            assert side.ingest(INGEST) == 0
        else:
            ops = {"A": PHASES[0], "B": PHASES[1], "C": PHASES[2], "F": FIXED, "D": FIXED_DEL, "O": FIXED_OVER}.get(step)
            for op in ops if ops is not None else UPDATES[int(step[1:])]:
                assert side.apply(_batch(op)) == 0, (layout, op)
    return snaps


def case_names():
    """every merge operator on every layout but "fixed", which holds Puts only and is recorded once"""
    return ["%s-%s" % (m, lay) for m in MERGES for lay in LAYOUTS if lay != "fixed"] + ["uint64add-fixed"]


class OkvSide(BO.OkvSide):
    """ingest: the binary ingests an SST file (with a global sequence number behind the live snapshots); the port has no
    ingestion and applies the rows as one batch of Puts, which every snapshot taken before it sees the same way"""

    def __init__(self, db, ref):
        super().__init__(db)
        self.ref = ref

    def ingest(self, rows):
        if not self.ref:
            wb = WriteBatch()
            for k, v in rows:
                wb.put(k, v)
            return self.db.apply(wb.data(), 0)
        from rocksplicator_b200 import sst
        tmp = tempfile.mkdtemp()
        try:
            path = os.path.join(tmp, "ingest.sst")
            with open(path, "wb") as f:
                f.write(sst.write_sst(rows))
            err = C.create_string_buffer(256)
            return self.db.lib.okv_ingest_sst_consistency(self.db.h, path.encode(), 1, 1, err, 256)
        finally:
            shutil.rmtree(tmp)


def run_on_oracle(lib, name, ref=False):
    merge, layout = name.split("-", 1)
    db = BO.BoundedOkv(lib, merge_op=MERGES[merge])
    try:
        snaps = build_layout(OkvSide(db, ref), layout)
        out = {}
        for sn, snap in snaps.items():
            out[sn] = {walk_tag(w): run_walk(lambda ub: db.iterator(snap, ub), w) for w in walks(layout)}
        for snap in snaps.values():
            snap.release()
        return out
    finally:
        db.close()


def generate():
    ref = load_ref()
    out = {name: run_on_oracle(ref, name, ref=True) for name in case_names()}
    with open(GOLDEN, "w") as f:
        json.dump({"generator": "tests/snapshot_scan_oracle.py --generate",
                   "source": "rocksdb_admin/tests/librocksdb.so.5.4", "cases": out}, f, separators=(",", ":"),
                  sort_keys=True)
        f.write("\n")
    print("snapshot_scans.json", os.path.getsize(GOLDEN), "bytes")


if __name__ == "__main__":
    if "--generate" in sys.argv:
        generate()
    else:
        print(__doc__)
