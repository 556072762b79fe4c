"""Reverse range reads on the oracle (TEST INFRASTRUCTURE ONLY): batched reverse scans (rsp_multi_scan_reverse) stated
as the iterator walk they stand for -- SeekForPrev(key) (SeekToLast without a key), one Prev past the start key when the
scan is exclusive and the iterator landed on it, then Prev until max_entries or a key below the low -- on the port and on
the reference's own RocksDB binary, and the edge cases recorded from the binary into tests/golden/reverse_scans.json.

It uses the bounded oracle libraries of tests/bounded_oracle.py as they are (SeekForPrev, SeekToLast and Prev are already
exported by both).

    python tests/reverse_oracle.py --generate    # tests/golden/reverse_scans.json from the binary
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import bounded_oracle as BO  # noqa: E402
from rocksplicator_b200.write_batch import WriteBatch  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "reverse_scans.json")
load_port, load_ref, MERGES = BO.load_port, BO.load_ref, BO.MERGES


def reverse_walk(it, key, exclusive, low, max_entries):
    """the walk a reverse scan stands for, on an unbounded iterator -> {"pre": the status raised on an excluded start key
    (0 when none was excluded), "taken": [[key hex, value hex, status on landing]], "stop": [key hex or None, status]
    where the walk stopped (None when it stopped at max_entries)}"""
    pre = 0
    if key is None:
        it.seek_to_last()
    else:
        it.seek_for_prev(key)
        if exclusive and it.valid() and it.key() == key:
            pre = it.status()
            it.prev()
    taken, stop = [], None
    while True:
        if len(taken) == max_entries:
            break
        if not it.valid() or (low is not None and it.key() < low):
            stop = [it.key().hex() if it.valid() else None, it.status()]
            break
        taken.append([it.key().hex(), it.value().hex(), it.status()])
        it.prev()
    return {"pre": pre, "taken": taken, "stop": stop}


def expected_scan(walk):
    """what rsp_multi_scan_reverse answers for a recorded walk -> (status, [(key, value)]).  DBIter's status is sticky,
    so the binary cannot tell a failing merge on an excluded start key (walk["pre"]) or below the low (walk["stop"])
    from one among the keys taken; the scan reads neither.  The status of the scan is the one the walk first raised on a
    key it took.  (In the recorded data sets k60 is the one key whose merge fails, so a status already raised before the
    first key taken is always k60's, excluded; the port pins that case too.)"""
    st, prev = 0, walk["pre"]
    for _, _, s in walk["taken"]:
        if s and not prev and not st:
            st = s
        prev = s
    return st, [(bytes.fromhex(k), bytes.fromhex(v)) for k, v, _ in walk["taken"]]


# ---- the recorded edge cases ------------------------------------------------------------------------------------------
# the write phases of tests/bounded_oracle.py: k30 ends deleted, k40 and k85 hold merge operands only, k60 an operand on
# a 3-byte Put (a counter merge that fails; uint64add counts it as 0; append appends), k70 and k90 end deleted; the last
# phase stays in the memtable (RocksDB fails a flush that would merge k60)
PHASES = BO.PHASES
# fixed-size Puts (16-byte keys, 8-byte values) for the one-compacted-run fast path; "D" deletes two of them
FIXED = [("put", b"key-%012d" % (3 * i), b"v%07d" % i) for i in range(40)]
FIXED_DEL = [("del", b"key-%012d" % (3 * i), None) for i in (5, 6)]
LAYOUTS = {
    "mem": ["A", "B", "C"],                                    # memtable only
    "run+mem": ["A", "B", "flush", "C"],                       # a flush without a merge
    "runs+mem": ["A", "flush", "B", "flush", "C"],             # several runs of mixed shapes
    "compacted+mem": ["A", "flush", "B", "flush", "compact", "C"],  # a compaction over tombstones
    "fixed": ["F", "D", "compact"],                            # one compacted run of fixed-size Puts
}
# start keys: a live key, a deleted key, a merge-only key, the failing merge key, between keys, before the first key,
# past the last key, the empty key, none (SeekToLast); fixed layout: a live key, between keys, a deleted key
STARTS = [b"k50", b"k30", b"k40", b"k60", b"k55", b"a", b"z", b"", None]
FIXED_STARTS = [b"key-000000000030", b"key-000000000031", b"key-000000000015", b"key-", b"z", None]


def walks(layout):
    """(start, exclusive, low, max_entries) of every recorded walk on a layout"""
    fixed = layout == "fixed"
    # every start, inclusive and exclusive: where the walk lands and its first entries
    out = [(s, x, None, 3) for s in (FIXED_STARTS if fixed else STARTS) for x in (0, 1)]
    # lows from one start: at a key, between keys, equal to the start, above the start (empty), a prefix of longer keys,
    # the empty key; and (general layouts) the failing merge key k60 just below the low
    if fixed:
        s, lows = b"key-000000000030", [b"key-000000000012", b"key-000000000013", b"key-000000000030",
                                        b"key-000000000031", b"key-00000000001", b""]
    else:
        s, lows = b"k80", [b"k50", b"k55", b"k80", b"k81", b"k6", b"", b"k65"]
    out += [(s, x, lo, 100) for lo in lows for x in (0, 1)]
    # limits: 1, the exact count (three live keys), more than exist; and the whole shard from its last key
    s = b"key-000000000006" if fixed else b"k40"
    out += [(s, 0, None, m) for m in (1, 3, 6)] + [(None, 0, None, 100)]
    return out


def _apply(side, ops):
    for op in ops:
        wb = WriteBatch()
        if op[0] == "put":
            wb.put(op[1], op[2])
        elif op[0] == "merge":
            wb.merge(op[1], op[2])
        else:
            wb.delete(op[1])
        assert side.apply(wb.data()) == 0, op


def build_layout(side, layout):
    """side: apply(batch) -> rc, flush(), compact()"""
    for step in LAYOUTS[layout]:
        if step in ("A", "B", "C"):
            _apply(side, PHASES["ABC".index(step)])
        elif step == "F":
            _apply(side, FIXED)
        elif step == "D":
            _apply(side, FIXED_DEL)
        elif step == "flush":
            assert side.flush() == 0
        else:
            assert side.compact() == 0


def walk_tag(w):
    s, x, lo, m = w
    return "%s|%d|%s|%d" % ("-" if s is None else s.hex(), x, "-" if lo is None else lo.hex(), m)


def run_walks(make_iter, layout):
    out = {}
    for w in walks(layout):
        it = make_iter()
        out[walk_tag(w)] = reverse_walk(it, *w)
        it.close()
    return out


def case_names():
    """every merge operator on every layout but "fixed", which holds Puts only and is recorded once"""
    return ["%s-%s" % (m, lay) for m in MERGES for lay in LAYOUTS if lay != "fixed"] + ["uint64add-fixed"]


def run_on_oracle(lib, name):
    merge, layout = name.split("-", 1)
    db = BO.BoundedOkv(lib, merge_op=MERGES[merge])
    try:
        build_layout(BO.OkvSide(db), layout)
        return run_walks(lambda: db.iterator(), layout)
    finally:
        db.close()


def generate():
    ref = load_ref()
    out = {name: run_on_oracle(ref, name) for name in case_names()}
    with open(GOLDEN, "w") as f:
        json.dump({"generator": "tests/reverse_oracle.py --generate", "source": "rocksdb_admin/tests/librocksdb.so.5.4",
                   "cases": out}, f, separators=(",", ":"), sort_keys=True)
        f.write("\n")
    print("reverse_scans.json", os.path.getsize(GOLDEN), "bytes")


if __name__ == "__main__":
    if "--generate" in sys.argv:
        generate()
    else:
        print(__doc__)
