"""Seeded snapshot scenarios shared by oracle/gen_golden.py (which records what the reference's RocksDB binary answers,
tests/golden/snapshots.json) and the tests that replay them on the oracle port and on the engine.

A scenario drives one DB through a side object (OkvSide for the oracle, EngineSide for an engine shard) and returns a
list of events: ["snap", seq], ["release", i] and, at the end, ["view", i or "latest", fingerprint] for every live
snapshot and the latest state.  Snapshots are taken at random points, with flushes and compactions in between.
"""
import random

from streams import random_stream

MERGES = {"none": 0, "counter": 1, "uint64add": 2, "append": 3}
STREAM_CASES = [(m, seed) for m in ("counter", "uint64add", "append", "none") for seed in (0, 1)]


class OkvSide:
    """an oracle DB with snapshot reads (tests/snapshot_oracle.py: the port or the reference's binary)"""

    def __init__(self, db):
        self.db = db

    def apply(self, b, ts): return self.db.apply(b, ts)
    def latest_seq(self): return self.db.latest_seq()
    def flush(self): return self.db.flush()
    def compact(self): return self.db.compact()
    def snapshot(self): return self.db.snapshot()
    def release(self, s): s.release()
    def get(self, k, s=None): return self.db.get(k, snapshot=s)
    def multi_get(self, keys, s=None): return self.db.multi_get(keys, snapshot=s)
    def iterator(self, s=None): return self.db.iterator(s)


class EngineSide:
    """an engine shard (rocksplicator_b200.engine.Shard) read through its snapshots"""

    def __init__(self, shard):
        self.shard = shard

    def apply(self, b, ts): return self.shard.apply(b, ts)
    def latest_seq(self): return self.shard.latest_seq()
    def flush(self): return self.shard.flush()
    def compact(self): return self.shard.compact()
    def snapshot(self): return self.shard.snapshot()
    def release(self, s): s.release()
    def get(self, k, s=None): return s.get(k) if s is not None else self.shard.get(k)
    def multi_get(self, keys, s=None): return s.multi_get(keys) if s is not None else self.shard.multi_get(keys)
    def iterator(self, s=None): return s.iterator() if s is not None else self.shard.iterator()


def observe(side, keys, snap=None):
    """everything a reader sees at `snap` (None = latest): Get, MultiGet with duplicates and a miss, forward and
    backward walks, a few Seeks with Next / Prev, the iterator's status"""
    probe = list(keys) + [b"zz-missing"] + list(keys[:3])
    it = side.iterator(snap)
    fwd, rev, seeks = [], [], []
    it.seek_to_first()
    while it.valid():
        fwd.append((it.key(), it.value()))
        it.next()
    it.seek_to_last()
    while it.valid():
        rev.append((it.key(), it.value()))
        it.prev()
    for k in list(keys[:6]) + [b"", b"\x00", b"m", b"\xff\xff"]:
        it.seek(k)
        row = [k]
        for step in ("next", "prev", "prev"):
            row.append((it.key(), it.value()) if it.valid() else None)
            if not it.valid():
                break
            getattr(it, step)()
        seeks.append(row)
    st = it.status()
    it.close()
    return [[side.get(k, snap) for k in probe], side.multi_get(probe, snap), fwd, rev, seeks, st]


def run_stream(side, merge, seed, digest):
    """one seeded stream with snapshots taken, released, flushed over and compacted over at random points"""
    rng = random.Random(7000 + 31 * seed + MERGES[merge])
    keys, stream = random_stream(5000 + 17 * seed + MERGES[merge], 70, n_keys=24,
                                 merge=None if merge == "none" else ("counter" if merge == "uint64add" else merge))
    ev, live = [], {}
    for i, (b, ts) in enumerate(stream):
        ev.append(["apply", side.apply(b, ts)])
        r = rng.random()
        if r < 0.15:
            j = len(ev)
            live[j] = side.snapshot()
            ev.append(["snap", live[j].seq])
        elif r < 0.22:
            side.flush()
        elif r < 0.26:
            side.compact()
        elif r < 0.30 and live:
            j = rng.choice(sorted(live))
            side.release(live.pop(j))
            ev.append(["release", j])
    for j in sorted(live):
        ev.append(["view", j, digest(observe(side, keys, live[j]))])
    ev.append(["view", "latest", side.latest_seq(), digest(observe(side, keys))])
    for j in sorted(live):
        side.release(live.pop(j))
    return ev


INGEST_BASE = [(b"k%04d" % i, b"base-%d" % i) for i in range(0, 200, 2)]


def ingest_steps():
    """(name, rows, allow_global_seqno, take a snapshot first): ingestion while snapshots are live.  Each step runs on
    a fresh DB holding INGEST_BASE (flushed) and a snapshot taken before the ingestion."""
    beyond = [(b"z%04d" % i, b"beyond-%d" % i) for i in range(20)]
    overlap = [(b"k%04d" % i, b"over-%d" % i) for i in range(0, 60, 3)]
    return [
        ("beyond-allow", beyond, True, True),
        ("beyond-refuse", beyond, False, True),
        ("overlap-allow", overlap, True, True),
        ("overlap-refuse", overlap, False, True),
        ("beyond-refuse-no-snapshot", beyond, False, False),
        ("empty-db-allow", beyond, True, True),
    ]


def run_ingest(side, name, rows, allow, with_snapshot, ingest, digest):
    """one step of ingest_steps() on a fresh DB: `ingest(rows, allow)` -> (rc, text).  Returns [name, rc, text, latest
    seq, snapshot seq, view at the old snapshot, view at a snapshot taken afterwards, latest view]."""
    base = [] if name.startswith("empty-db") else INGEST_BASE
    for k, v in base:
        assert side.apply(_put(k, v), 1) == 0
    if base:
        side.flush()
    old = side.snapshot() if with_snapshot else None
    rc, text = ingest(rows, allow)
    new = side.snapshot()
    keys = [k for k, _ in base[:8]] + [k for k, _ in rows[:6]]
    out = [name, rc, text, side.latest_seq(), old.seq if old else None,
           digest(observe(side, keys, old)) if old else None, digest(observe(side, keys, new)),
           digest(observe(side, keys))]
    if old:
        side.release(old)
    side.release(new)
    return out


def _put(k, v):
    from rocksplicator_b200.write_batch import WriteBatch
    return WriteBatch().put(k, v).data()
