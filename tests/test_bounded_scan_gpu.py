"""GPU: bounded range reads — iterators with an upper bound and SeekForPrev (rsp_iter_set_upper_bound,
rsp_iter_seek_for_prev) and batched scans with an end key (rsp_multi_scan_bounded, rsp_multi_scan_bounded_device) —
against the reference's RocksDB binary (tests/golden/bounded_scans.json) and against the oracle port."""
import os
import random
import struct

import numpy as np
import pytest

import bounded_oracle as BO
import golden_util as G
from oracle import okv
from rocksplicator_b200.write_batch import WriteBatch

pytestmark = pytest.mark.gpu
EMUL = bool(os.environ.get("RSP_TEST_EMUL_LIB"))
if not EMUL:
    import torch
CASES = G.load("bounded_scans.json")
NOT_SUPPORTED, INCOMPLETE = 3, 7


@pytest.fixture(scope="module")
def eng():
    from rocksplicator_b200 import engine
    e = engine.Engine(0, l0_compaction_trigger=64)  # several runs stay side by side until a test compacts
    yield e
    e.close()


_n = [0]


def new_shard(eng, merge_op=0):
    _n[0] += 1
    return eng.open_shard("bnd%05d" % _n[0], merge_op=merge_op)


class EngineSide:
    def __init__(self, shard):
        self.s = shard

    def apply(self, batch): return self.s.apply(batch, 0)
    def flush(self): return self.s.flush()
    def compact(self): return self.s.compact()
    def snapshot(self): return self.s.snapshot()
    def release(self, snap): snap.release()

    def iterator(self, upper_bound, snapshot):
        return (snapshot or self.s).iterator(upper_bound=upper_bound)


def put_all(shard, db, rows):
    for k, v in rows:
        b = WriteBatch().put(k, v).data()
        assert shard.apply(b, 0) == 0
        if db is not None:
            assert db.apply(b, 0) == 0


def want_scan(rows, start, end, limit):
    """live (key, value) of sorted Put-only rows in [start, end), at most limit"""
    return [(k, v) for k, v in rows if k >= start and (end is None or k < end)][:limit]


@pytest.mark.parametrize("name", BO.case_names())
def test_golden_bounded_iterators(eng, name):
    merge, layout = name.split("-", 1)
    s = new_shard(eng, BO.MERGES[merge])
    assert BO.run_case(EngineSide(s), layout) == CASES[name]
    s.close()


# ---- the fast path: one compacted run of fixed-size Puts ---------------------------------------------------------------
@pytest.fixture(scope="module")
def fixed_run(eng):
    s = new_shard(eng)
    rows = [(b"key-%012d" % (3 * i), bytes([i & 0xff]) * 64) for i in range(2000)]
    put_all(s, None, rows)
    assert s.compact() == 0
    assert s.stats()["n_runs"] == 1
    yield s, rows
    s.close()


def test_fast_path_bounds(eng, fixed_run):
    s, rows = fixed_run
    keys = [k for k, _ in rows]
    starts, ends = [], []
    marks = [keys[0], keys[-1], b"a", b"z", b""] + [keys[j] for j in range(0, len(keys), 32)] + \
            [keys[j] for j in range(7, len(keys), 32)] + [keys[j] + b"\0" for j in range(31, len(keys), 97)] + \
            [b"key-", b"key-00000000001"]
    rng = random.Random(1)
    for e in marks:
        for st in (keys[0], b"", rng.choice(keys), e, keys[max(0, keys.index(e) - 40)] if e in keys else b"key-0"):
            starts.append(st)
            ends.append(e)
    for max_entries in (128, 16):
        res = eng.multi_scan([s.index] * len(starts), starts, max_entries, 128 * 96, ends=ends)
        for st, e, (rc, recs) in zip(starts, ends, res):
            assert rc == 0 and recs == want_scan(rows, st, e, max_entries), (st, e, max_entries)


def test_fast_path_incomplete_with_bound(eng, fixed_run):
    s, rows = fixed_run
    keys = [k for k, _ in rows]
    # room for 5 records of 8 + 16 + 64 bytes; the bound leaves 10 (INCOMPLETE) or 3 (complete)
    res = eng.multi_scan([s.index] * 2, [keys[100], keys[100]], 128, 5 * 88, ends=[keys[110], keys[103]])
    assert res[0] == (INCOMPLETE, want_scan(rows, keys[100], keys[105], 128))
    assert res[1] == (0, want_scan(rows, keys[100], keys[103], 128))


def test_bounded_equals_unbounded_cut(eng, fixed_run):
    """random (start, end) pairs: the bounded scan is the unbounded scan cut at end"""
    s, rows = fixed_run
    keys = [k for k, _ in rows]
    rng = random.Random(7)
    starts, ends = [], []
    for _ in range(300):
        a = rng.choice(keys) if rng.random() < 0.7 else b"key-%012d" % rng.randrange(6100)
        b = rng.choice(keys) if rng.random() < 0.7 else b"key-%012d" % rng.randrange(6100)
        starts.append(a)
        ends.append(b)
    six = [s.index] * len(starts)
    full = eng.multi_scan(six, starts, 128, 128 * 96)
    cut = eng.multi_scan(six, starts, 128, 128 * 96, ends=ends)
    for e, (rc0, r0), (rc1, r1) in zip(ends, full, cut):
        assert rc0 == rc1 == 0 and r1 == [(k, v) for k, v in r0 if k < e]


# ---- the general path: several runs, variable sizes, merges and deletes ------------------------------------------------
def general_stream(shard, db, seed, n_rounds=4):
    """random writes with a flush after every round but the last (several runs + a memtable)"""
    rng = random.Random(seed)
    keys = [b"g%0*d" % (rng.choice((2, 5, 11)), i) for i in range(0, 400, 3)]
    for rnd in range(n_rounds):
        for _ in range(150):
            k, r = rng.choice(keys), rng.random()
            wb = WriteBatch()
            if r < 0.55:
                wb.put(k, bytes(rng.randrange(256) for _ in range(rng.randrange(0, 90))))
            elif r < 0.75:
                wb.delete(k)
            else:
                wb.merge(k, struct.pack("<Q", rng.randrange(1 << 40)))
            b = wb.data()
            assert shard.apply(b, 0) == 0 and db.apply(b, 0) == 0
        if rnd < n_rounds - 1:
            assert shard.flush() == 0
    return sorted(set(keys))


def random_moves(rng, it, probes):
    got = []
    for _ in range(10):
        m = rng.randrange(6)
        if m == 0:
            it.seek_to_first()
        elif m == 1:
            it.seek_to_last()
        elif m == 2:
            it.seek(rng.choice(probes))
        elif m == 3:
            it.seek_for_prev(rng.choice(probes))
        elif it.valid():
            it.next() if m == 4 else it.prev()
        got.append(BO._state(it))
    return got


@pytest.mark.parametrize("seed", range(3))
def test_general_path_iterators_and_scans_match_port(eng, seed):
    s = new_shard(eng, okv.MERGE_UINT64ADD)
    db = BO.BoundedOkv(BO.load_port(), merge_op=okv.MERGE_UINT64ADD)
    keys = general_stream(s, db, seed)
    assert s.stats()["n_runs"] >= 2 and s.stats()["memtable_entries"] > 0
    rng = random.Random(100 + seed)
    probes = keys + [k + b"\0" for k in keys[::5]] + [b"g", b"g1", b"g00000", b"h", b""]
    # iterators: the memtable becomes the iterator's private run; a snapshot is taken before later writes
    snap_e, snap_o = s.snapshot(), db.snapshot()
    wb = WriteBatch().put(keys[3], b"late").delete(keys[10]).data()
    assert s.apply(wb, 0) == 0 and db.apply(wb, 0) == 0
    for i in range(40):
        bound = None if i % 10 == 0 else rng.choice(probes)
        at = i % 2 == 1
        ie = (snap_e if at else s).iterator(upper_bound=bound)
        io = db.iterator(snap_o if at else None, bound)
        r = rng.random()
        assert random_moves(random.Random(r), ie, probes) == random_moves(random.Random(r), io, probes), (i, bound, at)
        ie.close()
        io.close()
    snap_e.release()
    snap_o.release()
    # batched scans (the memtable is flushed first): bounded, and with max_entries below the range
    starts = [rng.choice(probes) for _ in range(60)]
    ends = [rng.choice(probes) for _ in range(60)]
    for max_entries in (200, 5):
        res = eng.multi_scan([s.index] * 60, starts, max_entries, 64 * 1024, ends=ends)
        for a, b, (rc, recs) in zip(starts, ends, res):
            assert rc == 0 and recs == db.scan(start=a, end=b, limit=max_entries), (a, b)
    db.close()
    s.close()


def test_keys_beyond_the_bound_are_not_read(eng):
    """tombstones, host-folded (append) keys and failing counter merges at or beyond the end raise nothing"""
    from rocksplicator_b200 import engine
    rows = [(b"p%03d" % i, b"v%d" % i) for i in range(50)]
    for merge, tail in ((engine.MERGE_COUNTER, [("put", b"q1", b"abc"), ("merge", b"q1", struct.pack("<q", 5))]),
                        (engine.MERGE_APPEND, [("merge", b"q1", b"x"), ("merge", b"q1", b"y")])):
        s = new_shard(eng, merge)
        db = BO.BoundedOkv(BO.load_port(), merge_op=merge)
        put_all(s, db, rows)
        assert s.flush() == 0
        for op in [("del", b"p%03d" % i, None) for i in range(40, 50)] + tail:
            wb = WriteBatch()
            if op[0] == "put":
                wb.put(op[1], op[2])
            elif op[0] == "merge":
                wb.merge(op[1], op[2])
            else:
                wb.delete(op[1])
            assert s.apply(wb.data(), 0) == 0 and db.apply(wb.data(), 0) == 0
        bounded = eng.multi_scan([s.index] * 3, [b"p", b"p030", b"p045"], 100, 8192, ends=[b"p040", b"q1", b"q"])
        assert bounded == [(0, want_scan(rows, b"p", b"p040", 100)), (0, want_scan(rows, b"p030", b"p040", 100)),
                           (0, [])]
        full = eng.multi_scan([s.index], [b"p"], 100, 8192)
        assert full[0][0] != 0  # unbounded, the scan reaches q1 and reports it
        for bound in (b"p040", b"q1", b"q"):
            ie, io = s.iterator(upper_bound=bound), db.iterator(upper_bound=bound)
            for it in (ie, io):
                it.seek(b"p035")
            ge, go = [], []
            while ie.valid():
                ge.append(BO._state(ie))
                ie.next()
            while io.valid():
                go.append(BO._state(io))
                io.next()
            assert ge == go and ie.status() == io.status() == 0, bound
            ie.close()
            io.close()
        db.close()
        s.close()


# ---- the device form on a caller's stream ------------------------------------------------------------------------------
def test_device_form_on_caller_stream(eng, fixed_run):
    s, rows = fixed_run
    keys = [k for k, _ in rows]
    rng = random.Random(3)
    n, max_entries, stride = 512, 64, 64 * 88
    st_i = [rng.randrange(len(keys)) for _ in range(n)]
    en_i = [min(len(keys) - 1, i + rng.randrange(-5, 100)) for i in st_i]
    six = np.full(n, s.index, dtype=np.uint32)
    kq = np.frombuffer(b"".join(keys[i] for i in st_i), dtype=np.uint8)
    ke = np.frombuffer(b"".join(keys[i] for i in en_i), dtype=np.uint8)
    arrays = [six, kq, ke, np.zeros(n * stride, np.uint8), np.zeros(n, np.uint32), np.full(n, -1, np.int32)]
    if EMUL:
        d = [a.copy() for a in arrays]
        ptr = [a.ctypes.data for a in d]
        stream = eng.lib.rsp_engine_stream(eng.h)
    else:
        d = [torch.from_numpy(a.copy()).cuda() for a in arrays]
        torch.cuda.synchronize()
        ptr = [t.data_ptr() for t in d]
        stream = torch.cuda.Stream()
    rc = eng.lib.rsp_multi_scan_bounded_device(eng.h, n, ptr[0], ptr[1], 16, ptr[2], 16, max_entries, ptr[3], stride,
                                               ptr[4], ptr[5], stream if EMUL else stream.cuda_stream)
    assert rc == 0
    if not EMUL:
        stream.synchronize()
        d = [t.cpu().numpy() for t in d]
    out, n_out, st = d[3], d[4], d[5]
    for q in range(n):
        want = want_scan(rows, keys[st_i[q]], keys[en_i[q]], max_entries)
        assert st[q] == 0 and n_out[q] == len(want), q
        at = q * stride
        for k, v in want:
            kl, vl = struct.unpack_from("<II", out, at)
            assert (out[at + 8:at + 8 + kl].tobytes(), out[at + 8 + kl:at + 8 + kl + vl].tobytes()) == (k, v)
            at += 8 + kl + vl
