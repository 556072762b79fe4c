"""GPU: batched range scans at snapshots (rsp_multi_scan_at, rsp_multi_scan_reverse_at and their device forms) against
the reference's RocksDB binary (tests/golden/snapshot_scans.json), against the oracle port at the same snapshot, and
against the snapshot's own iterator walks."""
import os
import random
import struct

import numpy as np
import pytest

import bounded_oracle as BO
import golden_util as G
import snapshot_scan_oracle as SS
from oracle import okv

pytestmark = pytest.mark.gpu
EMUL = bool(os.environ.get("RSP_TEST_EMUL_LIB"))
if not EMUL:
    import torch
CASES = G.load("snapshot_scans.json")
NOT_SUPPORTED, INVALID, INCOMPLETE = 3, 4, 7
MAX_SNAPSHOTS = 4096


@pytest.fixture(scope="module")
def eng():
    from rocksplicator_b200 import engine
    e = engine.Engine(0, l0_compaction_trigger=64)  # several runs stay side by side until a test compacts
    yield e
    e.close()


_n = [0]


def new_shard(eng, merge_op=0):
    _n[0] += 1
    return eng.open_shard("sscan%05d" % _n[0], merge_op=merge_op)


class EngineSide:
    def __init__(self, shard):
        self.s = shard

    def apply(self, batch): return self.s.apply(batch, 0)
    def flush(self): return self.s.flush()
    def compact(self): return self.s.compact()
    def snapshot(self): return self.s.snapshot()
    def ingest(self, rows): return self.s.ingest(rows)


def apply_ops(shard, db, ops):
    for op in ops:
        b = SS._batch(op)
        assert shard.apply(b, 0) == 0
        if db is not None:
            assert db.apply(b, 0) == 0


def check_host_fold(got, want_recs):
    """a host-form scan over keys of a host-side operator: NotSupported, those keys as (key, None), the rest as wanted"""
    rc, recs = got
    assert rc == NOT_SUPPORTED and [k for k, _ in recs] == [k for k, _ in want_recs]
    assert any(v is None for _, v in recs)
    for (k, v), (_, w) in zip(recs, want_recs):
        assert v is None or v == w, k


def check(got, want, host_fold_ok):
    if host_fold_ok and got[0] == NOT_SUPPORTED:
        check_host_fold(got, want[1])
    else:
        assert got == want


def scan_at(eng, w_list, snaps):
    """one batched call per (direction, start or none, exclusive, end or none, max_entries) group of walks, each walk
    at its snapshot -> {(snapshot index, walk): result}"""
    groups = {}
    for i, w in w_list:
        d, s, x, e, m = w
        groups.setdefault((d, s is None, x, e is None, m), []).append((i, w))
    out = {}
    for (d, no_start, x, no_end, m), ws in groups.items():
        args = ([snaps[i] for i, _ in ws], None if no_start else [w[1] for _, w in ws], m, 16384)
        kw = dict(exclusive=bool(x))
        if d == "f":
            res = eng.multi_scan_at(*args, ends=None if no_end else [w[3] for _, w in ws], **kw)
        else:
            res = eng.multi_scan_reverse_at(*args, lows=None if no_end else [w[3] for _, w in ws], **kw)
        out.update(zip(ws, res))
    return out


# ---- 1. the fixture: batched scans at every snapshot of a case in one launch per group, and the snapshot iterators ----
@pytest.mark.parametrize("name", SS.case_names())
def test_golden_snapshot_scans(eng, name):
    merge, layout = name.split("-", 1)
    s = new_shard(eng, SS.MERGES[merge])
    snaps = SS.build_layout(EngineSide(s), layout)
    names, want = list(snaps), CASES[name]
    walks = SS.walks(layout)
    before = s.stats()
    res = scan_at(eng, [(i, w) for i in range(len(names)) for w in walks], [snaps[n] for n in names])
    for (i, w), got in res.items():
        check(got, SS.expected_scan(want[names[i]][SS.walk_tag(w)]), merge == "append")
    # the exact count as the limit: the whole snapshot from either end
    for i, sn in enumerate(names):
        for d in "fr":
            full = want[sn][SS.walk_tag((d, None, 0, None, 100))]
            n = len(full["taken"])
            fn = eng.multi_scan_at if d == "f" else eng.multi_scan_reverse_at
            got = fn([snaps[sn]], None, max(n, 1), 16384)[0]
            exp = SS.expected_scan(full)
            check(got, (exp[0], exp[1][:max(n, 1)]), merge == "append")
    assert s.stats() == before  # no flush, no run, no memtable change
    # the snapshot's iterator walks are the same walks
    for sn in names:
        for w in walks:
            assert SS.run_walk(lambda ub: snaps[sn].iterator(upper_bound=ub), w) == want[sn][SS.walk_tag(w)], (sn, w)
    for sp in snaps.values():
        sp.release()
    s.close()


# ---- 2. one launch over snapshots of several shards, operators and ages; invalid handles and slots ------------------
def general_stream(shard, db, rng, keys, n, vlen8=False, merges=True):
    """random Puts, Deletes and 8-byte merge operands (vlen8: 8-byte Put values, so that no counter merge fails)"""
    for _ in range(n):
        k, r = rng.choice(keys), rng.random()
        if r < 0.55 or (r >= 0.75 and not merges):
            op = ("put", k, bytes(rng.randrange(256) for _ in range(8 if vlen8 else rng.randrange(0, 40))))
        elif r < 0.75:
            op = ("del", k, None)
        else:
            op = ("merge", k, struct.pack("<Q", rng.randrange(1 << 40)))
        apply_ops(shard, db, [op])


def port_fwd(db, snap, start, exclusive, end, m):
    it = db.iterator(snap, end)
    w = SS.forward_walk(it, start, exclusive, m)
    it.close()
    return SS.expected_scan(w)


def port_rev(db, snap, start, exclusive, low, m):
    it = db.iterator(snap)
    w = SS.reverse_walk(it, start, exclusive, low, m)
    it.close()
    return SS.expected_scan(w)


def test_mixed_batch_and_invalid_handles(eng):
    rng = random.Random(5)
    keys = [b"m%05d" % i for i in range(0, 300, 3)]
    sides = []
    for merge in (okv.MERGE_NONE, okv.MERGE_UINT64ADD, okv.MERGE_COUNTER):
        s = new_shard(eng, merge)
        db = BO.BoundedOkv(BO.load_port(), merge_op=merge)
        for age in range(3):
            general_stream(s, db, rng, keys, 120, vlen8=True, merges=merge != okv.MERGE_NONE)
            sides.append((s, db, s.snapshot(), db.snapshot()))
            if age < 2:
                assert s.flush() == 0 and db.flush() == 0
    probes = keys + [b"m", b"m00001", b"n", b""]
    q = [(rng.randrange(len(sides)), rng.choice(probes), rng.choice(probes)) for _ in range(120)]
    snaps = [sides[i][2] for i, _, _ in q]
    snaps[7] = None
    snaps[50] = None
    for x in (False, True):
        fwd = eng.multi_scan_at(snaps, [a for _, a, _ in q], 40, 8192, ends=[b for _, _, b in q], exclusive=x)
        rev = eng.multi_scan_reverse_at(snaps, [b for _, _, b in q], 40, 8192, lows=[a for _, a, _ in q], exclusive=x)
        for j, ((i, a, b), f, r) in enumerate(zip(q, fwd, rev)):
            if snaps[j] is None:
                assert f == (INVALID, []) and r == (INVALID, []), j
                continue
            s, db, _, so = sides[i]
            assert f == port_fwd(db, so, a, x, b, 40), (j, a, b, x)
            assert r == port_rev(db, so, b, x, a, 40), (j, a, b, x)
    # a snapshot of another engine is foreign: InvalidArgument
    from rocksplicator_b200 import engine
    other = engine.Engine(0)
    os_ = other.open_shard("foreign")
    apply_ops(os_, None, [("put", b"m00000", b"x")])
    fs = os_.snapshot()
    assert eng.multi_scan_at([fs, sides[0][2]], [b"", b""], 5, 4096)[0] == (INVALID, [])
    fs.release()
    other.close()
    # the device form: a released slot and a slot past the table answer InvalidArgument for their own scans only
    released = sides[0][0].snapshot()
    dead = released.slot
    released.release()
    slots = [sides[3][2].slot, dead, MAX_SNAPSHOTS, MAX_SNAPSHOTS + 7, sides[8][2].slot]
    kq = [keys[10], keys[10], keys[10], keys[10], keys[20]]
    for rev in (False, True):
        got = device_scan(eng, slots, kq, 6, None, 20, 4096, rev, False)
        assert [g[0] for g in got[1:4]] == [INVALID] * 3 and [g[1] for g in got[1:4]] == [[]] * 3
        for j in (0, 4):
            want = (eng.multi_scan_reverse_at if rev else eng.multi_scan_at)([snaps_of(sides, slots[j])], [kq[j]], 20,
                                                                             4096)[0]
            assert got[j] == want, (rev, j)
    for s, db, se, so in sides:
        se.release()
        so.release()
    for s, db, _, _ in sides[::3]:
        db.close()
        s.close()


def snaps_of(sides, slot):
    return next(se for _, _, se, _ in sides if se.slot == slot)


def to_dev(arrays):
    """device copies of host arrays (under the emulation: host copies)"""
    if EMUL:
        return [a.copy() for a in arrays]
    d = [torch.from_numpy(a.copy()).cuda() for a in arrays]
    torch.cuda.synchronize()
    return d


def ptrs(d): return [a.ctypes.data if EMUL else a.data_ptr() for a in d]
def to_host(d): return d if EMUL else [t.cpu().numpy() for t in d]


def device_scan(eng, slots, keys, klen, ends, max_entries, stride, reverse, exclusive, caller_stream=True,
                decode=True):
    """the device form on a caller's stream (or the engine's) -> [(status, [(key, value)])] as the host form decodes
    them (statuses as the kernel wrote them); decode=False: (out, n_out, st) as written"""
    from rocksplicator_b200.engine import _scan_records
    n = len(slots)
    arrs = [np.array(slots, dtype=np.uint32), np.frombuffer(b"".join(keys) + b"\0", dtype=np.uint8) if keys else
            np.zeros(1, np.uint8), np.frombuffer(b"".join(ends) + b"\0", dtype=np.uint8) if ends else np.zeros(1, np.uint8),
            np.zeros(n * stride, np.uint8), np.zeros(n, np.uint32), np.full(n, -1, np.int32)]
    d = to_dev(arrs)
    p = ptrs(d)
    if caller_stream:
        stream = eng.lib.rsp_engine_stream(eng.h) if EMUL else torch.cuda.Stream()
        sh = stream if EMUL else stream.cuda_stream
    else:
        stream, sh = None, None
    fn = eng.lib.rsp_multi_scan_reverse_at_device if reverse else eng.lib.rsp_multi_scan_at_device
    assert fn(eng.h, n, p[0], p[1] if keys else None, klen if keys else 0, 1 if exclusive else 0,
              p[2] if ends else None, len(ends[0]) if ends else 0, max_entries, p[3], stride, p[4], p[5], sh) == 0
    if not EMUL:
        if stream is not None:
            stream.synchronize()
        torch.cuda.synchronize()
    out, n_out, st = to_host(d[3:])
    return _scan_records(out, n_out, st, n, stride) if decode else (out, n_out, st)


# ---- 3. no snapshot was ever taken on the engine ---------------------------------------------------------------------
def test_engine_without_snapshot_table_answers_invalid():
    from rocksplicator_b200 import engine
    e = engine.Engine(0)
    s = e.open_shard("nosnap")
    apply_ops(s, None, [("put", b"a%05d" % i, b"v") for i in range(50)])
    assert s.compact() == 0
    for rev in (False, True):
        got = device_scan(e, [0, 1, s.index, MAX_SNAPSHOTS - 1], [b"a00000"] * 4, 6, None, 10, 1024, rev, False)
        assert got == [(INVALID, [])] * 4
    assert e.multi_scan_at([None, None], None, 10, 1024) == [(INVALID, [])] * 2
    s.close()
    e.close()


# ---- 4. no side effects: a shard whose memtable holds writes -----------------------------------------------------------
def test_scans_at_snapshot_leave_the_shard_alone(eng):
    s = new_shard(eng, okv.MERGE_UINT64ADD)
    rows = [(b"s%04d" % i, b"v%d" % i) for i in range(200)]
    apply_ops(s, None, [("put", k, v) for k, v in rows[::2]])
    assert s.flush() == 0
    apply_ops(s, None, [("put", k, v) for k, v in rows[1::2]])
    snap = s.snapshot()
    apply_ops(s, None, [("put", b"s0000", b"later")])
    before = s.stats()
    assert before["memtable_entries"] > 0
    fwd = eng.multi_scan_at([snap] * 3, [b"s0000", b"s0100", b"s"], 50, 8192, ends=[b"s0010", b"t", b"s0002"])
    rev = eng.multi_scan_reverse_at([snap] * 2, None, 30, 8192, lows=[b"s0190", b""])
    device_scan(eng, [snap.slot], [b"s0000"], 5, None, 10, 2048, False, True)
    assert s.stats() == before
    assert fwd == [(0, rows[0:10]), (0, rows[100:150]), (0, rows[0:2])]
    assert rev == [(0, rows[:189:-1]), (0, rows[:169:-1])]
    # the latest-state scan flushes the same shard first
    assert eng.multi_scan([s.index], [b"s0000"], 2, 8192)[0] == (0, [(b"s0000", b"later"), rows[1]])
    after = s.stats()
    assert after["memtable_entries"] == 0 and after["n_runs"] != before["n_runs"]
    snap.release()
    s.close()


# ---- 5. what a snapshot held survives writes, flushes, merges and ingestion --------------------------------------------
def test_results_survive_later_changes():
    from rocksplicator_b200 import engine
    e = engine.Engine(0, l0_compaction_trigger=3)  # background merges replace the pinned runs
    s = e.open_shard("later", merge_op=okv.MERGE_UINT64ADD)
    db = BO.BoundedOkv(BO.load_port(), merge_op=okv.MERGE_UINT64ADD)
    rng = random.Random(9)
    keys = [b"t%04d" % i for i in range(0, 400, 4)]
    general_stream(s, db, rng, keys, 200)
    assert s.flush() == 0 and db.flush() == 0
    general_stream(s, db, rng, keys, 100)
    se, so = s.snapshot(), db.snapshot()
    starts = [rng.choice(keys) for _ in range(40)]
    ends = [rng.choice(keys) + b"5" for _ in range(40)]

    def read():
        return (e.multi_scan_at([se] * 40, starts, 30, 8192, ends=ends),
                e.multi_scan_reverse_at([se] * 40, ends, 30, 8192, lows=starts, exclusive=True))

    first = read()
    assert first[0] == [port_fwd(db, so, a, 0, b, 30) for a, b in zip(starts, ends)]
    assert first[1] == [port_rev(db, so, b, 1, a, 30) for a, b in zip(starts, ends)]
    steps = ["write", "flush", "compact", "background", "ingest"]
    for st in steps:
        if st == "write":
            general_stream(s, db, rng, keys, 150)
        elif st == "flush":
            assert s.flush() == 0
        elif st == "compact":
            assert s.compact() == 0
        elif st == "background":
            for _ in range(4):
                general_stream(s, None, rng, keys, 40)
                assert s.flush() == 0
        else:
            assert s.ingest([(k, b"ingested") for k in keys[::5]]) == 0
        assert read() == first, st
    se.release()
    so.release()
    db.close()
    s.close()
    e.close()


# ---- 6. paging through a snapshot with exclusive continuation ----------------------------------------------------------
def test_paging_through_a_snapshot(eng):
    s = new_shard(eng, okv.MERGE_UINT64ADD)
    db = BO.BoundedOkv(BO.load_port(), merge_op=okv.MERGE_UINT64ADD)
    rng = random.Random(11)
    keys = [b"p%05d" % i for i in range(0, 3000, 7)]
    apply_ops(s, db, [("put", k, b"v" + k) for k in keys])
    assert s.flush() == 0 and db.flush() == 0
    general_stream(s, db, rng, keys, 300)
    se, so = s.snapshot(), db.snapshot()
    full_f = port_fwd(db, so, None, 0, None, 10 ** 6)[1]
    full_r = port_rev(db, so, None, 0, None, 10 ** 6)[1]
    for reverse, full in ((False, full_f), (True, full_r)):
        got, last, turn = [], None, 0
        while True:
            fn = eng.multi_scan_reverse_at if reverse else eng.multi_scan_at
            rc, page = fn([se], None if last is None else [last], 37, 8192, exclusive=last is not None)[0]
            assert rc == 0
            got += page
            if len(page) < 37:
                break
            last = page[-1][0]
            turn += 1
            general_stream(s, None, rng, keys, 30)  # the shard moves on between pages
            if turn % 3 == 0:
                assert s.flush() == 0
            if turn % 7 == 0:
                assert s.compact() == 0
        assert got == full, reverse
    se.release()
    so.release()
    db.close()
    s.close()


# ---- 7. the fast path at block edges, overwritten after the snapshot ---------------------------------------------------
def want_fwd(rows, start, exclusive, end, limit):
    out = [(k, v) for k, v in rows
           if (start is None or k > start or (k == start and not exclusive)) and (end is None or k < end)]
    return out[:limit]


def want_rev(rows, start, exclusive, low, limit):
    out = [(k, v) for k, v in reversed(rows)
           if (start is None or k < start or (k == start and not exclusive)) and (low is None or k >= low)]
    return out[:limit]


@pytest.fixture(scope="module")
def fixed_snap(eng):
    s = new_shard(eng)
    rows = [(b"key-%012d" % (3 * i), bytes([i & 0xff]) * 64) for i in range(2000)]
    apply_ops(s, None, [("put", k, v) for k, v in rows])
    assert s.compact() == 0
    assert s.stats()["n_runs"] == 1 and s.stats()["memtable_entries"] == 0
    snap = s.snapshot()
    apply_ops(s, None, [("put", k, b"new") for k, _ in rows[::3]] + [("del", k, None) for k, _ in rows[1::5]])
    assert s.compact() == 0
    yield s, snap, rows
    snap.release()
    s.close()


def test_fast_path_block_edges_at_snapshot(eng, fixed_snap):
    s, snap, rows = fixed_snap
    keys = [k for k, _ in rows]
    edges = [keys[j] for j in range(0, len(keys), 32)] + [keys[j] for j in range(31, len(keys), 32)]
    marks = edges[::3] + [keys[0], keys[-1], b"a", b"z", b"key-", keys[500] + b"\0"]
    rng = random.Random(2)
    starts, bounds = [], []
    for m in marks:
        for b in (rng.choice(edges), m, rng.choice(keys), rng.choice(edges) + b"\0"):
            starts.append(m)
            bounds.append(b)
    sn = [snap] * len(starts)
    for x in (False, True):
        for me in (128, 16):
            f = eng.multi_scan_at(sn, starts, me, 128 * 96, ends=bounds, exclusive=x)
            r = eng.multi_scan_reverse_at(sn, starts, me, 128 * 96, lows=bounds, exclusive=x)
            for a, b, gf, gr in zip(starts, bounds, f, r):
                assert gf == (0, want_fwd(rows, a, x, b, me)), (a, b, x, me)
                assert gr == (0, want_rev(rows, a, x, b, me)), (a, b, x, me)
    # Incomplete: room for 5 records of 8 + 16 + 64 bytes
    res = eng.multi_scan_at([snap] * 2, [keys[100]] * 2, 128, 5 * 88, ends=[keys[110], keys[103]])
    assert res == [(INCOMPLETE, rows[100:105]), (0, rows[100:103])]


# ---- 8. reverse equals forward reversed, per operator (the general path) ----------------------------------------------
@pytest.mark.parametrize("merge", [okv.MERGE_UINT64ADD, okv.MERGE_COUNTER, okv.MERGE_APPEND])
def test_reverse_equals_forward_reversed_at_snapshot(eng, merge):
    s = new_shard(eng, merge)
    db = BO.BoundedOkv(BO.load_port(), merge_op=merge)
    rng = random.Random(20 + merge)
    keys = [b"g%0*d" % (rng.choice((2, 5, 11)), i) for i in range(0, 400, 3)]
    for rnd in range(4):
        general_stream(s, db, rng, keys, 150)
        if rnd < 3:
            assert s.flush() == 0 and db.flush() == 0
    se, so = s.snapshot(), db.snapshot()
    general_stream(s, db, rng, keys, 100)
    probes = sorted(set(keys)) + [b"g", b"g1", b"g00000", b"h", b""]
    a = [rng.choice(probes) for _ in range(80)]
    b = [rng.choice(probes) for _ in range(80)]
    fwd = eng.multi_scan_at([se] * 80, a, 500, 64 * 1024, ends=b)
    rev = eng.multi_scan_reverse_at([se] * 80, b, 500, 64 * 1024, lows=a, exclusive=True)
    for lo, hi, (rc0, r0), (rc1, r1) in zip(a, b, fwd, rev):
        assert rc1 == rc0 and r1 == r0[::-1], (lo, hi)
        port = port_fwd(db, so, lo, 0, hi, 10 ** 6)
        if rc1 == NOT_SUPPORTED:
            check_host_fold((rc1, r1), port[1][::-1])
        else:
            assert (rc0, r0) == port, (lo, hi)
    se.release()
    so.release()
    db.close()
    s.close()


# ---- 9. Incomplete and truncation with a failed merge ----------------------------------------------------------------
def test_incomplete_and_failed_merge(eng):
    s = new_shard(eng, okv.MERGE_COUNTER)
    db = BO.BoundedOkv(BO.load_port(), merge_op=okv.MERGE_COUNTER)
    apply_ops(s, db, [("put", b"f%02d" % i, b"v%02d" % i) for i in range(20)])
    assert s.flush() == 0 and db.flush() == 0
    apply_ops(s, db, [("put", b"f05", b"abc"), ("merge", b"f05", struct.pack("<q", 5))])  # a failing counter merge
    se, so = s.snapshot(), db.snapshot()
    fail_st, full = port_fwd(db, so, None, 0, None, 100)
    assert fail_st not in (0, INCOMPLETE) and (b"f05", b"") in full
    # room for 8 records of 8 + 3 + 3 bytes: the scan runs out of room after the failed merge
    got = eng.multi_scan_at([se] * 3, [b"f00", b"f00", b"f06"], 20, 8 * 14)
    assert got[0] == (fail_st, full[:8]) and got[1] == got[0]
    assert got[2] == (INCOMPLETE, full[6:14])
    rev = eng.multi_scan_reverse_at([se], [b"f10"], 20, 8 * 14)[0]
    assert rev == (fail_st, full[10::-1][:8])
    # the device form: the failed merge's record carries 0xfffffffe (decoded as the marker's length) and the status has
    # bit 30 when the scan also ran out of room
    out, n_out, st = device_scan(eng, [se.slot], [b"f00"], 3, None, 20, 8 * 14, False, False, decode=False)
    assert n_out[0] == 8 and st[0] & (1 << 30) and (int(st[0]) & ~(1 << 30)) >> 8 == fail_st
    assert struct.unpack_from("<II", out, 5 * 14) == (3, 0xfffffffe)  # f05: key only, no value bytes
    se.release()
    so.release()
    db.close()
    s.close()


# ---- 10. the device forms on a caller's stream equal the host forms ---------------------------------------------------
def test_device_forms_equal_host_forms(eng, fixed_snap):
    s, snap, rows = fixed_snap
    g = new_shard(eng, okv.MERGE_UINT64ADD)
    rng = random.Random(4)
    gkeys = [b"d%05d" % i for i in range(0, 900, 3)]
    for _ in range(3):
        general_stream(g, None, rng, gkeys, 200)
        assert g.flush() == 0
    general_stream(g, None, rng, gkeys, 50)
    gs = g.snapshot()
    keys = [k for k, _ in rows]
    n = 300
    pick = [(snap, rng.choice(keys), rng.choice(keys)) if i % 2 else
            (gs, rng.choice(gkeys) + b"000000000", rng.choice(gkeys) + b"0" * 9 + b"\xff" * 2) for i in range(n)]
    # fixed-length keys on the device: 16 bytes each (the general shard's keys are padded to 16)
    sk = [k[:16].ljust(16, b"\0") for _, k, _ in pick]
    ek = [k[:16].ljust(16, b"\0") for _, _, k in pick]
    for rev in (False, True):
        for x in (False, True):
            for caller in (True, False):
                dev = device_scan(eng, [p[0].slot for p in pick], sk, 16, ek, 40, 40 * 88, rev, x, caller)
                fn = eng.multi_scan_reverse_at if rev else eng.multi_scan_at
                kw = {"lows" if rev else "ends": ek}
                host = fn([p[0] for p in pick], sk, 40, 40 * 88, exclusive=x, **kw)
                assert dev == host, (rev, x, caller)
    # from either end (keys NULL)
    for rev in (False, True):
        dev = device_scan(eng, [snap.slot, gs.slot], None, 0, None, 5, 5 * 88, rev, False)
        host = (eng.multi_scan_reverse_at if rev else eng.multi_scan_at)([snap, gs], None, 5, 5 * 88)
        assert dev == host and len(dev[0][1]) == 5
    gs.release()
    g.close()


# ---- 11. batched scans equal the snapshot's iterator walks over 1-8 runs -------------------------------------------------
@pytest.mark.parametrize("n_runs", [1, 3, 8])
def test_batched_scans_equal_iterator_walks(eng, n_runs):
    s = new_shard(eng, okv.MERGE_UINT64ADD)
    rng = random.Random(30 + n_runs)
    keys = [b"w%0*d" % (rng.choice((2, 5)), i) for i in range(0, 300, 3)]
    for rnd in range(n_runs):
        general_stream(s, None, rng, keys, 100)
        if rnd < n_runs - 1:
            assert s.flush() == 0
    snap = s.snapshot()
    general_stream(s, None, rng, keys, 100)
    probes = sorted(set(keys)) + [b"w", b"x", b""]
    ws = [(rng.choice("fr"), None if rng.random() < 0.1 else rng.choice(probes), rng.randrange(2),
           None if rng.random() < 0.3 else rng.choice(probes), rng.choice((1, 5, 400))) for _ in range(60)]
    res = scan_at(eng, list(enumerate(ws)), [snap] * len(ws))
    for (i, w), got in res.items():
        assert got == SS.expected_scan(SS.run_walk(lambda ub: snap.iterator(upper_bound=ub), w)), w
    snap.release()
    s.close()
