"""GPU: batched reverse range scans (rsp_multi_scan_reverse, rsp_multi_scan_reverse_device: SeekForPrev + Prev with an
optional inclusive low key) and the iterator's backward moves, which run on the same kernel instances, against the
reference's RocksDB binary (tests/golden/reverse_scans.json) and against the oracle port."""
import os
import random
import struct

import numpy as np
import pytest

import bounded_oracle as BO
import golden_util as G
import reverse_oracle as RO
from oracle import okv
from rocksplicator_b200.write_batch import WriteBatch

pytestmark = pytest.mark.gpu
EMUL = bool(os.environ.get("RSP_TEST_EMUL_LIB"))
if not EMUL:
    import torch
CASES = G.load("reverse_scans.json")
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
    return eng.open_shard("rev%05d" % _n[0], merge_op=merge_op)


class EngineSide:
    def __init__(self, shard):
        self.s = shard

    def apply(self, batch): return self.s.apply(batch, 0)
    def flush(self): return self.s.flush()
    def compact(self): return self.s.compact()


def apply_ops(shard, db, ops):
    for op in ops:
        wb = WriteBatch()
        if op[0] == "put":
            wb.put(op[1], op[2])
        elif op[0] == "merge":
            wb.merge(op[1], op[2])
        else:
            wb.delete(op[1])
        assert shard.apply(wb.data(), 0) == 0
        if db is not None:
            assert db.apply(wb.data(), 0) == 0


def want_rev(rows, start, exclusive, low, limit):
    """live (key, value) of sorted Put-only rows, descending from start (None: the last key), down to low (inclusive)"""
    out = [(k, v) for k, v in reversed(rows)
           if (start is None or k < start or (k == start and not exclusive)) and (low is None or k >= low)]
    return out[:limit]


def check_host_fold(got, want_recs):
    """a host-form scan over keys of a host-side operator: NotSupported, those keys as (key, None), the rest as wanted"""
    rc, recs = got
    assert rc == NOT_SUPPORTED and [k for k, _ in recs] == [k for k, _ in want_recs]
    assert any(v is None for _, v in recs)
    for (k, v), (_, w) in zip(recs, want_recs):
        assert v is None or v == w, k


# ---- 1. the fixture -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", RO.case_names())
def test_golden_reverse_scans(eng, name):
    merge, layout = name.split("-", 1)
    s = new_shard(eng, RO.MERGES[merge])
    RO.build_layout(EngineSide(s), layout)
    walks, want = RO.walks(layout), CASES[name]
    # the iterator walk (SeekForPrev / SeekToLast + Prev) before the batched form flushes the memtable
    for w in walks:
        it = s.iterator()
        assert RO.reverse_walk(it, *w) == want[RO.walk_tag(w)], w
        it.close()
    # the batched form: one call per (from the last key, exclusive, with lows, max_entries)
    groups = {}
    for w in walks:
        groups.setdefault((w[0] is None, w[1], w[2] is None, w[3]), []).append(w)
    for (from_last, x, no_low, m), ws in groups.items():
        res = eng.multi_scan_reverse([s.index] * len(ws), None if from_last else [w[0] for w in ws], m, 8192,
                                     lows=None if no_low else [w[2] for w in ws], exclusive=bool(x))
        for w, got in zip(ws, res):
            exp = RO.expected_scan(want[RO.walk_tag(w)])
            if merge == "append" and got[0] == NOT_SUPPORTED:
                check_host_fold(got, exp[1])
            else:
                assert got == exp, w
    s.close()


# ---- 2. the fast path: one compacted run of fixed-size Puts --------------------------------------------------------------
@pytest.fixture(scope="module")
def fixed_run(eng):
    s = new_shard(eng)
    rows = [(b"key-%012d" % (3 * i), bytes([i & 0xff]) * 64) for i in range(2000)]
    apply_ops(s, None, [("put", k, v) for k, v in rows])
    assert s.compact() == 0
    assert s.stats()["n_runs"] == 1
    yield s, rows
    s.close()


def test_fast_path_boundaries(eng, fixed_run):
    s, rows = fixed_run
    keys = [k for k, _ in rows]
    # block edges (32 entries per block), inside blocks, first and last entry, between keys, before and past the end
    marks = [keys[0], keys[1], keys[-1], keys[-2], b"a", b"z", b"", b"key-", b"key-00000000001"] + \
            [keys[j] for j in range(0, len(keys), 32)] + [keys[j] for j in range(31, len(keys), 32)] + \
            [keys[j] for j in range(7, len(keys), 97)] + [keys[j] + b"\0" for j in range(31, len(keys), 97)]
    rng = random.Random(1)
    starts, lows = [], []
    for m in marks:
        for lo in (keys[0], b"", rng.choice(keys), m, keys[max(0, keys.index(m) - 40)] if m in keys else b"key-0",
                   keys[(keys.index(m) // 32) * 32] if m in keys else keys[-1]):
            starts.append(m)
            lows.append(lo)
    six = [s.index] * len(starts)
    for x in (False, True):
        for max_entries in (128, 16):
            res = eng.multi_scan_reverse(six, starts, max_entries, 128 * 96, lows=lows, exclusive=x)
            for st, lo, got in zip(starts, lows, res):
                assert got == (0, want_rev(rows, st, x, lo, max_entries)), (st, lo, x, max_entries)
            res = eng.multi_scan_reverse(six, starts, max_entries, 128 * 96, exclusive=x)
            for st, got in zip(starts, res):
                assert got == (0, want_rev(rows, st, x, None, max_entries)), (st, x, max_entries)
    res = eng.multi_scan_reverse([s.index] * 3, None, 100, 128 * 96, lows=[keys[-5], keys[0], b"zz"])
    assert res == [(0, want_rev(rows, None, False, keys[-5], 100)), (0, want_rev(rows, None, False, None, 100)),
                   (0, [])]


# ---- 3. reverse equals forward reversed (the general path) ---------------------------------------------------------------
def random_stream(shard, db, seed, n_rounds):
    """random writes with a flush after every round but the last (several runs + a memtable)"""
    rng = random.Random(seed)
    keys = [b"g%0*d" % (rng.choice((2, 5, 11)), i) for i in range(0, 400, 3)]
    for rnd in range(n_rounds):
        for _ in range(150):
            k, r = rng.choice(keys), rng.random()
            if r < 0.55:
                op = ("put", k, bytes(rng.randrange(256) for _ in range(rng.randrange(0, 90))))
            elif r < 0.75:
                op = ("del", k, None)
            else:
                op = ("merge", k, struct.pack("<Q", rng.randrange(1 << 40)))
            apply_ops(shard, db, [op])
        if rnd < n_rounds - 1:
            assert shard.flush() == 0
    return sorted(set(keys))


@pytest.mark.parametrize("merge", [okv.MERGE_UINT64ADD, okv.MERGE_COUNTER, okv.MERGE_APPEND])
def test_reverse_equals_forward_reversed(eng, merge):
    s = new_shard(eng, merge)
    db = BO.BoundedOkv(BO.load_port(), merge_op=merge)
    keys = random_stream(s, db, 10 + merge, 4)
    assert s.stats()["n_runs"] >= 2
    rng = random.Random(merge)
    probes = keys + [k + b"\0" for k in keys[::5]] + [b"g", b"g1", b"g00000", b"h", b""]
    a = [rng.choice(probes) for _ in range(80)]
    b = [rng.choice(probes) for _ in range(80)]
    six = [s.index] * 80
    fwd = eng.multi_scan(six, a, 500, 64 * 1024, ends=b)
    rev = eng.multi_scan_reverse(six, b, 500, 64 * 1024, lows=a, exclusive=True)
    for lo, hi, (rc0, r0), (rc1, r1) in zip(a, b, fwd, rev):
        assert rc1 == rc0 and r1 == r0[::-1], (lo, hi)
        port = db.scan(start=lo, end=hi)
        if rc1 == NOT_SUPPORTED:
            check_host_fold((rc1, r1), port[::-1])
        else:
            assert r1 == port[::-1], (lo, hi)
    db.close()
    s.close()


# ---- 4. keys below the low, or at an excluded start, are not read -------------------------------------------------------
def test_keys_below_the_low_or_excluded_are_not_read(eng):
    from rocksplicator_b200 import engine
    rows = [(b"p%03d" % i, b"v%d" % i) for i in range(50)]
    bad = {engine.MERGE_COUNTER: lambda k: [("put", k, b"abc"), ("merge", k, struct.pack("<q", 5))],
           engine.MERGE_APPEND: lambda k: [("merge", k, b"x"), ("merge", k, b"y")]}
    for merge, tail in bad.items():
        s = new_shard(eng, merge)
        db = BO.BoundedOkv(BO.load_port(), merge_op=merge)
        apply_ops(s, db, [("put", k, v) for k, v in rows])
        assert s.flush() == 0
        # below the low: o9 (failing or host-folded) and deleted p000 .. p009; at the start: q1
        apply_ops(s, db, [("del", b"p%03d" % i, None) for i in range(10)] + tail(b"o9") + tail(b"q1"))
        live = rows[10:]
        res = eng.multi_scan_reverse([s.index] * 3, [b"q1", b"p040", b"q1"], 100, 8192,
                                     lows=[b"p", b"p000", b"p045"], exclusive=True)
        assert res == [(0, want_rev(live, b"q1", True, b"p", 100)), (0, want_rev(live, b"p040", True, b"p000", 100)),
                       (0, want_rev(live, b"q1", True, b"p045", 100))]
        full = eng.multi_scan_reverse([s.index], [b"q1"], 100, 8192)
        assert full[0][0] != 0  # inclusive and without a low, the scan reads q1 and o9 and reports them
        # the port's iterator: the walk that skips q1 and stops before o9 has the same keys and raises nothing on them
        it = db.iterator()
        walk = RO.reverse_walk(it, b"q1", 1, b"p", 100)
        it.close()
        assert [bytes.fromhex(k) for k, _, _ in walk["taken"]] == [k for k, _ in res[0][1]]
        db.close()
        s.close()


# ---- 5. limits with a low ------------------------------------------------------------------------------------------------
def test_limits_with_low(eng, fixed_run):
    s, rows = fixed_run
    keys = [k for k, _ in rows]
    # room for 5 records of 8 + 16 + 64 bytes; the low leaves 10 (INCOMPLETE) or 3 (complete)
    res = eng.multi_scan_reverse([s.index] * 2, [keys[110]] * 2, 128, 5 * 88, lows=[keys[101], keys[108]])
    assert res[0] == (INCOMPLETE, want_rev(rows, keys[110], False, keys[106], 128))
    assert res[1] == (0, want_rev(rows, keys[110], False, keys[108], 128))
    res = eng.multi_scan_reverse([s.index], [keys[110]], 4, 5 * 88, lows=[keys[101]])
    assert res[0] == (0, want_rev(rows, keys[110], False, keys[101], 4))
    # the general path: a second run
    s2 = new_shard(eng)
    apply_ops(s2, None, [("put", k, v) for k, v in rows[:300:2]])
    assert s2.flush() == 0
    apply_ops(s2, None, [("put", k, v) for k, v in rows[1:300:2]])
    res = eng.multi_scan_reverse([s2.index] * 3, [keys[110]] * 3, 128, 5 * 88, lows=[keys[101], keys[108], keys[90]])
    assert res[0] == (INCOMPLETE, want_rev(rows, keys[110], False, keys[106], 128))
    assert res[1] == (0, want_rev(rows, keys[110], False, keys[108], 128))
    res = eng.multi_scan_reverse([s2.index], [keys[110]], 7, 100 * 88, lows=[keys[90]])
    assert res[0] == (0, want_rev(rows, keys[110], False, keys[90], 7))
    s2.close()


def to_dev(arrays):
    """device copies of host arrays (under the emulation: host copies)"""
    if EMUL:
        return [a.copy() for a in arrays]
    d = [torch.from_numpy(a.copy()).cuda() for a in arrays]
    torch.cuda.synchronize()
    return d


def ptrs(d): return [a.ctypes.data if EMUL else a.data_ptr() for a in d]
def to_host(d): return d if EMUL else [t.cpu().numpy() for t in d]


# ---- 6. the device form on a caller's stream -----------------------------------------------------------------------------
def test_device_form_on_caller_stream(eng):
    s = new_shard(eng)
    rows = [(b"dev-%012d" % (3 * i), bytes([i & 0xff]) * 64) for i in range(3000)]
    apply_ops(s, None, [("put", k, v) for k, v in rows])
    assert s.compact() == 0
    keys = [k for k, _ in rows]
    rng = random.Random(3)
    n, max_entries, stride = 512, 64, 64 * 88
    st_i = [rng.randrange(len(keys)) for _ in range(n)]
    lo_i = [max(0, i - rng.randrange(-5, 100)) for i in st_i]
    six = np.full(n, s.index, dtype=np.uint32)
    kq = np.frombuffer(b"".join(keys[i] for i in st_i), dtype=np.uint8)
    kl = np.frombuffer(b"".join(keys[i] for i in lo_i), dtype=np.uint8)
    d = to_dev([six, kq, kl, np.zeros(n * stride, np.uint8), np.zeros(n, np.uint32), np.full(n, -1, np.int32)])
    stream = eng.lib.rsp_engine_stream(eng.h) if EMUL else torch.cuda.Stream()
    p = ptrs(d)
    assert eng.lib.rsp_multi_scan_reverse_device(eng.h, n, p[0], p[1], 16, 1, p[2], 16, max_entries, p[3], stride, p[4],
                                                 p[5], stream if EMUL else stream.cuda_stream) == 0
    # issued after the scan: it waits for the scan, which reads the runs as they were
    apply_ops(s, None, [("del", k, None) for k in keys[::2]])
    assert s.compact() == 0
    if not EMUL:
        stream.synchronize()
    out, n_out, st = to_host(d[3:])
    for q in range(n):
        want = want_rev(rows, keys[st_i[q]], True, keys[lo_i[q]], max_entries)
        assert st[q] == 0 and n_out[q] == len(want), q
        at = q * stride
        for k, v in want:
            klen, vlen = struct.unpack_from("<II", out, at)
            assert (out[at + 8:at + 8 + klen].tobytes(), out[at + 8 + klen:at + 8 + klen + vlen].tobytes()) == (k, v)
            at += 8 + klen + vlen
    # from the last key (d_keys == NULL), no low, on the engine's stream, after the deletes
    d = to_dev([six[:2], np.zeros(2 * stride, np.uint8), np.zeros(2, np.uint32), np.full(2, -1, np.int32)])
    p = ptrs(d)
    assert eng.lib.rsp_multi_scan_reverse_device(eng.h, 2, p[0], None, 0, 0, None, 0, 3, p[1], stride, p[2], p[3],
                                                 None) == 0
    if not EMUL:
        torch.cuda.synchronize()
    out, n_out, st = to_host(d[1:])
    assert list(n_out) == [3, 3] and list(st) == [0, 0]
    assert out[8:8 + 16].tobytes() == keys[-1]  # (odd positions survive the deletes; 2999 is one)


# ---- 7. iterator parity over 1-8 runs and a memtable ---------------------------------------------------------------------
@pytest.mark.parametrize("n_runs", [1, 3, 8])
def test_iterator_prev_walks_match_port(eng, n_runs):
    s = new_shard(eng, okv.MERGE_COUNTER)
    db = BO.BoundedOkv(BO.load_port(), merge_op=okv.MERGE_COUNTER)
    keys = random_stream(s, db, 40 + n_runs, n_runs + 1)
    # a failing counter merge: an operand on a 3-byte value, in the memtable
    apply_ops(s, db, [("put", keys[20], b"abc"), ("merge", keys[20], struct.pack("<q", 5))])
    assert s.stats()["memtable_entries"] > 0
    snap_e, snap_o = s.snapshot(), db.snapshot()
    apply_ops(s, db, [("put", keys[3], b"late"), ("del", keys[30], None), ("put", keys[-1], b"late2")])
    rng = random.Random(n_runs)
    probes = keys + [k + b"\0" for k in keys[::7]] + [b"g", b"h", b""]
    for i in range(30):
        at = i % 2 == 1
        start = None if i % 5 == 0 else rng.choice(probes)
        x = rng.randrange(2)
        ie = (snap_e if at else s).iterator()
        io = db.iterator(snap_o if at else None)
        assert RO.reverse_walk(ie, start, x, None, 400) == RO.reverse_walk(io, start, x, None, 400), (i, start, x, at)
        ie.close()
        io.close()
    snap_e.release()
    snap_o.release()
    db.close()
    s.close()
