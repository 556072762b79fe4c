"""GPU: files ingested behind a shard's data (rsp_shard_open_ex with RSP_SHARD_ALLOW_INGEST_BEHIND,
rsp_ingest_sorted_behind, rsp_compact_ex) and the device-built runs of both ingest forms.

The model is RocksDB's own equivalence for visible contents: ingesting a file F behind a history H answers like
ingesting F into an empty DB first (which leaves the sequence number at 0) and then replaying H.  Here that DB is the
oracle port with every behind file applied first as Puts; the engine's sequence number is the port's less those Puts.
Every check reads through rsp_get, the generic and the 16-byte-key MultiGet (host and device forms), forward, bounded
and reverse batched scans, the device scan and the iterator; snapshots taken after an ingest are read at the end.
Refusals are checked for their code, their text and for leaving the shard as it was.
"""
import os
import random
import struct

import numpy as np
import pytest

import ingest_behind_oracle as IB
import string_append_model as SA
from oracle import okv
from rocksplicator_b200 import engine as E
from rocksplicator_b200.write_batch import WriteBatch

pytestmark = pytest.mark.gpu
EMUL = bool(os.environ.get("RSP_TEST_EMUL_LIB"))
if not EMUL:
    import torch

OK, NOT_FOUND, NOT_SUPPORTED, INVALID = 0, 1, 3, 4
NO_OPTION = "can't ingest_behind file in DB with allow_ingest_behind=false"
NO_FIT = "Can't ingest_behind file as it doesn't fit at the bottommost level!"
SEQ0_ABOVE = "Can't ingest_behind file as despite allow_ingest_behind=true there are files with 0 seqno in database at upper levels!"
STRIDE = 1 << 15
# merge operators: the three the oracle port folds, and RocksDB's StringAppendOperator with a ',' delimiter and without
# one, modelled by tests/string_append_model.py
SA_COMMA, SA_NONE = "sa_comma", "sa_none"
OPS = [okv.MERGE_NONE, okv.MERGE_COUNTER, okv.MERGE_UINT64ADD, SA_COMMA, SA_NONE]
SA_DELIM = {SA_COMMA: b",", SA_NONE: None}


@pytest.fixture(scope="module")
def engines():
    es = {t: E.Engine(0, l0_compaction_trigger=t) for t in (2, 4)}
    yield es
    for e in es.values():
        e.close()


_n = [0]


def key(i):
    return b"k%015d" % i  # 16 bytes: the 16-byte-key MultiGet serves them


def val(op, rnd, n=None):
    if op in (okv.MERGE_COUNTER, okv.MERGE_UINT64ADD):
        return struct.pack("<q", rnd.randrange(-1000, 1000))
    return rnd.randbytes(rnd.randrange(0, 40) if n is None else n)


class Pair:
    """an engine shard and its model: the port with the files ingested behind applied first, then the history"""

    def __init__(self, e, merge_op=okv.MERGE_NONE, allow=True, write_buffer_bytes=0):
        _n[0] += 1
        self.e = e
        self.op = merge_op
        kw = {"merge_op": merge_op}
        if merge_op in SA_DELIM:
            kw = {"merge_op": E.MERGE_STRING_APPEND, "merge_delim": SA_DELIM[merge_op]}
        self.s = e.open_shard("behind%05d" % _n[0], allow_ingest_behind=allow, write_buffer_bytes=write_buffer_bytes,
                              **kw)
        self.files, self.hist, self.snaps = [], [], []

    def apply(self, batches):
        if batches:
            st = self.e.apply_many([self.s.index] * len(batches), batches, [7] * len(batches))
            assert not st.any(), st
            self.hist += batches

    def behind(self, kvs):
        rc = self.s.ingest(kvs, behind=True)
        if rc == OK:
            self.files.append(list(kvs))
        return rc

    def model(self):
        o = StringAppendSide(SA_DELIM[self.op]) if self.op in SA_DELIM else okv.Okv(okv.load_port(), merge_op=self.op)
        for f in self.files:
            wb = WriteBatch()
            for k, v in f:
                wb.put(k, v)
            assert o.apply(wb.data(), 0) == 0
        for b in self.hist:
            assert o.apply(b, 7) == 0
        return o, sum(len(f) for f in self.files)

    def close(self):
        for sn, _ in self.snaps:
            sn.release()
        self.s.close()


def parse_batch(data):
    """WriteBatch bytes -> [(kind, key, value)] of tests/string_append_model.py"""
    def varint(at):
        v, sh = 0, 0
        while True:
            b = data[at]
            at += 1
            v |= (b & 0x7F) << sh
            if b < 0x80:
                return v, at
            sh += 7

    def lp(at):
        n, at = varint(at)
        return data[at:at + n], at + n
    ops, at = [], 12
    while at < len(data):
        tag = data[at]
        k, at = lp(at + 1)
        if tag in (0x1, 0x2):
            v, at = lp(at)
            ops.append((SA.PUT if tag == 0x1 else SA.MERGE, k, v))
        elif tag in (0x0, 0x7):
            ops.append((SA.DEL if tag == 0x0 else SA.SDEL, k, None))
        else:
            raise ValueError("tag %d" % tag)
    return ops


class StringAppendSide:
    """tests/string_append_model.py behind the oracle's interface (apply / latest_seq / multi_get / scan)"""

    def __init__(self, delim):
        self.m = SA.Model(delim)

    def apply(self, batch, ts_ms=0):
        self.m.apply(parse_batch(batch))
        return 0

    def latest_seq(self):
        return self.m.seq

    def multi_get(self, keys):
        return [(OK, v) if v is not None else (NOT_FOUND, None) for v in (self.m.get(k) for k in keys)]

    def scan(self):
        return self.m.items()

    def close(self):
        pass


# ---- the read paths -------------------------------------------------------------------------------------------
def _dev(arrays):
    if EMUL:
        return [np.ascontiguousarray(a).copy() for a in arrays]
    t = [torch.from_numpy(np.ascontiguousarray(a).copy()).cuda() for a in arrays]
    torch.cuda.synchronize()
    return t


def _ptr(a):
    return a.ctypes.data if EMUL else a.data_ptr()


def _host(arrays):
    if EMUL:
        return arrays
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in arrays]


def fixed_gets(p, keys, device):
    """the 16-byte-key MultiGet: rsp_multi_get_fixed (host form) or rsp_multi_get_device"""
    e, n, stride = p.e, len(keys), 256
    if not device:
        vals = np.zeros(n * stride, dtype=np.uint8)
        vlen = np.zeros(n, dtype=np.uint32)
        st = np.full(n, -1, dtype=np.int32)
        kb = np.frombuffer(b"".join(keys), dtype=np.uint8).copy()
        assert e.multi_get_fixed(np.full(n, p.s.index, dtype=np.uint32), kb, 16, vals, stride, vlen, st) == OK
    else:
        d = _dev([np.full(n, p.s.index, dtype=np.uint32), np.frombuffer(b"".join(keys), dtype=np.uint8),
                  np.zeros(n * stride, dtype=np.uint8), np.zeros(n, dtype=np.uint32), np.full(n, -1, dtype=np.int32)])
        pp = [_ptr(a) for a in d]
        assert e.lib.rsp_multi_get_device(e.h, n, pp[0], pp[1], 16, pp[2], stride, pp[3], pp[4], None) == OK
        _, _, vals, vlen, st = _host(d)
    return [(int(st[i]), vals[i * stride:i * stride + int(vlen[i])].tobytes() if st[i] == OK else None)
            for i in range(n)]


def device_scans(p, starts, limit):
    """rsp_multi_scan_device (the sorted runs only: the caller flushed)"""
    e, n = p.e, len(starts)
    d = _dev([np.full(n, p.s.index, dtype=np.uint32), np.frombuffer(b"".join(starts), dtype=np.uint8),
              np.zeros(n * STRIDE, dtype=np.uint8), np.zeros(n, dtype=np.uint32), np.full(n, -1, dtype=np.int32)])
    pp = [_ptr(a) for a in d]
    assert e.lib.rsp_multi_scan_device(e.h, n, pp[0], pp[1], 16, limit, pp[2], STRIDE, pp[3], pp[4], None) == OK
    _, _, out, n_out, st = _host(d)
    return E._scan_records(out, n_out, st, n, STRIDE)


def probes(live, rnd, extra=()):
    keys = sorted({k for k, _ in live} | set(extra))
    pick = rnd.sample(keys, min(len(keys), 48)) if keys else []
    return pick + [b"k%015d" % rnd.randrange(0, 10 ** 6) for _ in range(8)] + [b"a" * 16, b"z" * 16]


def check(p, rnd, extra=(), point_only=False):
    """every read path of the shard against the model; snapshots taken earlier against what they saw then"""
    o, nf = p.model()
    try:
        assert p.s.latest_seq() == o.latest_seq() - nf
        live = [] if point_only else o.scan()
        keys = probes(live or [(k, None) for k in extra], rnd, extra)
        want = o.multi_get(keys)
        assert p.s.multi_get(keys) == want
        assert [p.s.get(k) for k in keys[:12]] == want[:12]
        assert fixed_gets(p, keys, device=False) == want
        assert fixed_gets(p, keys, device=True) == want
        if point_only:
            return
        assert p.s.scan() == live
        lim = 24
        starts = [k for k, _ in rnd.sample(live, min(4, len(live)))] + [b"a" * 16, key(rnd.randrange(0, 400))]
        ends = [key(int(s[1:]) + rnd.randrange(1, 60)) if s[:1] == b"k" else b"k%015d" % 50 for s in starts]
        six = [p.s.index] * len(starts)
        assert p.e.multi_scan(six, starts, lim, STRIDE) == \
            [(OK, [kv for kv in live if kv[0] >= s][:lim]) for s in starts]
        assert p.e.multi_scan(six, starts, lim, STRIDE, ends=ends) == \
            [(OK, [kv for kv in live if s <= kv[0] < t][:lim]) for s, t in zip(starts, ends)]
        lows = [b"a" * 16] + [key(max(0, int(t[1:]) - 80)) for t in ends[1:]]
        assert p.e.multi_scan_reverse(six, ends, lim, STRIDE, lows=lows) == \
            [(OK, [kv for kv in reversed(live) if lo <= kv[0] <= t][:lim]) for t, lo in zip(ends, lows)]
        it = p.s.iterator(upper_bound=ends[0])
        it.seek_for_prev(starts[0])
        walk = []
        while it.valid() and len(walk) < 30:
            walk.append((it.key(), it.value()))
            it.prev()
        it.close()
        assert walk == [kv for kv in reversed(live) if kv[0] <= starts[0]][:30]
        assert p.s.flush() == OK
        assert device_scans(p, starts, lim) == [(OK, [kv for kv in live if kv[0] >= s][:lim]) for s in starts]
        for sn, (skeys, sget, sall) in p.snaps:
            assert p.e.multi_get_at([sn] * len(skeys), skeys) == sget
            assert p.e.multi_scan_at([sn], None, 1000, STRIDE) == [(OK, sall[:1000])]
    finally:
        o.close()


def take_snapshot(p, rnd):
    o, _ = p.model()
    try:
        live = o.scan()
        keys = probes(live, rnd)
        p.snaps.append((p.s.snapshot(), (keys, o.multi_get(keys), live)))
    finally:
        o.close()


def shape(p):
    st = p.s.stats()
    return {k: st[k] for k in ("latest_seq", "memtable_entries", "n_runs", "run_entries", "run_bytes")}, \
        p.s.behind_bytes(), p.s.scan()


def kv_file(rnd, lo, hi, op, n=None, step=1):
    ks = list(range(lo, hi, step))
    if n is not None:
        ks = sorted(rnd.sample(ks, min(n, len(ks))))
    return [(key(i), val(op, rnd)) for i in ks]


def puts(rnd, ks, op):
    return [WriteBatch().put(key(i), val(op, rnd)).data() for i in ks]


# ---- refusals ----------------------------------------------------------------------------------------------------
def test_refusals_leave_the_shard_unchanged(engines):
    e = engines[4]
    rnd = random.Random(1)
    plain = Pair(e, allow=False)
    plain.apply(puts(rnd, range(0, 40), okv.MERGE_NONE))
    before = shape(plain)
    assert plain.s.ingest(kv_file(rnd, 100, 120, 0), behind=True) == INVALID
    assert plain.s.last_error == "Invalid argument: " + NO_OPTION
    assert shape(plain) == before and before[1] == 0
    plain.close()

    p = Pair(e)
    p.apply(puts(rnd, range(0, 40), okv.MERGE_NONE))
    assert p.behind(kv_file(rnd, 100, 200, 0, step=3)) == OK
    check(p, rnd)
    before = shape(p)
    assert before[1] > 0
    for lo, hi in ((150, 160), (199, 230), (40, 101), (0, 1000)):  # inside, over either end, around
        assert p.behind(kv_file(rnd, lo, hi, 0)) == INVALID
        assert p.s.last_error == "Invalid argument: " + NO_FIT
        assert shape(p) == before
    assert p.behind([(key(5), b"x"), (key(3), b"y")]) == INVALID
    assert p.s.last_error == "Invalid argument: Keys must be added in order"
    assert p.behind(kv_file(rnd, 300, 310, 0)) == OK  # disjoint from the first file: fits
    check(p, rnd)

    sn = p.s.snapshot()
    before = shape(p)
    assert p.behind(kv_file(rnd, 400, 410, 0)) == NOT_SUPPORTED
    assert shape(p) == before
    sn.release()
    assert p.behind(kv_file(rnd, 400, 410, 0)) == OK
    check(p, rnd)

    # a normal ingest that takes no global sequence number leaves sequence-0 data above the tier
    norm = kv_file(rnd, 500, 520, 0)
    assert p.s.ingest(norm) == OK
    p.files.append(norm)  # (same visible contents: it overlaps nothing and takes no sequence number)
    before = shape(p)
    for how in ("refused", "compact", "compact_level"):
        if how == "compact":
            assert p.s.compact() == OK
        elif how == "compact_level":
            assert p.s.compact(change_level=True) == OK
            assert p.s.behind_bytes() == 0 and p.s.stats()["n_runs"] == 1
        assert p.behind(kv_file(rnd, 600, 610, 0)) == INVALID
        assert p.s.last_error == "Invalid argument: " + SEQ0_ABOVE
        check(p, rnd)
    p.close()

    # an overlapping normal ingest takes a global sequence number: no sequence-0 data, the tier stays open
    q = Pair(e)
    q.apply(puts(rnd, range(0, 40), okv.MERGE_NONE))
    assert q.s.flush() == OK
    ov = kv_file(rnd, 30, 50, 0)
    seq = q.s.latest_seq()
    assert q.s.ingest(ov) == OK and q.s.latest_seq() == seq + 1
    assert q.s.ingest(kv_file(rnd, 60, 90, 0), behind=True) == OK
    assert q.s.latest_seq() == seq + 1
    q.close()


# ---- the tier through flushes and compactions ------------------------------------------------------------------
@pytest.mark.parametrize("op", OPS)
def test_history_then_behind(engines, op):
    """Puts, deletes and merges written, flushed and compacted before the file; a merge whose base arrives behind
    later; a delete compacted away before the behind value of its key arrives (NotFound stays)"""
    e = engines[4]
    rnd = random.Random(10 + OPS.index(op))
    p = Pair(e, merge_op=op)
    p.apply(puts(rnd, range(0, 200, 2), op))
    p.apply([WriteBatch().delete(key(i)).data() for i in range(0, 200, 10)])
    p.apply([WriteBatch().single_delete(key(i)).data() for i in range(1000, 1010)])
    if op != okv.MERGE_NONE:
        p.apply([WriteBatch().merge(key(i), val(op, rnd)).data() for i in range(0, 200, 3)])
        p.apply([WriteBatch().merge(key(i), val(op, rnd)).data() for i in range(0, 60, 3)])
    assert p.s.flush() == OK
    p.apply([WriteBatch().delete(key(i)).data() for i in range(201, 260, 4)])
    assert p.s.compact() == OK
    take_snapshot(p, rnd)
    check(p, rnd)
    for sn, _ in p.snaps:
        sn.release()
    p.snaps = []
    assert p.behind(kv_file(rnd, 0, 300, op)) == OK  # under every key written so far
    check(p, rnd)
    take_snapshot(p, rnd)
    p.apply(puts(rnd, range(100, 140, 3), op))
    if op != okv.MERGE_NONE:
        p.apply([WriteBatch().merge(key(i), val(op, rnd)).data() for i in range(3000, 3010)])
    check(p, rnd)
    for sn, _ in p.snaps:
        sn.release()
    p.snaps = []
    assert p.behind(kv_file(rnd, 3000, 3020, op)) == OK  # the bases of those merges arrive behind them
    check(p, rnd)
    assert p.s.compact() == OK and p.s.behind_bytes() > 0
    check(p, rnd)
    assert p.s.compact(change_level=True) == OK and p.s.behind_bytes() == 0
    check(p, rnd)
    p.close()


def test_failing_counter_merge_over_behind_base(engines):
    rnd = random.Random(3)
    p = Pair(engines[4], merge_op=okv.MERGE_COUNTER)
    p.apply([WriteBatch().merge(key(i), struct.pack("<q", i)).data() for i in range(0, 20)])
    p.apply([WriteBatch().merge(key(7), b"abc").data()])  # a bad operand
    assert p.s.flush() == OK and p.s.compact() == OK
    assert p.behind([(key(i), b"xyz" if i % 4 == 0 else struct.pack("<q", 100 * i)) for i in range(0, 20)]) == OK
    check(p, rnd, extra=[key(i) for i in range(0, 20)], point_only=True)
    p.apply([WriteBatch().merge(key(i), struct.pack("<q", 1)).data() for i in range(0, 20, 3)])
    check(p, rnd, extra=[key(i) for i in range(0, 20)], point_only=True)
    p.close()


def test_iterator_before_ingest_keeps_its_view(engines):
    rnd = random.Random(4)
    p = Pair(engines[4])
    p.apply(puts(rnd, range(0, 100, 2), okv.MERGE_NONE))
    o, _ = p.model()
    before = o.scan()
    o.close()
    it = p.s.iterator()
    assert p.behind(kv_file(rnd, 1, 100, 0, step=2)) == OK
    it.seek_to_first()
    walk = []
    while it.valid():
        walk.append((it.key(), it.value()))
        it.next()
    it.close()
    assert walk == before
    check(p, rnd)
    p.close()


def test_stats_and_behind_bytes_follow_the_tier(engines):
    rnd = random.Random(5)
    p = Pair(engines[4])
    p.apply(puts(rnd, range(0, 50), okv.MERGE_NONE))
    assert p.s.flush() == OK
    st0 = p.s.stats()
    assert st0["n_runs"] == 1 and p.s.behind_bytes() == 0
    f = kv_file(rnd, 1000, 1500, 0)
    assert p.behind(f) == OK
    st1 = p.s.stats()
    assert st1["n_runs"] == 2 and st1["run_entries"] == st0["run_entries"] + len(f)
    bb = p.s.behind_bytes()
    assert bb == st1["run_bytes"] - st0["run_bytes"] and bb >= len(f) * 48
    p.apply(puts(rnd, range(1000, 1100, 7), okv.MERGE_NONE))
    assert p.s.flush() == OK and p.s.compact() == OK  # the tier is not an input
    st2 = p.s.stats()
    assert p.s.behind_bytes() == bb and st2["n_runs"] == 2
    check(p, rnd)
    # more behind files than the run table holds: the tier's runs merge with each other
    for i in range(10):
        assert p.behind(kv_file(rnd, 2000 + 100 * i, 2050 + 100 * i, 0)) == OK
        st = p.s.stats()
        assert st["n_runs"] <= 8 and p.s.behind_bytes() > bb
    check(p, rnd)
    assert p.s.compact(change_level=True) == OK
    st3 = p.s.stats()
    assert p.s.behind_bytes() == 0 and st3["n_runs"] == 1
    check(p, rnd)
    p.close()


# ---- the builder at its size boundaries, both forms -----------------------------------------------------------
@pytest.mark.parametrize("n", [1, 31, 32, 33, 1023, 1025, 2047, 2048, 2049, 4097, 65535, 65537])
def test_builder_sizes(engines, n):
    rnd = random.Random(n)
    small = n < 5000
    for behind in (False, True):
        p = Pair(engines[4])
        kv = [(key(i), rnd.randbytes(rnd.choice([0, 1, 15, 16, 17, 64, 200]) if small else 8)) for i in range(n)]
        if behind:
            assert p.behind(kv) == OK
        else:
            assert p.s.ingest(kv) == OK
            p.files.append(kv)
        assert p.s.stats()["run_entries"] == n
        if small:
            check(p, rnd)
        else:
            o, _ = p.model()
            assert p.s.scan() == o.scan()
            ks = [key(i) for i in range(0, n, 97)] + [key(n), key(n + 1)]
            assert fixed_gets(p, ks, device=False) == o.multi_get(ks)
            o.close()
        p.close()


def test_builder_beyond_one_scan_pass_and_one_staging_buffer(engines):
    """more than 1024 tiles of 2048 entries (k_ingest_scan loops) and more than two 8 MB staging halves of keys and
    values (the pinned buffer is reused after its event): the whole run read back through the iterator, both forms"""
    if EMUL:
        pytest.skip("2 M entries: the H100 run covers it; the emulation covers the smaller sizes above")
    n = (1 << 21) + 4097
    rnd = np.random.default_rng(11)
    vals = rnd.integers(0, 256, size=(n, 12), dtype=np.uint8)
    kv = [(key(i), vals[i].tobytes()) for i in range(n)]
    for behind in (False, True):
        p = Pair(engines[4])
        assert (p.s.ingest(kv, behind=True) if behind else p.s.ingest(kv)) == OK
        st = p.s.stats()
        assert st["run_entries"] == n and st["latest_seq"] == 0
        assert p.s.behind_bytes() == (st["run_bytes"] if behind else 0)
        assert p.s.scan() == kv
        p.close()


def test_builder_key_and_value_shapes(engines):
    """keys of every length around the unit and prefix sizes, values around the unit size, large values"""
    rnd = random.Random(7)
    kv = sorted({bytes([97 + i % 26]) * l + bytes([i]): rnd.randbytes(v)
                 for i, (l, v) in enumerate((l, v) for l in (0, 1, 7, 8, 9, 15, 16, 17, 31, 33, 100)
                                            for v in (0, 1, 15, 16, 17, 100, 5000))}.items())
    p = Pair(engines[4])
    assert p.s.ingest(kv) == OK
    p.files.append(kv)
    o, _ = p.model()
    assert p.s.scan() == o.scan() == kv
    ks = [k for k, _ in kv] + [b"", b"q"]
    assert p.s.multi_get(ks, stride=8192) == o.multi_get(ks)
    o.close()
    p.close()


# ---- the random differential ----------------------------------------------------------------------------------
@pytest.mark.parametrize("trigger", [2, 4])
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("seed", [0, 1])
def test_random_streams(engines, trigger, op, seed):
    rnd = random.Random(seed * 100 + OPS.index(op) * 10 + trigger)
    p = Pair(engines[trigger], merge_op=op, write_buffer_bytes=rnd.choice([0, 4096]))
    used = []  # key ranges of the behind files

    def free_range(w):
        for _ in range(20):
            lo = rnd.randrange(0, 2000)
            if all(hi < lo or lo + w <= a for a, hi in used):
                return lo
        return None

    for step in range(40):
        r = rnd.random()
        if r < 0.45:
            bs = []
            for _ in range(rnd.randrange(1, 12)):
                wb, i = WriteBatch(), rnd.randrange(0, 2000)
                c = rnd.random()
                if c < 0.5 or op == okv.MERGE_NONE and c < 0.8:
                    wb.put(key(i), val(op, rnd))
                elif c < 0.8:
                    wb.merge(key(i), val(op, rnd))
                else:
                    wb.delete(key(i))
                bs.append(wb.data())
            p.apply(bs)
        elif r < 0.6:
            assert p.s.flush() == OK
        elif r < 0.68:
            assert p.s.compact() == OK
        elif r < 0.71:
            assert p.s.compact(change_level=True) == OK
            assert p.s.behind_bytes() == 0
            break  # the tier is closed from here on (sequence-0 data above it)
        elif r < 0.85:
            w = rnd.randrange(1, 120)
            lo = free_range(w)
            if lo is None:
                continue
            f = kv_file(rnd, lo, lo + w, op, n=rnd.randrange(1, w + 1))
            assert p.behind(f) == OK, p.s.last_error
            used.append((lo, lo + w - 1))
        else:
            check(p, rnd)
    check(p, rnd)
    p.close()


# ---- the scripted cases against the reference's RocksDB (tests/golden/ingest_behind.json) ---------------------------
class EngineSide:
    def __init__(self, p):
        self.p = p

    def latest_seq(self):
        return self.p.s.latest_seq()

    def multi_get(self, keys):
        got = self.p.s.multi_get(keys)
        assert fixed_gets(self.p, keys, device=False) == got
        assert fixed_gets(self.p, keys, device=True) == got
        assert [self.p.s.get(k) for k in keys] == got
        return got

    def scan(self):
        return self.p.s.scan()

    def fwd(self, lo, hi):
        (st, recs), = self.p.e.multi_scan([self.p.s.index], [lo], 4096, 1 << 20, ends=[hi])
        assert st == OK
        return recs

    def rev(self, lo, hi):
        (st, recs), = self.p.e.multi_scan_reverse([self.p.s.index], [hi], 4096, 1 << 20, lows=[lo], exclusive=True)
        assert st == OK
        return recs


@pytest.mark.parametrize("name", sorted(IB.cases()))
def test_reference_cases(engines, name):
    """each case's writes and behind files in their own order on the engine; at every checkpoint the answers the
    reference gave with the files ingested first"""
    import golden_util as G
    op, steps, probes, seams, scans = IB.cases()[name]
    want = {r[0]: r[1:] for r in G.load("ingest_behind.json")[name]}
    p = Pair(engines[4], merge_op=IB.MERGES[op])
    for c, st in enumerate(steps):
        if st[0] == "w":
            p.apply(st[1])
        elif st[0] == "flush":
            assert p.s.flush() == OK
        elif st[0] == "compact":
            assert p.s.compact() == OK
        elif st[0] == "behind":
            assert p.behind(st[1]) == OK, p.s.last_error
        else:
            r = IB.record(EngineSide(p), probes, seams, scans)
            assert [r[0]] + [G.digest(x) for x in r[1:]] == want[c], (name, c)
    p.close()
