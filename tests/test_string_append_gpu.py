"""GPU: RSP_MERGE_STRING_APPEND (RocksDB's StringAppendOperator, folded on the device) against what the reference's RocksDB
binary answered on the recorded streams of tests/golden/string_append.json, and against the port of
tests/string_append_model.py (checked against the same recordings by tests/test_string_append_oracle_cpu.py) on every
read path: Get, MultiGet (host forms, the fixed-key form and the device form),
forward / bounded / reverse batched scans (host and device forms), iterators, and reads at snapshots.  Each is read with
the data in the memtable, after a flush, after merges of runs and after a full compaction."""
import os
import random

import numpy as np
import pytest

import string_append_model as SA
import string_append_oracle as O
from string_append_model import DEL, MERGE, PUT, SDEL

pytestmark = pytest.mark.gpu
EMUL = bool(os.environ.get("RSP_TEST_EMUL_LIB"))
if not EMUL:
    import torch
OK, NOT_FOUND, INVALID, INCOMPLETE = 0, 1, 4, 7
DELIMS = [b",", None, b"\0"]


@pytest.fixture(scope="module")
def eng():
    from rocksplicator_b200 import engine
    e = engine.Engine(0, l0_compaction_trigger=3)  # merges of runs happen while the streams run
    yield e
    e.close()


_n = [0]


def new_shard(eng, delim, merge_op=None):
    from rocksplicator_b200 import engine
    _n[0] += 1
    return eng.open_shard("sapp%05d" % _n[0], merge_op=engine.MERGE_STRING_APPEND if merge_op is None else merge_op,
                          merge_delim=delim)


def key(i):
    return b"key-%012d" % i  # 16 bytes: every MultiGet form and the device forms take them


def apply(shard, model, ops):
    assert shard.apply(SA.batch_of(ops), 0) == 0
    model.apply(ops)


def to_dev(arrays):
    """device copies of host arrays (under the emulation: host copies)"""
    if EMUL:
        return [a.copy() for a in arrays]
    d = [torch.from_numpy(a.copy()).cuda() for a in arrays]
    torch.cuda.synchronize()
    return d


def ptrs(d): return [a.ctypes.data if EMUL else a.data_ptr() for a in d]


def to_host(d):
    if EMUL:
        return d
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in d]


def multi_get_device(eng, six, keys, stride):
    n = len(keys)
    d = to_dev([np.full(n, six, np.uint32), np.frombuffer(b"".join(keys), np.uint8).copy(), np.zeros(n * stride, np.uint8),
                np.zeros(n, np.uint32), np.full(n, -1, np.int32)])
    p = ptrs(d)
    assert eng.lib.rsp_multi_get_device(eng.h, n, p[0], p[1], 16, p[2], stride, p[3], p[4], None) == 0
    vals, vlen, st = to_host(d[2:])
    return [(int(st[i]), vals[i * stride:i * stride + vlen[i]].tobytes() if st[i] == OK else int(vlen[i]))
            for i in range(n)]


def scan_device(eng, six, starts, max_entries, stride, ends=None, reverse=False, exclusive=False):
    from rocksplicator_b200.engine import _scan_records
    n = len(starts)
    arrs = [np.full(n, six, np.uint32), np.frombuffer(b"".join(starts), np.uint8).copy(),
            np.frombuffer(b"".join(ends), np.uint8).copy() if ends else np.zeros(1, np.uint8),
            np.zeros(n * stride, np.uint8), np.zeros(n, np.uint32), np.full(n, -1, np.int32)]
    d = to_dev(arrs)
    p = ptrs(d)
    if reverse:
        rc = eng.lib.rsp_multi_scan_reverse_device(eng.h, n, p[0], p[1], 16, 1 if exclusive else 0,
                                                   p[2] if ends else None, 16 if ends else 0, max_entries, p[3],
                                                   stride, p[4], p[5], None)
    elif ends:
        rc = eng.lib.rsp_multi_scan_bounded_device(eng.h, n, p[0], p[1], 16, p[2], 16, max_entries, p[3], stride, p[4],
                                                   p[5], None)
    else:
        rc = eng.lib.rsp_multi_scan_device(eng.h, n, p[0], p[1], 16, max_entries, p[3], stride, p[4], p[5], None)
    assert rc == 0
    out, n_out, st = to_host(d[3:])
    return _scan_records(out, n_out, st, n, stride)


def iter_walk(it, model_items, rng, upper=None):
    """Seek / SeekForPrev / SeekToFirst / SeekToLast, then Next or Prev: every position against the model"""
    keys = [k for k, _ in model_items]
    vals = dict(model_items)
    bounded = [k for k in keys if upper is None or k < upper]
    for _ in range(6):
        m = rng.randrange(4)
        t = key(rng.randrange(-2, 70))
        if m == 0:
            it.seek(t)
            want = [k for k in bounded if k >= t]
        elif m == 1:
            it.seek_for_prev(t)
            want = [k for k in reversed(keys) if k <= t]
        elif m == 2:
            it.seek_to_first()
            want = bounded
        else:
            it.seek_to_last()
            want = list(reversed(bounded))
        fwd = m in (0, 2)
        for w in want[:4]:
            assert it.valid() and it.key() == w and it.value() == vals[w], (m, t, w)
            it.next() if fwd else it.prev()
        if len(want) <= 4:
            assert not it.valid()
        assert it.status() == 0


def check_reads(eng, shard, model, rng, snaps=(), device=True):
    """every read path against the model; device: the memtable is empty, so the runs-only device forms see it all"""
    keys = [key(i) for i in range(-1, 66)]
    want = {k: model.get(k) for k in keys}
    for k in keys[::5]:
        rc, v = shard.get(k, cap=4)
        assert (rc, v) == ((OK, want[k]) if want[k] is not None else (NOT_FOUND, None)), k
    got = shard.multi_get(keys, stride=8)  # (the binding grows the stride on INCOMPLETE)
    assert got == [(OK, want[k]) if want[k] is not None else (NOT_FOUND, None) for k in keys]
    stride = max([len(v) for v in want.values() if v is not None] + [16])
    stride = (stride + 15) & ~15
    n = len(keys)
    vals = np.zeros(n * stride, np.uint8)
    vlen = np.zeros(n, np.uint32)
    st = np.full(n, -1, np.int32)
    assert eng.multi_get_fixed(np.full(n, shard.index, np.uint32), np.frombuffer(b"".join(keys), np.uint8), 16, vals,
                               stride, vlen, st) == 0
    for i, k in enumerate(keys):
        if want[k] is None:
            assert st[i] == NOT_FOUND
        else:
            assert st[i] == OK and vals[i * stride:i * stride + vlen[i]].tobytes() == want[k]
    dev = multi_get_device(eng, shard.index, keys, stride)
    assert all(s != 100 for s, _ in dev)
    assert dev == [(OK, want[k]) if want[k] is not None else (NOT_FOUND, 0) for k in keys]
    # batched scans, host forms
    starts = [key(rng.randrange(-1, 66)) for _ in range(6)]
    ends = [key(rng.randrange(-1, 66)) for _ in range(6)]
    m = 9
    sstride = 8 * m + 16 * m + m * stride + 64
    six = [shard.index] * len(starts)
    assert eng.multi_scan(six, starts, m, sstride) == [(0, model.scan(start=s, limit=m)) for s in starts]
    assert eng.multi_scan(six, starts, m, sstride, ends=ends) == \
        [(0, model.scan(start=s, end=e, limit=m)) for s, e in zip(starts, ends)]
    assert eng.multi_scan_reverse(six, starts, m, sstride, lows=ends) == \
        [(0, model.scan(start=s, end=e, limit=m, reverse=True)) for s, e in zip(starts, ends)]
    assert eng.multi_scan_reverse(six, starts, m, sstride, exclusive=True) == \
        [(0, model.scan(start=s, limit=m, reverse=True, exclusive=True)) for s in starts]
    if device:
        assert scan_device(eng, shard.index, starts, m, sstride) == [(0, model.scan(start=s, limit=m)) for s in starts]
        assert scan_device(eng, shard.index, starts, m, sstride, ends=ends) == \
            [(0, model.scan(start=s, end=e, limit=m)) for s, e in zip(starts, ends)]
        assert scan_device(eng, shard.index, starts, m, sstride, ends=ends, reverse=True) == \
            [(0, model.scan(start=s, end=e, limit=m, reverse=True)) for s, e in zip(starts, ends)]
    # iterators
    upper = key(rng.randrange(0, 66))
    for ub in (None, upper):
        it = shard.iterator(upper_bound=ub)
        iter_walk(it, model.items(), rng, ub)
        it.close()
    # snapshots taken earlier
    for snap, seq in snaps:
        sw = {k: model.get(k, seq) for k in keys}
        for k in keys[::7]:
            assert snap.get(k, cap=4) == ((OK, sw[k]) if sw[k] is not None else (NOT_FOUND, None))
        assert snap.multi_get(keys, stride=8) == [(OK, sw[k]) if sw[k] is not None else (NOT_FOUND, None) for k in keys]
        assert eng.multi_scan_at([snap] * len(starts), starts, m, sstride, ends=ends) == \
            [(0, model.scan(seq, start=s, end=e, limit=m)) for s, e in zip(starts, ends)]
        assert eng.multi_scan_reverse_at([snap] * len(starts), starts, m, sstride) == \
            [(0, model.scan(seq, start=s, limit=m, reverse=True)) for s in starts]
        it = snap.iterator()
        iter_walk(it, model.items(seq), rng)
        it.close()


def random_ops(rng, n, lo=0, hi=64):
    ops = []
    for _ in range(n):
        k = key(rng.randrange(lo, hi))
        r = rng.random()
        if r < 0.55:
            ops.append((MERGE, k, bytes(rng.randrange(256) for _ in range(rng.choice([0, 1, 3, 8, 16])))))
        elif r < 0.75:
            ops.append((PUT, k, b"" if rng.random() < 0.2 else b"base%d" % rng.randrange(1000)))
        elif r < 0.9:
            ops.append((DEL, k, b""))
        else:
            ops.append((SDEL, k, b""))
    return ops


@pytest.mark.parametrize("name", sorted(O.cases()))
def test_recorded_reference_streams(eng, name):
    """Get, MultiGet, both iteration directions, Seek / SeekForPrev, at the latest state and at snapshots: what the
    reference's RocksDB binary answered, checkpoint by checkpoint"""
    delim, steps = O.cases()[name]
    side = O.EngineSide(eng, "sagold%05d" % sorted(O.cases()).index(name), delim)
    try:
        assert O.run_case(side, steps) == O.load_cases()[name]
    finally:
        side.close()


@pytest.mark.parametrize("delim", DELIMS, ids=["comma", "none", "nul"])
def test_every_read_path_through_flushes_and_merges(eng, delim):
    rng = random.Random(11 + DELIMS.index(delim))
    shard, model = new_shard(eng, delim), SA.Model(delim)
    snaps = []
    try:
        for phase in range(5):
            for _ in range(6):
                apply(shard, model, random_ops(rng, 12))
            if phase == 1:
                s = shard.snapshot()
                snaps.append((s, model.seq))
            check_reads(eng, shard, model, rng, snaps, device=False)  # memtable
            assert shard.flush() == 0  # a run; with l0_compaction_trigger = 3, merges of runs follow
            check_reads(eng, shard, model, rng, snaps)
        assert shard.compact() == 0
        check_reads(eng, shard, model, rng, snaps)
        assert shard.stats()["run_entries"] == len(model.items())  # every chain folded to one Put
    finally:
        for s, _ in snaps:
            s.release()
        shard.close()


def test_long_chain_across_memtable_and_runs(eng):
    shard, model = new_shard(eng, b","), SA.Model(b",")
    k = key(7)
    try:
        apply(shard, model, [(PUT, k, b"base")])
        for i in range(1000):
            apply(shard, model, [(MERGE, k, b"%d" % i)])
            if i in (150, 400, 700):
                assert shard.flush() == 0
        want = model.get(k)
        assert want.startswith(b"base,0,1,2,") and want.endswith(b",998,999")
        assert shard.get(k, cap=16) == (OK, want)
        assert shard.multi_get([k, key(8)], stride=16) == [(OK, want), (NOT_FOUND, None)]
        # INCOMPLETE reports the exact size needed
        vals, vlen, st = np.zeros(64, np.uint8), np.zeros(1, np.uint32), np.full(1, -1, np.int32)
        assert eng.multi_get_fixed(np.array([shard.index], np.uint32), np.frombuffer(k, np.uint8), 16, vals, 64, vlen,
                                   st) == 0
        assert (st[0], vlen[0]) == (INCOMPLETE, len(want))
        assert shard.flush() == 0
        assert multi_get_device(eng, shard.index, [k], 64) == [(INCOMPLETE, len(want))]
        assert multi_get_device(eng, shard.index, [k], (len(want) + 15) & ~15) == [(OK, want)]
        # a scan whose folded value does not fit: INCOMPLETE with the records that fit
        assert eng.multi_scan([shard.index], [key(0)], 4, 64) == [(INCOMPLETE, [])]
        assert eng.multi_scan([shard.index], [key(0)], 4, len(want) + 64) == [(0, [(k, want)])]
        assert scan_device(eng, shard.index, [key(0)], 4, 64) == [(INCOMPLETE, [])]
        assert shard.scan() == [(k, want)]
        assert shard.compact() == 0
        st_ = shard.stats()
        assert st_["run_entries"] == 1 and shard.get(k) == (OK, want)
    finally:
        shard.close()


def test_delete_inside_chain_and_empty_base(eng):
    for delim in DELIMS:
        shard, model = new_shard(eng, delim), SA.Model(delim)
        d = delim or b""
        try:
            apply(shard, model, [(MERGE, key(1), b"a"), (MERGE, key(1), b"b")])
            assert shard.flush() == 0
            apply(shard, model, [(DEL, key(1), b""), (MERGE, key(1), b"c"), (MERGE, key(1), b"")])
            apply(shard, model, [(PUT, key(2), b""), (MERGE, key(2), b"x")])   # empty base: an existing value
            apply(shard, model, [(MERGE, key(3), b"x")])                        # no base
            apply(shard, model, [(SDEL, key(4), b""), (MERGE, key(4), b"y"), (MERGE, key(4), b"z")])
            want = {key(1): b"c" + d, key(2): d + b"x", key(3): b"x", key(4): b"y" + d + b"z"}
            for k, v in want.items():
                assert model.get(k) == v
            for phase in range(3):
                assert shard.multi_get(list(want)) == [(OK, v) for v in want.values()]
                assert shard.scan() == sorted(want.items())
                assert [shard.get(k) for k in want] == [(OK, v) for v in want.values()]
                assert shard.flush() == 0 if phase == 0 else shard.compact() == 0
            assert shard.stats()["run_entries"] == 4
        finally:
            shard.close()


def test_partial_merge_keeps_one_operand(eng):
    """a flush above an older run is not at the bottom: operands without a base in the memtable become ONE Merge
    operand o_1 d .. d o_n (the partial merge), which later reads and the full compaction fold onto the base below"""
    shard, model = new_shard(eng, b"|"), SA.Model(b"|")
    try:
        apply(shard, model, [(PUT, key(5), b"old")])
        assert shard.flush() == 0
        snap = shard.snapshot()
        seq = model.seq
        apply(shard, model, [(MERGE, key(5), b"m%d" % i) for i in range(3)] + [(MERGE, key(6), b"n%d" % i) for i in range(3)] +
              [(MERGE, key(7), b"solo")])
        assert shard.flush() == 0
        st = shard.stats()
        # the base, one operand per key instead of three, and the lone operand as it was (two runs: below the trigger)
        assert (st["n_runs"], st["run_entries"]) == (2, 4)
        assert shard.get(key(5)) == (OK, b"old|m0|m1|m2")
        assert shard.get(key(6)) == (OK, b"n0|n1|n2")
        assert snap.get(key(5)) == (OK, b"old") and model.get(key(5), seq) == b"old"
        apply(shard, model, [(MERGE, key(6), b"n3")])
        assert shard.compact() == 0
        assert shard.multi_get([key(5), key(6), key(7)]) == [(OK, b"old|m0|m1|m2"), (OK, b"n0|n1|n2|n3"), (OK, b"solo")]
        assert [model.get(key(5)), model.get(key(6))] == [b"old|m0|m1|m2", b"n0|n1|n2|n3"]
        assert shard.stats()["run_entries"] == 3
        snap.release()
    finally:
        shard.close()


def test_open_refuses_bad_delimiter(eng):
    from rocksplicator_b200 import engine
    lib = eng.lib
    import ctypes as C
    h = C.c_void_p()
    for bad in (0x200, 0x1ff | 0x400, 0x80000000):
        o = engine.ShardOpts(merge_op=engine.MERGE_STRING_APPEND, merge_delim=bad)
        assert lib.rsp_shard_open(eng.h, b"sapp_bad", C.byref(o), C.byref(h)) == INVALID
    # other operators ignore the field
    o = engine.ShardOpts(merge_op=engine.MERGE_UINT64ADD, merge_delim=0x200)
    assert lib.rsp_shard_open(eng.h, b"sapp_other", C.byref(o), C.byref(h)) == OK
    assert lib.rsp_shard_close(h) == OK


def test_multi_get_launches_do_not_grow_with_merged_keys(eng):
    """host-form MultiGet: no host round trip per merged key"""
    shard, model = new_shard(eng, b","), SA.Model(b",")
    try:
        n = 4096 if not EMUL else 256
        ops = []
        for i in range(n):
            ops += [(PUT, key(i), b"b"), (MERGE, key(i), b"o%d" % i)]
        for c in range(0, len(ops), 512):
            apply(shard, model, ops[c:c + 512])
        deltas = []
        for m in (1, n):
            keys = [key(i) for i in range(m)]
            l0 = eng.kernel_launches()
            got = shard.multi_get(keys, stride=32)
            deltas.append(eng.kernel_launches() - l0)
            assert got == [(OK, model.get(k)) for k in keys]
        assert deltas[0] == deltas[1]
    finally:
        shard.close()
