"""GPU: the device-pointer forms (rsp_multi_get_device, rsp_multi_scan_device, rsp_multi_get_at_device,
rsp_apply_staged_device) on callers' CUDA streams, against the oracle port, and their ordering against the engine's own
flushes, compactions, memtable re-allocations, merge installs, snapshot pins and shard closes.

A read that must be ordered is held back on its stream by a bounded device delay (torch.cuda._sleep, about 300 ms,
calibrated once with CUDA events) that the test enqueues itself in front of it; the engine call that follows must not
return before the held read has run, and the read must answer what the shard held when it was issued.  Nothing here
waits for a race: every held read runs after the engine's change, against an installed run set or a zeroed shard.

Under the CPU emulation (tests/test_streams_emul_cpu.py) streams are synchronous and there is no device to delay, so
only the parity items and the scan-with-memtable item run there, on the engine's own stream."""
import ctypes as C
import os
import struct
import time

import numpy as np
import pytest

from oracle import okv
from rocksplicator_b200.write_batch import WriteBatch
from snapshot_oracle import SnapOkv

pytestmark = pytest.mark.gpu
EMUL = bool(os.environ.get("RSP_TEST_EMUL_LIB"))
needs_device = pytest.mark.skipif(EMUL, reason="the CPU emulation's streams are synchronous and torch.cuda._sleep "
                                               "needs a device")
if not EMUL:
    import torch

OK, NOT_FOUND, NOT_SUPPORTED, INVALID, INCOMPLETE, BUSY = 0, 1, 3, 4, 7, 11
HOLD_MS = 300


@pytest.fixture(scope="module")
def eng():
    from rocksplicator_b200 import engine
    e = engine.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def eng2():
    """merges after every second run: background merge installs"""
    from rocksplicator_b200 import engine
    e = engine.Engine(0, l0_compaction_trigger=2)
    yield e
    e.close()


_n = [0]
_ts = [1000]


def key(i):
    return b"key-%012d" % i  # 16 bytes: the fixed-key MultiGet kernels


def val(i, ver, n=64):
    return (b"%d.%d:" % (i, ver) * n)[:n]


class Pair:
    """an engine shard and an oracle DB fed the same batches"""

    def __init__(self, e, merge_op=okv.MERGE_COUNTER, snapshots=False, **kw):
        _n[0] += 1
        self.e = e
        self.s = e.open_shard("strm%05d" % _n[0], merge_op=merge_op, **kw)
        self.o = SnapOkv(merge_op=merge_op) if snapshots else okv.Okv(okv.load_port(), merge_op=merge_op)

    def apply(self, batches):
        ts = list(range(_ts[0], _ts[0] + len(batches)))
        _ts[0] += len(batches)
        st = self.e.apply_many([self.s.index] * len(batches), batches, ts)
        assert not st.any(), st
        for b, t in zip(batches, ts):
            assert self.o.apply(b, t) == 0

    def puts(self, idx, ver, vlen=64):
        self.apply([WriteBatch().put(key(i), val(i, ver, vlen)).data() for i in idx])

    def mixed(self, idx, ver, ctr_keys=False):
        """overwrites, Deletes and counter Merges (onto Puts of 64 bytes, which fails the merge as RocksDB does, or with
        ctr_keys onto counter keys of their own)"""
        out = []
        for i in idx:
            wb = WriteBatch()
            if i % 7 == 0:
                wb.delete(key(i))
            elif i % 5 == 0:
                wb.merge(key(10 ** 6 + i % 97 if ctr_keys else i), struct.pack("<q", i + ver))
            else:
                wb.put(key(i), val(i, ver))
            out.append(wb.data())
        self.apply(out)

    def close(self):
        self.s.close()
        self.o.close()


def compacted(e, n, **kw):
    p = Pair(e, **kw)
    p.puts(range(n), 0)
    assert p.s.compact() == 0
    return p


def ingested(e, n, **kw):
    """n Puts as one ingested run: no flush, so the memtable keeps its configured size and no background merge is
    left to run later"""
    p = Pair(e, **kw)
    assert p.s.ingest([(key(i), val(i, 0)) for i in range(n)]) == OK
    for i in range(n):
        assert p.o.apply(WriteBatch().put(key(i), val(i, 0)).data(), 0) == 0
    return p


# ---- device buffers and the device forms --------------------------------------------------------------------------
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


def new_stream(eng):
    """a caller's stream (non-blocking); under the emulation the engine's own"""
    return eng.lib.rsp_engine_stream(eng.h) if EMUL else torch.cuda.Stream()


def _sp(stream):
    return stream if EMUL else stream.cuda_stream


class MGet:
    """rsp_multi_get_device over shard indices, or with at=True rsp_multi_get_at_device over snapshot slots.  Its
    buffers are uploaded (a device-wide synchronisation) when it is made; with stream=None it is launched later
    (launch), so that a held stream is not waited for by the upload."""

    def __init__(self, e, ix, keys, stride, stream=None, at=False):
        n = len(keys)
        self.e, self.at, self.stride, self.n = e, at, stride, n
        self.d = _dev([np.asarray(ix, dtype=np.uint32), np.frombuffer(b"".join(keys), dtype=np.uint8),
                       np.zeros(max(n * stride, 1), dtype=np.uint8), np.zeros(n, dtype=np.uint32),
                       np.full(n, -1, dtype=np.int32)])
        if stream is not None:
            self.launch(stream)

    def launch(self, stream):
        e, p = self.e, [_ptr(a) for a in self.d]
        fn = e.lib.rsp_multi_get_at_device if self.at else e.lib.rsp_multi_get_device
        assert fn(e.h, self.n, p[0], p[1], 16, p[2], self.stride, p[3], p[4], _sp(stream)) == OK
        return self

    def result(self):
        _, _, vals, vlen, st = _host(self.d)
        out = []
        for i in range(self.n):
            s = int(st[i])
            if s == OK:
                out.append((s, vals[i * self.stride:i * self.stride + int(vlen[i])].tobytes()))
            else:
                out.append((s, int(vlen[i]) if s == INCOMPLETE else None))
        return out


def want_get(o, keys, stride, snapshot=None):
    res = o.multi_get(keys) if snapshot is None else o.multi_get(keys, snapshot=snapshot)
    return [(INCOMPLETE, len(v)) if st == OK and len(v) > stride else (st, v) for st, v in res]


def same(got, want):
    """got == want, failing with a short report (pytest's full diff of thousands of answers takes minutes)"""
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    if len(got) != len(want) or bad:
        i = bad[0] if bad else min(len(got), len(want))
        g = got[i] if i < len(got) else None
        w = want[i] if i < len(want) else None
        raise AssertionError("%d of %d answers differ (lengths %d / %d); first at %d: got %.300r, want %.300r" % (
            len(bad), len(want), len(got), len(want), i, g, w))


class MScan:
    """rsp_multi_scan_device; made and launched as MGet"""

    def __init__(self, e, six, starts, max_entries, stride, stream=None):
        n = len(starts)
        self.e, self.max_entries, self.stride, self.n = e, max_entries, stride, n
        self.d = _dev([np.asarray(six, dtype=np.uint32), np.frombuffer(b"".join(starts), dtype=np.uint8),
                       np.zeros(n * stride, dtype=np.uint8), np.full(n, 0xFFFFFFFF, dtype=np.uint32),
                       np.full(n, -1, dtype=np.int32)])
        if stream is not None:
            self.launch(stream)

    def launch(self, stream):
        e, p = self.e, [_ptr(a) for a in self.d]
        assert e.lib.rsp_multi_scan_device(e.h, self.n, p[0], p[1], 16, self.max_entries, p[2], self.stride, p[3],
                                           p[4], _sp(stream)) == OK
        return self

    def result(self):
        _, _, out, n_out, st = _host(self.d)
        res = []
        for i in range(self.n):
            recs, at = [], i * self.stride
            for _ in range(int(n_out[i])):
                kl = int(out[at:at + 4].view(np.uint32)[0])
                vl = int(out[at + 4:at + 8].view(np.uint32)[0])
                recs.append((out[at + 8:at + 8 + kl].tobytes(), out[at + 8 + kl:at + 8 + kl + vl].tobytes()))
                at += 8 + kl + vl
            res.append((int(st[i]), recs))
        return res


def staged_tick(e, six, batches):
    """rsp_stage_build + rsp_reserve: the handle for launch_tick / finish_tick, and the batches' timestamps"""
    n = len(batches)
    off = np.zeros(n + 1, dtype=np.uint64)
    np.cumsum([len(b) for b in batches], out=off[1:])
    blob = np.frombuffer(b"".join(batches) + b"\0", dtype=np.uint8).copy()
    six = np.ascontiguousarray(six, dtype=np.uint32)
    ts = np.arange(_ts[0], _ts[0] + n, dtype=np.uint64)
    _ts[0] += n
    h = C.c_void_p()
    assert e.lib.rsp_stage_build(e.h, n, six.ctypes.data, blob.ctypes.data, off.ctypes.data, ts.ctypes.data,
                                 C.byref(h)) == OK
    assert e.lib.rsp_reserve(e.h, h) == OK
    return h, ts


def launch_tick(e, h, stream):
    assert e.lib.rsp_apply_staged_device(e.h, h, _sp(stream)) == OK


def finish_tick(e, h, n):
    st = np.full(n, -1, dtype=np.int32)
    assert e.lib.rsp_apply_staged_finish(e.h, h, st.ctypes.data) == OK
    e.lib.rsp_stage_free(h)
    return st


# ---- holding a read back: a bounded device delay on a stream the test owns ------------------------------------------
_cycles_per_ms = []


def held(stream, ms=HOLD_MS):
    if not _cycles_per_ms:
        s = torch.cuda.Stream()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        rates = []
        for _ in range(3):  # the fastest of three: a clock still ramping up would make later holds shorter
            with torch.cuda.stream(s):
                e0.record(s)
                torch.cuda._sleep(40_000_000)
                e1.record(s)
            e1.synchronize()
            rates.append(40_000_000 / e0.elapsed_time(e1))
        _cycles_per_ms.append(max(rates))
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(_cycles_per_ms[0] * ms))


def done_event(stream):
    ev = torch.cuda.Event()
    ev.record(stream)
    return ev


def require_held(a_done):
    """the held read has not run yet, so the engine call that follows comes before it.  Anything that synchronises the
    whole device in between (a cudaFree when a scratch buffer grows) ends the hold early: then the scenario did not
    happen and is skipped, as it says nothing either way."""
    if a_done.query():
        pytest.skip("the held read ran before the engine call was issued (the device was synchronised in between)")


# ================================================================================================================
# 1. parity of every device form on one caller stream and on two alternating ones
# ================================================================================================================
@pytest.fixture(scope="module")
def shapes(eng):
    """shards of every shape the read kernels tell apart, each with its oracle"""
    one = compacted(eng, 3000)                       # one run of fixed-size Puts
    several = Pair(eng)                              # three runs (the engine merges at four)
    for v in range(3):
        several.mixed(range(v * 500, 3000, 3), v + 1)
        assert several.s.flush() == 0
    mem = compacted(eng, 2000)                       # a run and a live memtable
    mem.mixed(range(0, 2400, 2), 5)
    big = Pair(eng)                                  # values beyond the stride
    big.puts(range(300), 0, vlen=200)
    assert big.s.flush() == 0
    big.puts(range(0, 300, 4), 1, vlen=40)
    ps = {"one": one, "several": several, "mem": mem, "big": big}
    assert several.s.stats()["n_runs"] == 3 and mem.s.stats()["memtable_entries"] > 0
    yield ps
    for p in ps.values():
        p.close()


def _lookups(p, seed, n=700, space=3300):
    rng = np.random.default_rng(seed)
    return [key(int(i)) for i in rng.integers(0, space, size=n)]  # keys beyond the written range miss


@pytest.mark.parametrize("n_streams", [1, 2])
def test_multi_get_device_parity_on_caller_streams(eng, shapes, n_streams):
    streams = [new_stream(eng) for _ in range(n_streams)]
    calls = []
    for r in range(3):
        for j, (name, p) in enumerate(sorted(shapes.items())):
            stride = 64 if name == "big" else 128
            keys = _lookups(p, 17 * r + j, space=400 if name == "big" else 3300)
            calls.append((MGet(eng, [p.s.index] * len(keys), keys, stride, streams[len(calls) % n_streams]),
                          want_get(p.o, keys, stride)))
    # one launch across every shape at once
    keys, six, want = [], [], []
    for j, p in enumerate(shapes.values()):
        k = _lookups(p, 99 + j, n=300)
        keys += k
        six += [p.s.index] * len(k)
        want += want_get(p.o, k, 96)
    calls.append((MGet(eng, six, keys, 96, streams[-1]), want))
    for got, want in calls:
        r = got.result()
        same(r, want)
    assert any(s == INCOMPLETE for s, _ in calls[-1][1]) and any(s == NOT_FOUND for s, _ in calls[-1][1])


@pytest.mark.parametrize("n_streams", [1, 2])
def test_multi_scan_device_parity_on_caller_streams(eng, shapes, n_streams):
    streams = [new_stream(eng) for _ in range(n_streams)]
    one, several = shapes["one"], shapes["several"]
    rng = np.random.default_rng(5)
    calls = []
    for r in range(4):
        starts = [key(int(i)) for i in rng.integers(0, 3100, size=40)]
        six = [(one if i % 2 else several).s.index for i in range(40)]
        calls.append((MScan(eng, six, starts, 50, 50 * 96, streams[r % n_streams]),
                      [(OK, (one if i % 2 else several).o.scan(s, 50)) for i, s in enumerate(starts)]))
    for got, want in calls:
        same(got.result(), want)


@pytest.mark.parametrize("n_streams", [1, 2])
def test_multi_get_at_device_parity_on_caller_streams(eng, n_streams):
    streams = [new_stream(eng) for _ in range(n_streams)]
    p = Pair(eng, snapshots=True)
    p.puts(range(1500), 0)
    snaps = []
    for v in range(4):
        snaps.append((p.s.snapshot(), p.o.snapshot()))
        p.mixed(range(v, 1600, 3), v + 1)
        if v == 1:
            assert p.s.flush() == 0
    calls = []
    for r in range(6):
        keys = _lookups(p, r, n=400, space=1700)
        which = [(i + r) % len(snaps) for i in range(len(keys))]
        want = []
        for j, (_, osn) in enumerate(snaps):
            sel = [k for k, w in zip(keys, which) if w == j]
            want.append(iter(want_get(p.o, sel, 128, snapshot=osn)))
        calls.append((MGet(eng, [snaps[w][0].slot for w in which], keys, 128, streams[r % n_streams], at=True),
                      [next(want[w]) for w in which]))
    for got, want in calls:
        same(got.result(), want)
    for sn, osn in snaps:
        sn.release()
        osn.release()
    p.close()


@pytest.mark.parametrize("n_streams", [1, 2])
def test_apply_staged_device_on_caller_streams(eng, n_streams):
    streams = [new_stream(eng) for _ in range(n_streams)]
    ps = [Pair(eng) for _ in range(3)]
    for t in range(4):
        six, batches = [], []
        for i in range(300):
            p = ps[i % 3]
            wb = WriteBatch().put(key(i + 7 * t), val(i, t)).merge(key(5000 + i % 11), struct.pack("<q", i))
            if i % 9 == 0:
                wb.delete(key(i * 3))
            six.append(p.s.index)
            batches.append(wb.data())
        h, ts = staged_tick(eng, six, batches)
        launch_tick(eng, h, streams[t % n_streams])
        assert not finish_tick(eng, h, len(batches)).any()
        for j, b, tt in zip(six, batches, ts):
            assert [p for p in ps if p.s.index == j][0].o.apply(b, int(tt)) == 0
    for p in ps:
        keys = [key(i) for i in range(0, 400)] + [key(5000 + i) for i in range(12)]
        same(p.s.multi_get(keys, stride=64), p.o.multi_get(keys))
        assert p.s.latest_seq() == p.o.latest_seq()
        p.close()


# ================================================================================================================
# 7. a device-form scan of a shard with unflushed writes should answer NotSupported instead of the runs alone
# ================================================================================================================
@pytest.mark.xfail(strict=True, reason="rsp_multi_scan_device reads the sorted runs only and answers a shard with "
                   "unflushed writes with its runs and status 0; the check in k_multi_scan cost 0.7 % of the scan rate "
                   "and is left for a change of its own")
def test_device_scan_answers_not_supported_over_a_memtable(eng):
    stream = new_stream(eng)
    m = compacted(eng, 1200)
    m.mixed(range(0, 1400, 3), 1, ctr_keys=True)  # Puts, Deletes and Merges over the run, unflushed
    e = compacted(eng, 900)
    starts = [key(0), key(301), key(1380), key(0), key(450)]
    six = [m.s.index, e.s.index, m.s.index, e.s.index, m.s.index]
    got = MScan(eng, six, starts, 64, 64 * 96, stream).result()
    for (st, recs), j, s in zip(got, six, starts):
        if j == m.s.index:
            assert (st, recs) == (NOT_SUPPORTED, [])
        else:
            assert (st, recs) == (OK, e.o.scan(s, 64))
    assert m.s.flush() == 0
    got = MScan(eng, six, starts, 64, 64 * 96, stream).result()
    same(got, [(OK, (m if j == m.s.index else e).o.scan(s, 64)) for j, s in zip(six, starts)])
    m.close()
    e.close()


def test_device_forms_on_a_closed_shard(eng):
    """what a held read meets when a close was not ordered after it: a zeroed, not-live shard"""
    stream = new_stream(eng)
    x = compacted(eng, 500)
    ix = x.s.index
    x.close()
    keys = [key(i) for i in range(0, 500, 7)]
    same(MGet(eng, [ix] * len(keys), keys, 64, stream).result(), [(INVALID, None)] * len(keys))
    same(MScan(eng, [ix] * 3, keys[:3], 16, 16 * 96, stream).result(), [(OK, [])] * 3)


# ================================================================================================================
# 4. device MultiGets on two streams share the engine's pending list one after the other
# ================================================================================================================
@needs_device
def test_pending_list_across_streams(eng, shapes):
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    set_a = [shapes["one"], shapes["several"]]
    set_b = [shapes["mem"], shapes["big"], compacted(eng, 800)]
    calls = []
    for which, stream in ((set_a, a), (set_b, b)):
        keys, six, want = [], [], []
        for j, p in enumerate(which):
            k = _lookups(p, 40 + j, n=1500)
            keys += k
            six += [p.s.index] * len(k)
            want += want_get(p.o, k, 96)
        calls.append((MGet(eng, six, keys, 96), want, stream))
    held(a)
    for got, _, stream in calls:
        got.launch(stream)
    for got, want, _ in calls:
        same(got.result(), want)
    set_b[-1].close()


# ================================================================================================================
# 2. a shard close waits for a read held on a caller stream, however many reads follow it on other streams
# ================================================================================================================
@pytest.fixture(scope="module")
def others(eng):
    ps = [compacted(eng, 1000, snapshots=True) for _ in range(2)]
    snap = ps[0].s.snapshot()
    yield ps, snap
    snap.release()
    for p in ps:
        p.close()


def readers_between(eng, others, via, k):
    """k reads on other streams, made before the hold; call the result to issue them"""
    ps, snap = others
    keys = [key(i) for i in range(0, 1000, 97)]
    if via == "get":  # the read combiner: one device batch on its own stream per call
        def run(stream):
            for i in range(k):
                p = ps[i % 2]
                assert p.s.get(keys[i % len(keys)]) == p.o.get(keys[i % len(keys)])
        return run
    if via == "scan":
        rs = [MScan(eng, [ps[i % 2].s.index] * 2, keys[:2], 8, 8 * 96) for i in range(k)]
    else:
        rs = [MGet(eng, [snap.slot] * 4, keys[:4], 96, at=True) for _ in range(k)]

    def run(stream):
        for r in rs:
            r.launch(stream)
    return run


@needs_device
@pytest.mark.parametrize("via", ["get", "scan", "get_at"])
@pytest.mark.parametrize("k", [0, 1, 7, 8, 9, 32])
def test_close_waits_for_a_held_read(eng, others, k, via):
    a, c = torch.cuda.Stream(), torch.cuda.Stream()
    x = compacted(eng, 2000)
    x.mixed(range(0, 2000, 5), 1)
    keys = [key(i) for i in range(0, 2200, 3)]
    want = want_get(x.o, keys, 96)
    r, between = MGet(eng, [x.s.index] * len(keys), keys, 96), readers_between(eng, others, via, k)
    held(a)
    r.launch(a)
    a_done = done_event(a)
    between(c)
    require_held(a_done)
    x.s.close()
    at_close = a_done.query()
    same(r.result(), want)
    assert at_close, "rsp_shard_close returned before the read held on another stream had run"
    x.o.close()


# ================================================================================================================
# 3. every mutation of the engine waits for a read held on a caller stream, with nine combiner reads after it
# ================================================================================================================
@needs_device
@pytest.mark.parametrize("read", ["multi_get", "scan"])
@pytest.mark.parametrize("mutation", ["flush", "compact", "compact_all", "apply_flush", "apply_realloc", "snapshot"])
def test_mutation_waits_for_a_held_read(eng, others, mutation, read):
    a = torch.cuda.Stream()
    ps, _ = others
    s = ingested(eng, 1500, write_buffer_bytes=64 << 10)
    if mutation != "apply_realloc":
        s.mixed(range(0, 1500, 6), 1)  # a live memtable
    assert (s.s.stats()["memtable_entries"] > 0) == (mutation != "apply_realloc")
    if read == "multi_get":
        keys = [key(i) for i in range(0, 1700, 2)]
        want = want_get(s.o, keys, 96)
    else:
        starts = [key(i) for i in range(0, 1000, 50)]
        want = [(OK, ps[i % 2].o.scan(st, 32)) for i, st in enumerate(starts)]
    if read == "multi_get":
        r = MGet(eng, [s.s.index] * len(keys), keys, 96)
    else:
        r = MScan(eng, [ps[i % 2].s.index for i in range(len(starts))], starts, 32, 32 * 96)
    held(a)
    r.launch(a)
    a_done = done_event(a)
    readers_between(eng, others, "get", 9)(None)
    require_held(a_done)
    flushes0 = s.s.stats()["flushes"]
    snap = None
    if mutation == "flush":
        assert s.s.flush() == OK
    elif mutation == "compact":
        assert s.s.compact() == OK
    elif mutation == "compact_all":
        assert eng.compact_all() == OK
    elif mutation == "apply_flush":  # does not fit the live memtable: flushed on the apply path
        s.puts(range(0, 1500, 3), 2)
    elif mutation == "apply_realloc":  # larger than the empty memtable: re-allocated on the apply path
        s.apply([WriteBatch().put(key(i), val(i, 3)).data() for i in range(1200)])
    else:  # the memtable is sorted into the snapshot's private run
        snap = s.s.snapshot()
    at_return = a_done.query()
    same(r.result(), want)
    assert at_return, "%s returned before the read held on another stream had run" % mutation
    st = s.s.stats()
    if mutation in ("flush", "apply_flush"):
        assert st["flushes"] > flushes0
    if snap is not None:
        snap.release()
    s.close()


@needs_device
def test_merge_install_waits_for_a_held_read(eng2):
    a = torch.cuda.Stream()
    r_ = compacted(eng2, 200)
    s = Pair(eng2)
    s.puts(range(0, 150000), 0)
    assert s.s.flush() == OK
    s.mixed(range(0, 150000, 2), 1)
    keys = [key(i) for i in range(0, 151000, 151)]
    want = want_get(s.o, keys, 96)
    r = MGet(eng2, [s.s.index] * len(keys), keys, 96)
    assert s.s.flush() == OK  # the second run: a background merge is requested
    held(a)
    r.launch(a)
    a_done = done_event(a)
    if s.s.stats()["n_runs"] < 2:
        torch.cuda.synchronize()
        pytest.skip("the merge was installed before the read was issued")
    assert not a_done.query()
    for i in range(9):  # (these may wait for the install, which holds the engine lock while it waits for the read)
        assert r_.s.get(key(i)) == r_.o.get(key(i))
    t0 = time.monotonic()
    while s.s.stats()["n_runs"] >= 2:
        assert time.monotonic() - t0 < 30, "no merge install"
        time.sleep(0.0005)
    at_install = a_done.query()
    same(r.result(), want)
    assert at_install, "the merge was installed before the read held on another stream had run"
    same(s.s.multi_get(keys, stride=96), s.o.multi_get(keys))
    s.close()
    r_.close()


# ================================================================================================================
# 5. a read at a snapshot held on a caller stream while the shard takes applies, a flush, a compaction, a background
#    merge and another snapshot's release
# ================================================================================================================
@needs_device
def test_snapshot_read_held_on_a_caller_stream(eng2):
    a = torch.cuda.Stream()
    p = Pair(eng2, snapshots=True)
    p.puts(range(3000), 0)
    assert p.s.flush() == OK
    p.mixed(range(0, 3200, 4), 1)
    snap, osnap = p.s.snapshot(), p.o.snapshot()
    other, oother = p.s.snapshot(), p.o.snapshot()
    keys = [key(i) for i in range(0, 3300, 3)]
    want = want_get(p.o, keys, 96, snapshot=osnap)
    r = MGet(eng2, [snap.slot] * len(keys), keys, 96, at=True)
    held(a)
    r.launch(a)
    p.mixed(range(1, 3300, 2), 2)
    assert p.s.flush() == OK  # two runs: a background merge
    p.mixed(range(0, 3300, 5), 3)
    assert p.s.compact() == OK
    p.mixed(range(0, 3300, 7), 4)
    other.release()
    oother.release()
    same(r.result(), want)
    same(p.s.multi_get(keys, stride=96), p.o.multi_get(keys))
    snap.release()
    osnap.release()
    p.close()


# ================================================================================================================
# 6. a tick held on a caller stream: maintenance on its shards answers Busy, host reads see whole batches
# ================================================================================================================
@needs_device
def test_tick_held_on_a_caller_stream(eng):
    a = torch.cuda.Stream()
    p = Pair(eng)
    ctr = key(77)

    def three():
        return WriteBatch().merge(ctr, struct.pack("<q", 1)).merge(ctr, struct.pack("<q", 1)) \
            .merge(ctr, struct.pack("<q", 1)).data()
    p.apply([three() for _ in range(3)])
    batches = [three() for _ in range(40)]
    h, ts = staged_tick(eng, [p.s.index] * len(batches), batches)
    held(a)
    launch_tick(eng, h, a)
    assert p.s.flush() == BUSY
    assert p.s.compact() == BUSY
    out = C.c_void_p()
    assert eng.lib.rsp_snapshot_create(p.s.h, C.byref(out)) == BUSY
    for _ in range(5):
        st, v = p.s.get(ctr)
        assert st == OK and struct.unpack("<q", v)[0] % 3 == 0
    assert not finish_tick(eng, h, len(batches)).any()
    for b, t in zip(batches, ts):
        assert p.o.apply(b, int(t)) == 0
    assert p.s.get(ctr) == p.o.get(ctr) == (OK, struct.pack("<q", 129))
    assert p.s.flush() == OK and p.s.compact() == OK
    with p.s.snapshot() as sn:
        assert sn.get(ctr) == (OK, struct.pack("<q", 129))
    p.close()
