"""GPU: snapshots (rsp_snapshot_create / rsp_get_at / rsp_multi_get_at / rsp_multi_get_at_device / rsp_iter_create_at)
against the reference's RocksDB binary (tests/golden/snapshots.json) and against the oracle port on seeded streams,
while applies, flushes, foreground compactions and background merges go on."""
import ctypes as C
import os
import random
import struct
import threading

import numpy as np
import pytest

import golden_util as G
import snapshot_streams as S
from snapshot_oracle import SnapOkv
from oracle import okv
from rocksplicator_b200.write_batch import WriteBatch
from streams import random_stream

pytestmark = pytest.mark.gpu
EMUL = bool(os.environ.get("RSP_TEST_EMUL_LIB"))
CASES = G.load("snapshots.json")
BUSY = 11


@pytest.fixture(scope="module")
def eng():
    from rocksplicator_b200 import engine
    e = engine.Engine(0, l0_compaction_trigger=2)  # background merges replace pinned runs often
    yield e
    e.close()


_n = [0]


def new_shard(eng, merge_op=0, **kw):
    _n[0] += 1
    return eng.open_shard("snap%05d" % _n[0], merge_op=merge_op, **kw)


def append_fn(state, key, klen, ex, exl, op, opl, out_set, out_ctx):
    """RSP_MERGE_CALLBACK implementing the append operator on the host"""
    v = (C.string_at(ex, exl) if ex else b"") + C.string_at(op, opl)
    C.CFUNCTYPE(None, C.c_void_p, C.c_char_p, C.c_size_t)(out_set)(out_ctx, v, len(v))
    return 1


@pytest.mark.parametrize("merge,seed", S.STREAM_CASES, ids=lambda x: str(x))
def test_golden_snapshot_streams(eng, merge, seed):
    s = new_shard(eng, S.MERGES[merge])
    assert S.run_stream(S.EngineSide(s), merge, seed, G.digest) == CASES["streams"]["%s-%d" % (merge, seed)]
    s.close()


@pytest.mark.parametrize("seed", [0, 1])
def test_host_callback_operator_at_snapshots(eng, seed):
    from rocksplicator_b200 import engine
    s = new_shard(eng, engine.MERGE_CALLBACK, merge_fn=append_fn)
    assert S.run_stream(S.EngineSide(s), "append", seed, G.digest) == CASES["streams"]["append-%d" % seed]
    s.close()


@pytest.mark.parametrize("step", S.ingest_steps(), ids=lambda x: x[0])
def test_ingest_with_live_snapshots_matches_reference(eng, step):
    name, rows, allow, with_snapshot = step
    s = new_shard(eng)

    def ingest(rows, allow):
        rc = s.ingest(rows, allow_global_seqno=allow)
        return rc, s.last_error if rc else ""
    want = [r for r in CASES["ingest"] if r[0] == name][0]
    assert S.run_ingest(S.EngineSide(s), name, rows, allow, with_snapshot, ingest, G.digest) == want
    s.close()


def _device_form(eng, slots, keys, klen, stride):
    """rsp_multi_get_at_device over device buffers (numpy memory under the CPU emulation)"""
    n = len(keys)
    h = [np.ascontiguousarray(slots, dtype=np.uint32), np.frombuffer(b"".join(keys), dtype=np.uint8).copy(),
         np.zeros(n * stride, dtype=np.uint8), np.zeros(n, dtype=np.uint32), np.full(n, -1, dtype=np.int32)]
    if EMUL:
        d = h
        ptr = [a.ctypes.data for a in d]
    else:
        import torch
        d = [torch.from_numpy(a).cuda() for a in h]
        torch.cuda.synchronize()
        ptr = [t.data_ptr() for t in d]
    assert eng.lib.rsp_multi_get_at_device(eng.h, n, ptr[0], ptr[1], klen, ptr[2], stride, ptr[3], ptr[4], None) == 0
    if not EMUL:
        torch.cuda.synchronize()
        d = [t.cpu().numpy() for t in d]
    vals, vlen, st = d[2], d[3], d[4]
    return [(int(st[i]), vals[i * stride:i * stride + vlen[i]].tobytes() if st[i] == 0 else int(vlen[i]))
            for i in range(n)]


def test_cross_shard_reads_at_many_snapshots(eng):
    """Get, cross-shard MultiGet (host and device forms) and iterator walks at many live snapshots of three shards
    (device and host-folded operators, values larger than the stride, 16-byte keys) while writes, flushes, foreground
    compactions and background merges continue"""
    rng = random.Random(11)
    specs = [(okv.MERGE_COUNTER, "counter", False), (okv.MERGE_APPEND, "append", True),
             (okv.MERGE_UINT64ADD, "counter", False)]
    shards, ports, streams, keysets = [], [], [], []
    for i, (mop, mname, var_len) in enumerate(specs):
        keys, stream = random_stream(300 + i, 120, n_keys=30, merge=mname, var_len=var_len)
        shards.append(new_shard(eng, mop))
        ports.append(SnapOkv(merge_op=mop))
        streams.append(stream)
        keysets.append(keys)
    snaps = []  # (shard index, engine snapshot, port snapshot)
    for step in range(120):
        for i in range(3):
            b, ts = streams[i][step]
            assert shards[i].apply(b, ts) == ports[i].apply(b, ts)
        r = rng.random()
        i = rng.randrange(3)
        if r < 0.12:
            shards[i].flush()
        elif r < 0.16:
            shards[i].compact()
        if step % 6 == 5:
            i = rng.randrange(3)
            es, ps = shards[i].snapshot(), ports[i].snapshot()
            assert es.seq == ps.seq == ports[i].latest_seq()
            snaps.append((i, es, ps))
        if step % 20 == 19 and len(snaps) > 4:  # release some as we go
            i, es, ps = snaps.pop(rng.randrange(len(snaps)))
            es.release()
            ps.release()
    for i, es, ps in snaps:
        probe = keysets[i] + [b"zz-missing"]
        assert [es.get(k) for k in probe] == [ports[i].get(k, snapshot=ps) for k in probe]
        assert es.scan() == ports[i].scan(snapshot=ps)
        a, b = es.iterator(), ports[i].iterator(ps)
        a.seek_to_last(), b.seek_to_last()
        while b.valid():
            assert a.valid() and (a.key(), a.value()) == (b.key(), b.value())
            a.prev(), b.prev()
        assert not a.valid()
        a.close(), b.close()
    # one call over every shard's snapshots, with null handles and a stride smaller than many values
    pick = [(rng.randrange(len(snaps)), None) for _ in range(400)]
    pick = [(j, rng.choice(keysets[snaps[j][0]] + [b"zz-missing"])) for j, _ in pick]
    handles = [snaps[j][1] for j, _ in pick] + [None]
    got = eng.multi_get_at(handles, [k for _, k in pick] + [b"x"], stride=64)
    want = [ports[snaps[j][0]].get(k, snapshot=snaps[j][2]) for j, k in pick] + [(4, None)]
    assert got == want
    # Incomplete: the size needed comes back
    big = [(j, k) for j, k in pick if want[pick.index((j, k))][0] == 0 and len(want[pick.index((j, k))][1]) > 8]
    if big:
        j, k = big[0]
        n = C.c_size_t()
        buf = C.create_string_buffer(8)
        assert eng.lib.rsp_get_at(snaps[j][1].h, k, len(k), buf, 8, C.byref(n)) == 7
        assert n.value == len(ports[snaps[j][0]].get(k, snapshot=snaps[j][2])[1])
    # device form over the 16-byte-key shards (host-folded operators answer 100 there)
    dev = [(j, k) for j, k in pick if specs[snaps[j][0]][0] != okv.MERGE_APPEND and len(k) == 16]
    assert len(dev) > 100
    got = _device_form(eng, [snaps[j][1].slot for j, _ in dev] + [RSP_FREE_SLOT], [k for _, k in dev] + [b"\0" * 16],
                       16, 256)
    for (j, k), g in zip(dev, got):
        w = ports[snaps[j][0]].get(k, snapshot=snaps[j][2])
        assert g[0] == w[0] and (w[0] != 0 or g[1] == w[1]), (j, k, g, w)
    assert got[-1][0] == 4
    for i, es, ps in snaps:
        es.release()
        ps.release()
    for s in shards:
        s.close()
    for p in ports:
        p.close()


RSP_FREE_SLOT = 4095  # the table's last slot: no test holds 4096 snapshots


def test_empty_shard_snapshot(eng):
    s = new_shard(eng)
    with s.snapshot() as snap:
        assert snap.seq == 0
        assert snap.get(b"a") == (1, None) and snap.scan() == [] and snap.multi_get([b"a", b""]) == [(1, None)] * 2
        assert s.apply(WriteBatch().put(b"a", b"1").data(), 1) == 0
        assert snap.get(b"a") == (1, None) and s.get(b"a") == (0, b"1")
    s.close()


def test_snapshot_meets_the_run_table_fold_in():
    """eight sorted runs plus a memtable do not fit a view: the memtable is flushed into the shard first"""
    from rocksplicator_b200 import engine
    e = engine.Engine(0, l0_compaction_trigger=8)
    s = e.open_shard("fold")
    model = {}
    for r in range(7):
        for i in range(20):
            k, v = b"r%d-%03d" % (r, i), b"v%d" % (r * 100 + i)
            assert s.apply(WriteBatch().put(k, v).data(), 1) == 0
            model[k] = v
        assert s.flush() == 0
    rows = [(b"zz%03d" % i, b"ing%d" % i) for i in range(10)]
    assert s.ingest(rows) == 0
    model.update(rows)
    assert s.apply(WriteBatch().put(b"r0-000", b"newest").delete(b"r1-001").data(), 1) == 0
    model[b"r0-000"] = b"newest"
    del model[b"r1-001"]
    runs_before = s.stats()["n_runs"]
    with s.snapshot() as snap:
        if runs_before == 8:
            assert s.stats()["memtable_entries"] == 0
        assert snap.scan() == sorted(model.items())
        assert s.apply(WriteBatch().put(b"r0-000", b"later").data(), 1) == 0
        assert snap.get(b"r0-000") == (0, b"newest")
    s.close()
    e.close()


def test_iterator_outlives_its_snapshot(eng):
    s = new_shard(eng)
    for i in range(50):
        assert s.apply(WriteBatch().put(b"k%02d" % i, b"v%d" % i).data(), 1) == 0
    snap = s.snapshot()
    it = snap.iterator()
    snap.release()
    assert s.apply(WriteBatch().delete(b"k00").put(b"k01", b"new").data(), 1) == 0
    s.compact()
    it.seek_to_first()
    got = []
    while it.valid():
        got.append((it.key(), it.value()))
        it.next()
    it.close()
    assert got == [(b"k%02d" % i, b"v%d" % i) for i in range(50)]
    s.close()


def test_shard_close_is_busy_while_a_snapshot_is_live(eng):
    s = new_shard(eng)
    snap = s.snapshot()
    assert eng.lib.rsp_shard_close(s.h) == BUSY
    assert snap.get(b"x") == (1, None)
    snap.release()
    assert eng.lib.rsp_shard_close(s.h) == 0
    s.h = None


def test_snapshot_create_is_busy_while_staged_ticks_are_in_flight(eng):
    s = new_shard(eng)
    lib = eng.lib
    batches = [WriteBatch().put(b"a%d" % i, b"v").data() for i in range(4)]
    off = np.zeros(5, dtype=np.uint64)
    np.cumsum([len(b) for b in batches], out=off[1:])
    blob = np.frombuffer(b"".join(batches) + b"\0", dtype=np.uint8).copy()
    six = np.full(4, s.index, dtype=np.uint32)
    ts = np.ones(4, dtype=np.uint64)
    h = C.c_void_p()
    assert lib.rsp_stage_build(eng.h, 4, six.ctypes.data, blob.ctypes.data, off.ctypes.data, ts.ctypes.data, C.byref(h)) == 0
    assert lib.rsp_reserve(eng.h, h) == 0
    assert lib.rsp_apply_staged_device(eng.h, h, None) == 0
    out = C.c_void_p()
    assert lib.rsp_snapshot_create(s.h, C.byref(out)) == BUSY
    st = np.zeros(4, dtype=np.int32)
    assert lib.rsp_apply_staged_finish(eng.h, h, st.ctypes.data) == 0
    lib.rsp_stage_free(h)
    with s.snapshot() as snap:
        assert snap.seq == 4 and snap.get(b"a3") == (0, b"v")
    s.close()


def _in_use(eng):
    out = (C.c_uint64 * 4)()
    eng.lib.rsp_debug_arena(eng.h, out)
    return out[0]


def test_hbm_goes_back_after_release_and_merge():
    """a snapshot pins the runs a merge replaces; after the release, the shard holds exactly what a twin shard with
    the same history and no snapshot holds"""
    from rocksplicator_b200 import engine
    e = engine.Engine(0)
    a, b = e.open_shard("with"), e.open_shard("twin")
    keys, stream = random_stream(77, 200, n_keys=60, merge="counter")
    for s in (a, b):
        s._rc = [s.apply(bt, ts) for bt, ts in stream[:100]]
        s.flush()
        for bt, ts in stream[100:150]:
            s.apply(bt, ts)
    before = _in_use(e)
    snap = a.snapshot()  # the memtable's contents become a private run
    assert _in_use(e) > before
    for s in (a, b):
        for bt, ts in stream[150:]:
            s.apply(bt, ts)
        s.compact()  # the runs the snapshot pins leave the shard
    held = _in_use(e)
    snap.release()
    assert _in_use(e) < held
    level = _in_use(e)
    a.close()
    freed_a = level - _in_use(e)
    level = _in_use(e)
    b.close()
    assert freed_a == level - _in_use(e)
    e.close()


def test_apply_updates_while_another_thread_reads_at_snapshots(eng):
    """one thread applies through rsp_apply_updates; another takes snapshots and reads at them; every value equals the
    port's at the snapshot's sequence number"""
    from rocksplicator_b200 import engine
    s = new_shard(eng, engine.MERGE_COUNTER)
    keys, stream = random_stream(4242, 400, n_keys=40, merge="counter")
    lib = eng.lib
    done = threading.Event()
    errors = []

    class Slice(C.Structure):
        _fields_ = [("data", C.c_void_p), ("size", C.c_size_t)]

    def writer():
        try:
            for i in range(0, len(stream), 8):
                part = stream[i:i + 8]
                bufs = [C.create_string_buffer(b, len(b)) for b, _ in part]
                sl = (Slice * len(part))(*[Slice(C.cast(x, C.c_void_p), len(b)) for x, (b, _) in zip(bufs, part)])
                ts = (C.c_uint64 * len(part))(*[t for _, t in part])
                n = C.c_size_t()
                rc = lib.rsp_apply_updates(s.h, len(part), sl, ts, None, None, C.byref(n))
                if rc != 0:
                    errors.append(rc)
        finally:
            done.set()

    seen = []
    t = threading.Thread(target=writer)
    t.start()
    while not done.is_set() or len(seen) < 3:
        with s.snapshot() as snap:
            seen.append((snap.seq, [snap.get(k) for k in keys], snap.multi_get(keys)))
        if done.is_set() and len(seen) >= 3:
            break
    t.join()
    assert not errors
    port = SnapOkv(merge_op=okv.MERGE_COUNTER)
    at = {}
    want_seqs = {q for q, _, _ in seen}
    if 0 in want_seqs:
        at[0] = port.snapshot()
    for bt, ts in stream:
        port.apply(bt, ts)
        q = port.latest_seq()
        if q in want_seqs and q not in at:
            at[q] = port.snapshot()
    for q, gets, mg in seen:
        want = [port.get(k, snapshot=at[q]) for k in keys]
        assert gets == want and mg == want, q
    for p in at.values():
        p.release()
    port.close()
    s.close()


def test_snapshot_seq_is_latest_seq(eng):
    s = new_shard(eng, okv.MERGE_UINT64ADD)
    assert s.apply(WriteBatch().merge(b"c", struct.pack("<Q", 5)).put(b"p", b"q").data(), 1) == 0
    with s.snapshot() as snap:
        assert snap.seq == s.latest_seq() == 2
        assert eng.lib.rsp_snapshot_seq(snap.h) == 2
    s.close()
