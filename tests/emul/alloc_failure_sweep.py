"""Every device and pinned allocation of every maintenance operation made to fail, one at a time, on the emulation.

For each operation the shards are first brought to a seeded state (memtables and several runs, a counter shard, a
string-append shard, an ingested-behind tier, a live snapshot).  Then, for k = 0, 1, 2, ... the (k+1)-th cudaMalloc /
cudaHostAlloc of the call fails (alloc_fail_hook.cpp: emul_fail_alloc_after) until the call gets through without using the
failure.  After every failed attempt: the call answered an IO error (Busy for an apply whose room could not be made),
no device bytes are held that were not held before it, and every shard and the snapshot still read equal to the
oracle port through MultiGet and an iterator.  At the end every shard is closed and the engine destroyed: no device
byte is left.

Run with RSP_EMUL_EXACT_ALLOC=1 (every arena request its own allocation) against the AddressSanitizer build, so that a
block released while still installed shows as a use after free, with alloc_fail_hook.cpp built as a shared library and
preloaded.  Run by tests/test_alloc_failure_emul_cpu.py."""
import ctypes as C
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import numpy as np  # noqa: E402

import string_append_model as SA  # noqa: E402
from oracle import okv  # noqa: E402
from rocksplicator_b200 import engine  # noqa: E402
from rocksplicator_b200.write_batch import WriteBatch  # noqa: E402

assert os.environ.get("RSP_EMUL_EXACT_ALLOC") == "1", "run with RSP_EMUL_EXACT_ALLOC=1"
engine.SO_PATH = os.environ.get("RSP_TEST_EMUL_LIB", os.path.join(HERE, "build_asan", "librsp_b200_emul.so"))
okv.build(ref=False)
port = okv.load_port()
lib = engine.load_library()
hook = C.CDLL(None)  # alloc_fail_hook.cpp, preloaded
hook.emul_fail_alloc_after.argtypes = [C.c_long]
hook.emul_fail_alloc_after.restype = None
hook.emul_fail_alloc_armed.restype = C.c_int
hook.emul_live_device_bytes.restype = C.c_size_t
IO_ERROR, BUSY = 5, 11


def live():
    return hook.emul_live_device_bytes()


def key(p, i):
    return b"%s%06d" % (p, i)


def cnt(v):
    return int(v).to_bytes(8, "little")


class Plain:
    """an okv oracle beside an engine shard"""

    def __init__(self, shard, merge_op=okv.MERGE_NONE):
        self.shard, self.o = shard, okv.Okv(port, merge_op=merge_op)

    def apply(self, batch):
        assert self.o.apply(batch, 0) == 0

    def items(self):
        return self.o.scan()


class StrAppend:
    def __init__(self, shard):
        self.shard, self.m = shard, SA.Model(b",")

    def apply_ops(self, ops):
        self.m.apply(ops)
        return SA.batch_of(ops)

    def items(self):
        return self.m.items()


eng = engine.Engine(0, max_shards=64, arena_bytes=1 << 20, l0_compaction_trigger=64)  # no background merges
sides = {}


def open_side(name, kind=engine.MERGE_NONE, **kw):
    s = eng.open_shard(name, merge_op=kind, **kw)
    side = StrAppend(s) if kind == engine.MERGE_STRING_APPEND else Plain(s, kind)
    sides[name] = side
    return side


def apply(side, batch):
    st = eng.apply_many([side.shard.index], [batch])
    assert st[0] == 0, st
    side.apply(batch)


def puts(side, prefix, lo, hi, tag=b"v"):
    wb = WriteBatch()
    for i in range(lo, hi):
        wb.put(key(prefix, i), tag + b"%d" % i * 3)
    apply(side, wb.data())


# ---- seeded state ----------------------------------------------------------------------------------------------------
P = open_side("plain", write_buffer_bytes=64 << 10)
for r in range(4):  # several runs and a memtable
    puts(P, b"k", r * 40, r * 40 + 60, b"r%d" % r)
    if r < 3:
        assert P.shard.flush() == 0
Cn = open_side("counter", engine.MERGE_COUNTER, write_buffer_bytes=64 << 10)
for r in range(3):
    wb = WriteBatch()
    for i in range(50):
        wb.merge(key(b"c", i % 30), cnt(i + r))
    apply(Cn, wb.data())
    if r < 2:
        assert Cn.shard.flush() == 0
A = open_side("append", engine.MERGE_STRING_APPEND, merge_delim=b",", write_buffer_bytes=64 << 10)
for r in range(3):
    ops = [(SA.MERGE, key(b"a", i % 25), b"x%d" % (i + r)) for i in range(40)] + [(SA.PUT, key(b"a", 90 + r), b"p")]
    st = eng.apply_many([A.shard.index], [A.apply_ops(ops)])
    assert st[0] == 0
    if r < 2:
        assert A.shard.flush() == 0
B1 = open_side("behind1", allow_ingest_behind=True, write_buffer_bytes=64 << 10)  # two behind runs: a third merges them
B2 = open_side("behind2", allow_ingest_behind=True, write_buffer_bytes=64 << 10)
for side in (B1, B2):
    for f in range(2 if side is B1 else 1):
        kv = [(key(b"z%d" % f, i), b"b%d" % i) for i in range(30)]
        assert side.shard.ingest(kv, behind=True) == 0
        for k, v in kv:  # (key ranges of their own: below everything is the same as anywhere)
            side.apply(WriteBatch().put(k, v).data())
    puts(side, b"k", 0, 50)
    assert side.shard.flush() == 0
    puts(side, b"k", 20, 70, b"w")
E = open_side("empty", write_buffer_bytes=4096)  # its memtable is too small for BIG: it is re-sized
BIG = WriteBatch()
for i in range(400):
    BIG.put(key(b"e", i), b"y" * 40)
BIG = BIG.data()
apply(B2, BIG)  # (the tick image buffer grows to BIG's size here)
snap_items = P.items()
snap = P.shard.snapshot()
# warm the engine's scratch buffers, so that only the calls under test grow them (the read combiner's buffers too)
for side in sides.values():
    side.shard.multi_get([b"warm"])
puts(P, b"k", 200, 230)  # the memtable holds data again after the snapshot


def check(where):
    for name, side in sides.items():
        want = side.items()
        got = side.shard.scan()
        assert got == want, (where, name, len(got), len(want))
        keys = [k for k, _ in want] + [b"absent"]
        res = side.shard.multi_get(keys, stride=4096)
        exp = [(0, v) for _, v in want] + [(1, None)]
        assert res == exp, (where, name)
    assert snap.scan() == snap_items, where


check("seeded")


# ---- the operations ----------------------------------------------------------------------------------------------------
def op_shard_open(attempt):
    h = C.c_void_p()
    opts = engine.ShardOpts(merge_op=0, merge_delim=0, write_buffer_bytes=0)
    rc = lib.rsp_shard_open_ex(eng.h, b"opened", C.byref(opts), 0, C.byref(h))
    if rc == 0:
        s = engine.Shard.__new__(engine.Shard)
        s.engine, s.lib, s.kind, s.h, s.name, s._merge_fn = eng, lib, "b200", h, "opened", None
        s.index = lib.rsp_shard_index(h)
        sides["opened"] = Plain(s)
    return rc


def op_apply_grow(attempt):
    st = eng.apply_many([E.shard.index], [BIG])
    if st[0] == 0:
        E.apply(BIG)
        return 0
    assert eng.last_rc in (IO_ERROR, BUSY) and st[0] in (IO_ERROR, BUSY), (eng.last_rc, st)
    return IO_ERROR


def op_flush(attempt):
    return P.shard.flush()


def op_compact(attempt):
    return Cn.shard.compact()


def op_compact_level(attempt):
    return B2.shard.compact(change_level=True)


held = []


def op_snapshot(attempt):
    h = C.c_void_p()
    rc = lib.rsp_snapshot_create(A.shard.h, C.byref(h))
    if rc == 0:
        held.append(("snap", h))
    return rc


def op_iter(attempt):
    h = lib.rsp_iter_create(A.shard.h)
    if not h:
        return IO_ERROR
    lib.rsp_iter_destroy(h)
    return 0


def op_iter_at(attempt):
    h = lib.rsp_iter_create_at(snap.h)
    if not h:
        return IO_ERROR
    lib.rsp_iter_destroy(h)
    return 0


ING = [(key(b"k", i), b"ingested%d" % i) for i in range(10, 300, 3)]


def op_ingest(attempt):
    rc = P.shard.ingest(ING)
    if rc == 0:
        for k, v in ING:
            P.apply(WriteBatch().put(k, v).data())
    return rc


BEH = [(key(b"z9", i), b"late%d" % i) for i in range(40)]


def op_ingest_behind(attempt):
    rc = B1.shard.ingest(BEH, behind=True)
    if rc == 0:
        for k, v in BEH:
            B1.apply(WriteBatch().put(k, v).data())
    return rc


def op_stage_build(attempt):
    batch = WriteBatch().put(b"staged", b"s").data()
    six = np.array([P.shard.index], dtype=np.uint32)
    blob = np.frombuffer(batch + b"\0", dtype=np.uint8)
    off = np.array([0, len(batch)], dtype=np.uint64)
    h = C.c_void_p()
    rc = lib.rsp_stage_build(eng.h, 1, engine._ptr(six), engine._ptr(blob), engine._ptr(off), None, C.byref(h))
    if rc == 0:
        lib.rsp_stage_free(h)
    return rc


def op_multi_get(attempt):
    # a value stride beyond 1 MiB skips the read combiner: the direct path's query buffer grows to hold it
    try:
        res = eng.multi_get([P.shard.index] * 3, [key(b"k", 1), key(b"k", 2), b"absent"], stride=(1 << 20) + 4096)
    except RuntimeError as ex:
        assert str(ex).endswith("-> %d" % IO_ERROR), ex
        return IO_ERROR
    assert [r[0] for r in res] == [0, 0, 1]
    return 0


def op_scan(attempt):
    try:
        res = eng.multi_scan([Cn.shard.index] * 2, [key(b"c", 0), key(b"c", 10)], 8, 3 << 20)
    except RuntimeError as ex:
        assert str(ex).endswith("-> %d" % IO_ERROR), ex
        return IO_ERROR
    assert res[0][1] == Cn.items()[:8]
    return 0


# scratch: the call's only device memory is the engine's growable query buffers, which a failed growth leaves empty
# (all or nothing) and a later attempt may grow again, so their bytes are not compared
OPS = [("rsp_shard_open", op_shard_open, False), ("apply growing an empty memtable", op_apply_grow, False),
       ("rsp_flush", op_flush, False), ("rsp_compact", op_compact, False),
       ("rsp_compact_ex(CHANGE_LEVEL)", op_compact_level, False), ("rsp_snapshot_create", op_snapshot, False),
       ("rsp_iter_create", op_iter, False), ("rsp_iter_create_at", op_iter_at, False),
       ("rsp_ingest_sorted", op_ingest, False), ("rsp_ingest_sorted_behind", op_ingest_behind, False),
       ("rsp_stage_build", op_stage_build, False), ("host MultiGet", op_multi_get, True),
       ("host scan", op_scan, True)]

bad = []
for name, op, scratch in OPS:
    k = 0
    while True:
        runs = [side.shard.stats()["n_runs"] for side in sides.values()]
        before = live()
        hook.emul_fail_alloc_after(k)
        rc = op(k)
        used = not hook.emul_fail_alloc_armed()
        hook.emul_fail_alloc_after(-1)
        after = live()
        if rc == 0:
            check("%s: success after %d failure points" % (name, k))
            print("%-34s ok after %d failure points%s" % (name, k, "" if not used else " (the last failure was absorbed)"))
            break
        if rc not in (IO_ERROR, BUSY):
            bad.append("%s k=%d: rc %d" % (name, k, rc))
        # a run list that changed: a flush or merge the call needed first (rsp_ingest_sorted_behind merges the tier before
        # it builds the new run) completed before the failure, and its memory is that of a different run set
        stepped = runs != [side.shard.stats()["n_runs"] for side in sides.values()]
        if after != before and not scratch and not stepped:
            bad.append("%s k=%d: live device bytes %d -> %d" % (name, k, before, after))
        try:
            check("%s k=%d" % (name, k))
        except AssertionError as ex:
            bad.append("%s k=%d: contents: %s" % (name, k, ex))
            break
        k += 1
        if k > 400:
            bad.append("%s: never succeeded" % name)
            break

for _, h in held:
    lib.rsp_snapshot_release(h)
snap.release()
for side in sides.values():
    side.shard.close()
eng.close()
if live() != 0:
    bad.append("%d device bytes left after the engine was destroyed" % live())
for b in bad:
    print("FAIL", b)
print("ALLOC FAILURE SWEEP %s" % ("OK" if not bad else "FAILED (%d)" % len(bad)))
sys.exit(1 if bad else 0)
