"""GPU: the packed apply tick at full memtables, and the flushes the apply path triggers, against the oracle port.

A tick of >= 1024 batches already grouped by shard (the packed tick, rsp_apply_many) reserves memtable room from an
ESTIMATE, without a sizing round trip: per shard, `ents = nb + bytes / 256` entries and `bytes / 16 + 2 * ents + 1` heap
units.  Batches of several small ops cost more than that.  The fused tick kernels (k_tick_fused<64>, k_tick_fused<128>,
k_tick_chunks) then refuse the first batch that does not fit, and every later batch of its shard, with Busy and no
latch; the host retries the refused batches in order through the host-staged tick, which reserves exact bounds (and so
flushes, or re-sizes, the full memtable first).  The caller must see what a serial replay gives: statuses, sequence
numbers, contents.

Each case here is built with a few lines that restate the engine's arithmetic (the memtable of a fresh shard, the
true cost of a batch, the packed estimate, the fused kernels' chunks), so that the case PREDICTS which batch of which
shard the guard refuses and which kernel runs the tick — and then proves it from what the retry leaves behind: one more
flush, the flushed memtable holding the accepted prefix (compaction_bytes_read), the memtable holding the retried
suffix.  A case whose precondition does not hold fails instead of passing untested.

The flushes: a staged tick whose bound does not fit flushes every such shard in one batched pass (k_flush_sort, the LSD
radix sort over the V varying bits of the 8-byte key prefixes, for V <= 48 and at most FS_MAX_ITEMS entries; the bitonic
k_compact_sort for the rest).  One tick flushes shards on both sides of every selection boundary at once."""
import os
import random
import struct

import pytest

from oracle import okv
from rocksplicator_b200.write_batch import WriteBatch, varint32

pytestmark = pytest.mark.gpu
EMUL = bool(os.environ.get("RSP_TEST_EMUL_LIB"))

# ---- the engine's constants (kernels.h, k_compact.cu, include/rsp_b200.h)
DEVICE_SMS = 132
FUSED_MAX_BATCH_BYTES = 16384
FS_MAX_ITEMS = 24576
BUSY = 11  # RSP_BUSY: what the guard answers; never a final status
TRAILER = 10  # the follower's LogData(timestamp) record: tag, length 8, 8 bytes
N_FILLERS = 4 * DEVICE_SMS + 12


# ------------------------------------------------------------------------------------------------------------
# the mirror
# ------------------------------------------------------------------------------------------------------------
def next_pow2(x):
    p = 1
    while p < x:
        p <<= 1
    return p


def memtable_caps(write_buffer_bytes):
    """(heap units, entries, slots) of a shard's memtable as alloc_memtable(e, s, 0, 0) sizes it at open"""
    heap = (write_buffer_bytes or (1 << 20)) // 16
    ents = heap // 7
    return heap, ents, next_pow2(max(16, 2 * ents))


def units_of(n):
    return (n + 15) >> 4


def _varint(b, p):
    v = shift = 0
    while True:
        c = b[p]
        p += 1
        v |= (c & 127) << shift
        shift += 7
        if c < 128:
            return v, p


def cost(batch, ts):
    """(heap units, entries) a well-formed batch takes in the memtable: 2 + units_of(klen) + units_of(vlen) per data
    record (format.cuh entry_units), walked over the batch and the LogData(ts) record appended when ts is given"""
    b = batch + (b"\x03\x08" + struct.pack("<Q", ts) if ts is not None else b"")
    p, units, ents = 12, 0, 0
    while p < len(b):
        tag = b[p]
        p += 1
        if tag == 0x0D:  # Noop
            continue
        klen, p = _varint(b, p)
        p += klen
        if tag == 0x03:  # LogData: no entry
            continue
        vlen = 0
        if tag in (0x01, 0x02):
            vlen, p = _varint(b, p)
            p += vlen
        else:
            assert tag == 0x00, tag
        assert p <= len(b)
        units += 2 + units_of(klen) + units_of(vlen)
        ents += 1
    return units, ents


def packed_estimate(batches, ts_on):
    """what apply_many_packed reserves for one shard's group: (heap units, entries)"""
    nbytes = sum(len(b) for b in batches) + len(batches) * (TRAILER if ts_on else 0)
    ents = len(batches) + nbytes // 256
    return nbytes // 16 + 2 * ents + 1, ents


def staged_bound(batch, ts_on):
    """what stage_build reserves for one batch: (heap units, entries)"""
    len_eff = len(batch) + (TRAILER if ts_on else 0)
    claimed = struct.unpack_from("<I", batch, 8)[0]
    cap = min(claimed, (len_eff - 12) // 2)
    return cap * 4 + len_eff // 16 + 1, cap


def packed_builder(groups, ts_on):
    """the kernel that runs a packed tick of these groups (launch_tick_fused)"""
    trailer = TRAILER if ts_on else 0
    max_len = max(len(b) for g in groups for b in g)
    assert sum(len(g) for g in groups) >= 1024 and max_len + trailer <= FUSED_MAX_BATCH_BYTES, "not a packed tick"
    if max(len(g) for g in groups) <= 64 and max_len + trailer + 16 <= 4096:
        return "fused64"
    force = tick_chunks_override()
    if force is not None:
        return "chunks" if force else "fused128"
    return "fused128" if len(groups) >= 4 * DEVICE_SMS else "chunks"


def tick_chunks_override():
    """RSP_TICK_CHUNKS (read once by the library): 1 sends every long-group tick to k_tick_chunks, 0 to
    k_tick_fused<128>; None when unset and the number of groups decides"""
    v = os.environ.get("RSP_TICK_CHUNKS")
    if v is None:
        return None
    try:
        return int(v) != 0
    except ValueError:
        return False  # (atoi of a non-number is 0)


CHUNK_SHAPE = {"fused64": (64, 8192), "fused128": (128, 16384), "chunks": (128, 16384)}


def chunk_starts(batches, builder):
    """first batch of every chunk of a group: at most `max_batches` batches and `stage` bytes of the caller's blob (the
    host's cut_chunks for k_tick_chunks, the stage loop of k_tick_fused)"""
    max_batches, stage = CHUNK_SHAPE[builder]
    off = [0]
    for b in batches:
        off.append(off[-1] + len(b))
    starts, b = [], 0
    while b < len(batches):
        starts.append(b)
        e = b + 1
        while e < len(batches) and e - b < max_batches and off[e + 1] - off[b] <= stage:
            e += 1
        b = e
    return starts


def walk(batches, bad, ts, heap_cap, ent_cap, tail=0, cnt=0, latched=False):
    """the fused kernels' walk of one group, then the staged retry: which batch the guard refuses, which cap binds, the
    accepted prefix and the retried suffix that is applied (both (units, entries)), the first corrupt batch"""
    r = {"refused": None, "binds": None, "bad": None, "prefix": (0, 0), "suffix": (0, 0)}
    if latched:
        return r
    u = e = 0
    for i, b in enumerate(batches):
        if bad[i]:
            r["bad"] = i
            break
        cu, ce = cost(b, ts[i])
        if tail + u + cu > heap_cap or cnt + e + ce > ent_cap:
            r["refused"] = i
            r["binds"] = "heap" if tail + u + cu > heap_cap else "ents"
            break
        u += cu
        e += ce
    r["prefix"] = (u, e)
    if r["refused"] is not None:
        su = se = 0
        for i in range(r["refused"], len(batches)):
            if bad[i]:
                r["bad"] = i
                break
            cu, ce = cost(batches[i], ts[i])
            su += cu
            se += ce
        r["suffix"] = (su, se)
    return r


def wrong_count(batch):
    """the same records under a header that claims one more: Corruption, 'WriteBatch has wrong count'"""
    return batch[:8] + struct.pack("<I", struct.unpack_from("<I", batch, 8)[0] + 1) + batch[12:]


# ------------------------------------------------------------------------------------------------------------
# batches
# ------------------------------------------------------------------------------------------------------------
def key17(tag, i):
    return (b"%s-%d" % (tag, i)).ljust(17, b".")[:17]


def wide_batch(tag, b, n_keys=7, ops=6, merge=False, wide_first=False):
    """ops records with 17-byte keys and 65-byte values (9 heap units each): more than the 7 units per entry that the
    entry cap assumes, about 0.7 of the packed estimate"""
    wb = WriteBatch()
    for j in range(ops):
        k = key17(tag, (b * ops + j) % n_keys)
        v = ((b"%s.%d.%d|" % (tag, b, j)) * 12)[:81 if (wide_first and j == 0) else 65]
        wb.merge(k, v) if merge else wb.put(k, v)
    return wb.data()


def tiny_batch(tag, b, ops=8):
    """ops Deletes or Puts (alternating batches) of 1-byte keys: 3 or 4 heap units per record, about one entry per
    batch in the packed estimate"""
    wb = WriteBatch()
    for j in range(ops):
        k = bytes([0x61 + (b * ops + j) % 13])
        wb.delete(k) if b % 2 else wb.put(k, bytes([b & 0xFF]))
    return wb.data()


def small_put(tag, b, n_keys=7):
    return WriteBatch().put(key17(tag, b % n_keys), b"s%d" % b).data()


def counter_batch(tag, b):
    wb = WriteBatch()
    for j in range(6):
        k = key17(tag, (b + j) % 3)
        if (b * 6 + j) % 11 == 0:
            wb.put(k, struct.pack("<q", 1000 * b + j))
        else:
            wb.merge(k, struct.pack("<q", (b * 6 + j) * 7 - 100))
    return wb.data()


SWALLOW_TS = int.from_bytes(bytes([0x41] + [0x0D] * 7), "little")


def swallow_batch():
    """one Put whose value claims 3 more bytes than the batch holds: it legally swallows the first three bytes of the
    follower's LogData record (0x03, 0x08 and the timestamp's low byte); the other seven bytes of SWALLOW_TS parse as
    Noop tags"""
    v = b"tail-swallows-"
    return bytes(8) + struct.pack("<I", 1) + b"\x01" + varint32(3) + b"swk" + varint32(len(v) + 3) + v


# ------------------------------------------------------------------------------------------------------------
# fixtures
# ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng():
    from rocksplicator_b200 import engine
    e = engine.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def fillers(eng):
    """shards that take single-Put batches that fit: they make up the tick's 1024 batches, and the 4 groups per SM that
    send long groups to k_tick_fused<128>"""
    shards = [eng.open_shard("capfill%04d" % i, write_buffer_bytes=64 << 10) for i in range(N_FILLERS)]
    yield shards
    for s in shards:
        s.close()


_n = [0]


class Case:
    """one shard of a tick, its oracle, its batches and what the mirror predicts for them"""

    def __init__(self, name, batches, heap_cap, merge_op=okv.MERGE_NONE, bad=None, prefill=(), latched=False,
                 expect=None):
        self.name = name
        self.batches = batches
        self.bad = bad or [False] * len(batches)
        self.heap_cap = heap_cap
        self.merge_op = merge_op
        self.prefill = list(prefill)  # (batch, corrupt) applied by an earlier staged tick
        self.latched = latched
        self.expect = expect or {}

    def open(self, eng, port_lib):
        _n[0] += 1
        self.s = eng.open_shard("cap%05d" % _n[0], merge_op=self.merge_op, write_buffer_bytes=16 * self.heap_cap)
        self.o = okv.Okv(port_lib, merge_op=self.merge_op)
        return self

    def close(self):
        self.s.close()
        self.o.close()


def fit_cap(batches, ts_on, tail=0, cnt=0):
    """the smallest memtable (heap units) the packed estimate of these batches fits, after tail / cnt"""
    eu, ee = packed_estimate(batches, ts_on)
    return max(tail + eu, 7 * (cnt + ee))


def cap_at(batches, ts, k, extra):
    """heap units that end the true prefix of batches [0, k) `extra` units into batch k"""
    return sum(cost(b, t)[0] for b, t in zip(batches[:k], ts[:k])) + extra


def build_cases(builder, ts_on):
    """the scenarios of one tick, each on its own shard; L batches per group (longer than 64 and than one chunk for
    the builders of long groups)"""
    L = 64 if builder == "fused64" else 160
    T = (lambda n: [7] * n) if ts_on else (lambda n: [None] * n)
    cases = []

    # the entry cap binds: 8 records of 3-4 units per batch, about one entry per batch in the estimate.  The retried
    # suffix is several memtables long: the staged retry flushes AND re-sizes.
    bs = [tiny_batch(b"ent", b) for b in range(L)]
    cases.append(Case("entries", bs, fit_cap(bs, ts_on), expect={"binds": "ents", "resize": True}))

    # the heap cap binds, the refused batch inside a chunk (not its first batch); with a timestamp, the group's last
    # batch (in the retried suffix) swallows the first bytes of its LogData record
    bs = [wide_batch(b"heap", b) for b in range(L)]
    if ts_on:
        bs[-1] = swallow_batch()
    ts = T(L)
    if ts_on:
        ts[-1] = SWALLOW_TS
    cap = fit_cap(bs, ts_on)
    starts = chunk_starts(bs, builder)
    while walk(bs, [False] * L, ts, cap, cap // 7)["refused"] in starts:
        cap += 1
    cases.append(Case("heap", bs, cap, expect={"binds": "heap", "inside_chunk": True, "swallow": ts_on}))

    # exactly at the heap cap (batch k accepted with tail + units == heap_cap), and one unit over (batch k refused)
    bs = [wide_batch(b"exh", b) for b in range(L)]
    k = next(k for k in range(1, L - 1) if cap_at(bs, T(L), k + 1, 0) >= fit_cap(bs, ts_on))
    cap = cap_at(bs, T(L), k + 1, 0)
    cases.append(Case("exact_heap", bs, cap, expect={"refused": k + 1, "binds": "heap", "prefix_units": cap}))
    bs = list(bs)
    bs[k] = wide_batch(b"exh", k, wide_first=True)  # 55 units instead of 54
    cases.append(Case("over_heap", bs, cap, expect={"refused": k, "binds": "heap"}))

    # exactly at the entry cap, and one entry over
    bs = [tiny_batch(b"exe", 2 * b + 1) for b in range(L)]  # 8 Deletes each: 8 entries, 24 units
    k = next(k for k in range(1, L - 1) if 7 * 8 * (k + 1) >= fit_cap(bs, ts_on))
    cases.append(Case("exact_ents", bs, 7 * 8 * (k + 1), expect={"refused": k + 1, "binds": "ents",
                                                                  "prefix_ents": 8 * (k + 1)}))
    bs = list(bs)
    bs[k] = tiny_batch(b"exe", 2 * k + 1, ops=9)
    cases.append(Case("over_ents", bs, 7 * 8 * (k + 1), expect={"refused": k, "binds": "ents"}))

    # the first batch of its group: an earlier tick left the memtable nearly full; the estimate of the group fits the
    # rest, its first batch (8 Deletes: 24 units, 8 entries) does not
    bs = [tiny_batch(b"fog", 1)] + [small_put(b"fog", b) for b in range(3)]
    eu, _ = packed_estimate(bs, ts_on)
    cap = 1024
    room = eu + 2
    big = WriteBatch().put(b"fog-big", bytes(16 * (cap - room - 3))).data()  # 3 + units_of(vlen) = cap - room
    assert cost(big, 0)[0] == cap - room
    cases.append(Case("first_of_group", bs, cap, prefill=[(big, False)], expect={"refused": 0}))

    # the first batch of a later chunk: the stop must cross from one chunk to the next (k_tick_chunks: CHAIN_STOP in
    # the chain record); small batches in the later chunks would fit what is left, so a chunk that did not see the
    # stop would apply them ahead of the refused batch
    if builder == "fused64":
        bs = [small_put(b"chs", b) if b % 4 == 3 else wide_batch(b"chs", b) for b in range(L)]
    else:
        bs = [wide_batch(b"chs", b) for b in range(100)] + [small_put(b"chs", b) for b in range(100, 300)]
    n = len(bs)
    starts = chunk_starts(bs, builder)
    cap = None
    for cs in starts[1:]:
        c = cap_at(bs, T(n), cs, cost(bs[cs], T(1)[0])[0] - 1)
        if cs + 2 < n and c >= fit_cap(bs, ts_on) and walk(bs, [False] * n, T(n), c, c // 7)["refused"] == cs:
            cap = c
            break
    assert cap is not None, "no chunk start where the estimate fits and the true cost does not"
    cases.append(Case("chunk_start", bs, cap, expect={"refused": cs, "chunk_start": True,
                                                      "later_chunk": builder != "fused64"}))

    # corrupt batches before and after the refused one
    bs = [wide_batch(b"cbf", b) for b in range(L)]
    cap = fit_cap(bs, ts_on)
    r = walk(bs, [False] * L, T(L), cap, cap // 7)["refused"]
    assert r is not None and r >= 3 and r + 3 < L
    bad = [False] * L
    bad[r - 3] = True
    cases.append(Case("corrupt_before", [wrong_count(b) if x else b for b, x in zip(bs, bad)], cap, bad=bad,
                      expect={"refused": None, "bad": r - 3, "would_refuse": r}))
    bad = [False] * L
    bad[r + 3] = True
    cases.append(Case("corrupt_after", [wrong_count(b) if x else b for b, x in zip(bs, bad)], cap, bad=bad,
                      expect={"refused": r, "bad": r + 3}))

    # a shard latched by an earlier tick: its batches answer the latch, nothing is refused or retried
    bs = [wide_batch(b"lat", b) for b in range(L)]
    cap = fit_cap(bs, ts_on, *cost(small_put(b"lat", 0), 0))
    pre = [(small_put(b"lat", 0), False), (wrong_count(small_put(b"lat", 1)), True)]
    cases.append(Case("latched", bs, cap, prefill=pre, latched=True, expect={"refused": None, "would_refuse": True}))

    # order-sensitive operands: the append operator (folded on the host) and the counter, one key's operands on both
    # sides of the refused batch
    bs = [wide_batch(b"app", b, n_keys=3, merge=True) for b in range(L)]
    cases.append(Case("append", bs, fit_cap(bs, ts_on), merge_op=okv.MERGE_APPEND, expect={"straddle": True}))
    bs = [counter_batch(b"ctr", b) for b in range(L)]
    cases.append(Case("counter", bs, fit_cap(bs, ts_on), merge_op=okv.MERGE_COUNTER, expect={"straddle": True}))

    # the last batch of the tick (this group is the tick's last)
    bs = [wide_batch(b"lst", b) for b in range(L)]
    cap = cap_at(bs, T(L), L - 1, 1)
    cases.append(Case("last_of_tick", bs, cap, expect={"refused": L - 1, "last": True}))
    return cases


@pytest.mark.parametrize("ts_on", [True, False], ids=["ts", "no_ts"])
@pytest.mark.parametrize("builder", ["fused64", "fused128", "chunks"])
def test_capacity_guard_and_retry(eng, fillers, port_lib, builder, ts_on):
    """Every scenario of the capacity guard in ONE packed tick per builder: the entry cap, the heap cap, exactly at
    either cap and one over, the refused batch first in its group / inside a chunk / first in a later chunk / last in
    the tick, corrupt batches before and after it, a shard latched earlier, append and counter operands around it, a
    retried suffix larger than a memtable, and (ts) a batch that swallows part of its LogData record in the retried
    suffix.  Statuses, sequence numbers, Get / MultiGet / scan against the oracle replaying the batches one by one."""
    force = tick_chunks_override()
    if builder != "fused64" and force is not None and force != (builder == "chunks"):
        pytest.skip("RSP_TICK_CHUNKS=%s sends every long-group tick to the other kernel" % os.environ["RSP_TICK_CHUNKS"])
    cases = build_cases(builder, ts_on)
    for c in cases:
        c.open(eng, port_lib)
    try:
        # ---- the earlier tick (staged: < 1024 batches): memtables left nearly full, a shard latched
        pre = [(c, b) for c in cases for b, _ in c.prefill]
        if pre:
            pts = [3] * len(pre) if ts_on else None
            st = eng.apply_many([c.s.index for c, _ in pre], [b for _, b in pre], pts)
            assert list(st) == [c.o.apply(b, 3) for c, b in pre]
            for c in cases:
                for b, corrupt in c.prefill:
                    hu, he = staged_bound(b, ts_on)
                    assert corrupt or (hu <= c.heap_cap and he <= c.heap_cap // 7), (c.name, "prefill re-sized")
                assert c.s.stats()["flushes"] == 0
        # ---- the packed tick
        base_ts = 1000
        six, batches, ts, owner = [], [], [], []
        n_case = sum(len(c.batches) for c in cases)
        if builder == "fused64":
            fill_groups = [(fillers[i], 64) for i in range(max(0, -(-(1024 - n_case) // 64)) + 1)]
        elif builder == "fused128":
            fill_groups = [(f, 1) for f in fillers]
        else:
            fill_groups = [(fillers[i], 100) for i in range(2)]
        fill_pos = []
        for f, m in fill_groups:
            for i in range(m):
                fill_pos.append(len(batches))
                six.append(f.index)
                batches.append(WriteBatch().put(b"fill%05d" % i, b"%d" % len(batches)).data())
                ts.append(base_ts + len(ts))
                owner.append(None)
        case_ts = {}
        for c in cases:
            cts = []
            for i, b in enumerate(c.batches):
                t = base_ts + len(ts)
                if c.name == "heap" and ts_on and i == len(c.batches) - 1:
                    t = SWALLOW_TS
                cts.append(t)
                six.append(c.s.index)
                batches.append(b)
                ts.append(t)
                owner.append(c)
            case_ts[c.name] = cts
        groups = []
        for i, ix in enumerate(six):
            if i == 0 or ix != six[i - 1]:
                groups.append([])
            groups[-1].append(batches[i])
        assert len(groups) == len(fill_groups) + len(cases)
        assert packed_builder(groups, ts_on) == builder
        # ---- what the mirror predicts, and the preconditions that make it a test of the guard
        before, pred = {}, {}
        for c in cases:
            st = c.s.stats()
            before[c.name] = st
            tail, cnt = st["memtable_bytes"] // 16, st["memtable_entries"]
            heap_cap, ent_cap, slots = memtable_caps(16 * c.heap_cap)
            eu, ee = packed_estimate(c.batches, ts_on)
            assert tail + eu <= heap_cap and cnt + ee <= ent_cap and 2 * (cnt + ee) <= slots, \
                (c.name, "the estimate must fit the memtable, or the tick flushes before the kernel runs")
            cts = case_ts[c.name] if ts_on else [None] * len(c.batches)
            p = walk(c.batches, c.bad, cts, heap_cap, ent_cap, tail, cnt, c.latched)
            pred[c.name] = p
            x = c.expect
            unlatched = walk(c.batches, c.bad, cts, heap_cap, ent_cap, tail, cnt)
            truth = walk(c.batches, [False] * len(c.batches), cts, heap_cap, ent_cap, tail, cnt)
            assert truth["refused"] is not None, (c.name, "the true cost fits: the guard would not fire")
            if "refused" in x:
                assert p["refused"] == x["refused"], (c.name, p)
            else:
                assert p["refused"] is not None, (c.name, p)
            if "binds" in x:
                assert p["binds"] == x["binds"], (c.name, p)
            if "bad" in x:
                assert p["bad"] == x["bad"], (c.name, p)
            if x.get("would_refuse") is not None:
                assert truth["refused"] is not None and (x["would_refuse"] is True or
                                                         truth["refused"] == x["would_refuse"]), (c.name, truth)
            if c.latched:
                assert unlatched["refused"] is not None
            if "prefix_units" in x:
                assert tail + p["prefix"][0] == x["prefix_units"] == heap_cap, (c.name, p)
            if "prefix_ents" in x:
                assert cnt + p["prefix"][1] == x["prefix_ents"] == ent_cap, (c.name, p)
            starts = chunk_starts(c.batches, builder)
            if x.get("inside_chunk"):
                assert p["refused"] not in starts, (c.name, p, starts)
            if x.get("chunk_start"):
                assert p["refused"] in starts[1:], (c.name, p, starts)
            if x.get("later_chunk"):
                # a later chunk holds batches that would fit what the refused one left: only the stop refuses them
                nxt = [s for s in starts if s > p["refused"]]
                room = heap_cap - tail - p["prefix"][0]
                assert nxt and any(cost(b, 0)[0] <= room for b in c.batches[nxt[0]:]), (c.name, starts)
            if x.get("resize"):
                assert p["suffix"][1] > ent_cap, (c.name, "the retried suffix should outgrow a whole memtable")
            if x.get("swallow"):
                assert p["refused"] < len(c.batches) - 1, (c.name, "the swallowing batch must be retried")
            if x.get("straddle"):
                r = p["refused"]
                assert 0 < r < len(c.batches) - 1
        assert cases[-1].expect.get("last") and pred[cases[-1].name]["refused"] == len(cases[-1].batches) - 1
        # ---- the tick, and the serial replay
        st = eng.apply_many(six, batches, ts if ts_on else None)
        # (the oracle always appends the LogData(timestamp) record; without ts the engine appends none, the leader's
        # rsp_write semantics.  No batch of the no_ts cases reads into that record, so the serial replay is the same.)
        want = [0 if c is None else c.o.apply(b, t) for c, b, t in zip(owner, batches, ts)]
        assert [int(x) for x in st] == want
        assert all(int(st[i]) == 0 for i in fill_pos)
        assert BUSY not in want
        # ---- what the retry left behind proves where the guard stopped
        for c in cases:
            p, b0, a = pred[c.name], before[c.name], c.s.stats()
            tail0 = b0["memtable_bytes"] // 16
            cnt0 = b0["memtable_entries"]
            if p["refused"] is not None:
                assert a["flushes"] == b0["flushes"] + 1, (c.name, "the staged retry flushes the full memtable")
                assert a["compaction_bytes_read"] - b0["compaction_bytes_read"] == 16 * (tail0 + p["prefix"][0]), \
                    (c.name, "the flushed memtable holds the accepted prefix")
                assert (a["memtable_bytes"] // 16, a["memtable_entries"]) == p["suffix"], (c.name, p)
                assert a["memtable_bytes"] % 16 == 0
            else:
                assert a["flushes"] == b0["flushes"], c.name
                assert (a["memtable_bytes"] // 16, a["memtable_entries"]) == (tail0 + p["prefix"][0],
                                                                              cnt0 + p["prefix"][1]), (c.name, p)
            assert c.s.latest_seq() == c.o.latest_seq(), c.name
            if p["bad"] is not None or c.latched:
                assert c.s.last_error == c.o.last_error != "", c.name
            keys = sorted({k for k, _ in c.o.scan()} | {key17(t, i) for t in (b"heap", b"app", b"ctr", b"lat")
                                                         for i in range(7)} | {b"swk", b"zz-missing"})
            assert c.s.multi_get(keys, stride=512) == c.o.multi_get(keys), c.name
            assert [c.s.get(k) for k in keys[:12]] == [c.o.get(k) for k in keys[:12]], c.name
            assert c.s.scan() == c.o.scan(), c.name
        if ts_on:
            h = next(c for c in cases if c.name == "heap")
            assert h.s.get(b"swk") == h.o.get(b"swk") == (0, b"tail-swallows-" + bytes([0x03, 0x08, 0x41]))
    finally:
        for c in cases:
            c.close()


# ------------------------------------------------------------------------------------------------------------
# the flushes the apply path triggers: k_flush_sort or k_compact_sort, chosen per shard in one batched pass
# ------------------------------------------------------------------------------------------------------------
def prefix_of(k):
    return int.from_bytes(k[:8].ljust(8, b"\0"), "big")


def sort_selection(keys):
    """(path, V) of k_flush_sort's choice for a memtable of these entries: "size" (more than FS_MAX_ITEMS entries) and
    "bits" (prefixes varying in more than 48 bits: they would not fit beside the 16-bit rank) leave it to the comparison
    sort before the radix sort runs; the radix sort hands it over afterwards when distinct keys share their 8-byte
    prefix ("shared"); "radix" otherwise"""
    pre = [prefix_of(k) for k in keys]
    v = (min(pre) ^ max(pre)).bit_length()
    if len(keys) > FS_MAX_ITEMS:
        return "size", v
    if v > 48:
        return "bits", v
    owner = {}
    for k, p in zip(keys, pre):
        if owner.setdefault(p, k) != k:
            return "shared", v
    return "radix", v


HIGH = 0x6B << 56  # b"k": the prefixes' high bits, zero below bit 56


def v_keys(rng, v, n):
    """n keys of 8 bytes (plus a few versions of hot keys) whose prefixes vary in exactly their low v bits"""
    lo, hi = HIGH, HIGH | ((1 << v) - 1)
    distinct = min(n // 2, 1 << v)
    pool = {lo, hi}
    while len(pool) < distinct:
        pool.add(HIGH | rng.getrandbits(v))
    pool = [struct.pack(">Q", p) for p in sorted(pool)]
    hot = pool[:4]
    keys = list(pool) + [rng.choice(hot) if rng.random() < 0.5 else rng.choice(pool) for _ in range(n - len(pool))]
    rng.shuffle(keys)
    return keys


def flush_shapes(rng):
    """(name, keys written in order: one entry each, the selection's path, V or None) — both sides of every selection"""
    shapes = []
    small = 600 if EMUL else 3000
    for v in (1, 8, 9, 16, 17, 40, 47, 48, 49):
        shapes.append(("V%d" % v, v_keys(rng, v, small), "radix" if v <= 48 else "bits", v))
    shapes.append(("radix_max_items", v_keys(rng, 48, FS_MAX_ITEMS), "radix", 48))
    shapes.append(("radix_max_items_plus_1", v_keys(rng, 48, FS_MAX_ITEMS + 1), "size", 48))
    for n in (4096, 4097, 8192, 8193):  # the bitonic sort's tile, and its global-memory phase
        shapes.append(("bitonic_%d" % n, [b"user_profile_%06d" % rng.randrange(n // 2) for _ in range(n)], "shared", 0))
    # one key's versions spread across the whole memtable: the rank alone orders them
    one = struct.pack(">Q", HIGH | 0x5A5A)
    shapes.append(("versions", [one if i % 3 == 0 else struct.pack(">Q", HIGH | rng.getrandbits(20))
                                for i in range(FS_MAX_ITEMS - 7)], "radix", None))
    # keys shorter than 8 bytes beside the empty key (prefix 0), their first two bytes zero so that the prefixes vary in
    # 47 bits and the radix sort runs: distinct prefixes (radix) ...
    shorts = sorted({b"\0\0" + bytes([rng.randrange(97, 123) for _ in range(rng.randrange(1, 6))]) for _ in range(small)})
    shapes.append(("short_keys", [b""] + shorts + [rng.choice(shorts + [b""]) for _ in range(small // 4)], "radix", 47))
    # ... and beside their zero-extended forms, the empty key beside b"\0" and b"\0\0": equal prefixes of keys of
    # different lengths, which the radix sort must find and hand to the comparison sort
    ext = [k + b"\0" * rng.randrange(1, 9 - len(k)) for k in shorts[::3]]
    mixed = [b"", b"\0", b"\0\0"] + shorts + ext
    rng.shuffle(mixed)
    shapes.append(("short_and_zero_extended", mixed + [rng.choice(mixed) for _ in range(small // 4)], "shared", 47))
    return shapes


def test_flush_sort_selection_at_its_boundaries(eng, port_lib):
    """Memtables filled to exactly their entry cap by staged ticks, then ONE staged tick that writes one more entry to
    each: it flushes all of them in one batched pass whose jobs sit on both sides of every selection boundary — V = 1,
    8, 9, 16, 17, 40, 47, 48 (radix, both parities of ceil(V / 8), six passes at 48) and 49 (comparison sort), 24 576
    and 24 577 entries, 4 096 / 4 097 and 8 192 / 8 193 entries of shared prefixes (the bitonic tile and its
    global-memory phase), one key's versions across a 24 569-entry memtable, keys shorter than 8 bytes beside the empty
    key (47 varying bits: the radix sort runs) with and without their zero-extended forms.  Each shape is asserted to
    take the path it is named for; flush_comparison_sorts per shard as the selection predicts; scan / MultiGet / Get
    against the oracle."""
    rng = random.Random(2468)
    shapes = flush_shapes(rng)
    shards = []
    try:
        six, batches = [], []
        for name, keys, path, v in shapes:
            got = sort_selection(keys)
            assert got[0] == path and (v is None or got[1] == v), (name, "the shape must take the path it is named for", got)
            n = len(keys)
            s = eng.open_shard("capflush-%s" % name, write_buffer_bytes=16 * 7 * n)  # entry cap == n
            o = okv.Okv(port_lib)
            assert memtable_caps(16 * 7 * n)[1] == n
            shards.append((name, keys, s, o))
            wb, bound = WriteBatch(), [0, 0]
            for i, k in enumerate(keys):
                if i % 5 == 4:
                    wb.delete(k)
                else:
                    wb.put(k, b"%s:%d" % (name.encode()[:6], i))
                if wb.count() == 700 or i == n - 1:
                    b = wb.data()
                    six.append(s.index)
                    batches.append(b)
                    hu, he = staged_bound(b, True)
                    bound[0] += hu
                    bound[1] += he
                    wb = WriteBatch()
            heap, ents, _ = memtable_caps(16 * 7 * n)
            assert bound[0] <= heap and bound[1] <= ents, (name, "the fill must not re-size the memtable")
        # the fill: staged (< 1024 batches, or batches beyond 16 KB)
        for lo in range(0, len(six), 1000):
            st = eng.apply_many(six[lo:lo + 1000], batches[lo:lo + 1000], [5] * len(six[lo:lo + 1000]))
            assert not st.any(), st
        by_ix = {s.index: o for _, _, s, o in shards}
        for ix, b in zip(six, batches):
            assert by_ix[ix].apply(b, 5) == 0
        for name, keys, s, o in shards:
            st = s.stats()
            assert (st["memtable_entries"], st["flushes"]) == (len(keys), 0), name
        # the tick that flushes them all at once
        after = [WriteBatch().put(b"\xff-after", name.encode()).data() for name, _, _, _ in shards]
        st = eng.apply_many([s.index for _, _, s, _ in shards], after, [6] * len(shards))
        assert not st.any(), st
        for (name, keys, s, o), b in zip(shards, after):
            assert o.apply(b, 6) == 0
            path, v = sort_selection(keys)
            stt = s.stats()
            assert stt["flushes"] == 1 and stt["memtable_entries"] == 1, name
            assert stt["flush_comparison_sorts"] == (0 if path == "radix" else 1), (name, path, v, len(keys))
            assert s.latest_seq() == o.latest_seq(), name
            assert s.scan() == o.scan(), name
            probe = list(dict.fromkeys(keys))
            probe = probe[:400] + probe[-400:] + [b"\xff-after", b"zz-missing"]
            assert s.multi_get(probe) == o.multi_get(probe), name
            assert [s.get(k) for k in probe[:20]] == [o.get(k) for k in probe[:20]], name
        assert {sort_selection(k)[0] for _, k, _, _ in shards} == {"radix", "size", "bits", "shared"}
    finally:
        for _, _, s, o in shards:
            s.close()
            o.close()
