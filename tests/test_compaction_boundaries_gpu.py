"""GPU: the flush and compaction pipeline of k_compact.cu at every path switch and size boundary, against the oracle port.

Every run the engine holds is written by one pipeline: k_compact_fill, then k_flush_sort (LSD radix sort of the memtable
in shared memory: ceil(V / 8) passes over the V varying bits of the 8-byte key prefixes, for V <= 48 and at most
FS_MAX_ITEMS entries) or k_compact_sort (bitonic: 4096-item tiles in shared memory, the larger strides in global memory),
then the merge path over the sorted sources (k_merge_partition / k_merge_tiles, tiles of MERGE_TILE items), then
k_compact_size (groups of versions, the exclusive scans in 1024 chunks, the shape totals that mark a run
RUN_ALL_PUT_FIXED) and k_compact_write (the block index every RSP_BLOCK_ENTRIES entries).  A wrong run stays wrong: every
read path serves it.

Each case states the shape it claims and proves it from stats() read before and after (runs, memtable and run entries,
flushes, compactions), and every flush asserts the sort it took from a model of the selection (radix_expected).  Then
the shard is compared with the oracle: the full scan, MultiGet of every written key and of missing keys, the 16-byte-key
MultiGet where the keys are 16 bytes, forward and reverse batched scans (the reads that consult RUN_ALL_PUT_FIXED), and
the latest sequence number."""
import bisect
import random
import struct

import numpy as np
import pytest

from oracle import okv
from rocksplicator_b200.write_batch import WriteBatch

pytestmark = pytest.mark.gpu

# ---- the engine's constants (k_compact.cu, kernels.h, format.cuh)
FS_MAX_ITEMS = 24576
MERGE_TILE = 2048
OK, INCOMPLETE = 0, 7
MISSING = [b"", b"\x00", b"zz-missing-key-0", b"\xff" * 16, b"m" * 40]


def prefix_of(k):
    return int.from_bytes(k[:8].ljust(8, b"\0"), "big")


def radix_expected(keys):
    """True iff k_flush_sort sorts a memtable holding entries of these keys (versions included) without handing it to
    the comparison sort: 2 <= n <= FS_MAX_ITEMS, the prefixes vary in at most 48 bits, no two distinct keys share one"""
    if not 2 <= len(keys) <= FS_MAX_ITEMS:
        return False
    pre = [prefix_of(k) for k in keys]
    if (min(pre) ^ max(pre)).bit_length() > 48:
        return False
    owner = {}
    return all(owner.setdefault(p, k) == k for k, p in zip(keys, pre))


# ------------------------------------------------------------------------------------------------------------
# a shard and its oracle
# ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng():
    """l0_compaction_trigger = 8 (the clamp): no background merge while a shard holds fewer than eight runs"""
    from rocksplicator_b200 import engine
    e = engine.Engine(0, l0_compaction_trigger=8)
    yield e
    e.close()


_n = [0]


class Pair:
    def __init__(self, eng, port_lib, merge_op=okv.MERGE_NONE, write_buffer_bytes=16 << 20):
        _n[0] += 1
        self.eng = eng
        self.s = eng.open_shard("cb%05d" % _n[0], merge_op=merge_op, write_buffer_bytes=write_buffer_bytes)
        self.o = okv.Okv(port_lib, merge_op=merge_op)
        self.mem = []  # keys of the memtable's entries, versions included
        self.written = set()
        self.seq_lag = 0  # sequence numbers the oracle spent that the engine did not (ingestion)
        self.ts = 1

    def close(self):
        self.s.close()
        self.o.close()

    def stats(self):
        return self.s.stats()

    def write(self, ops, per_batch=512):
        """ops: (kind, key, value) with kind "put" / "del" / "merge", applied in order through staged ticks"""
        batches = []
        for lo in range(0, len(ops), per_batch):
            wb = WriteBatch()
            for kind, k, v in ops[lo:lo + per_batch]:
                {"put": lambda: wb.put(k, v), "del": lambda: wb.delete(k), "merge": lambda: wb.merge(k, v)}[kind]()
            batches.append(wb.data())
        before = self.stats()["flushes"]
        for lo in range(0, len(batches), 512):
            part = batches[lo:lo + 512]
            ts = list(range(self.ts, self.ts + len(part)))
            self.ts += len(part)
            st = self.eng.apply_many([self.s.index] * len(part), part, ts)
            assert not st.any(), st
            for b, t in zip(part, ts):
                assert self.o.apply(b, t) == 0, self.o.last_error
        assert self.stats()["flushes"] == before, "the load must fit the memtable"
        self.mem += [k for _, k, _ in ops]
        self.written |= {k for _, k, _ in ops}

    def ingest(self, rows):
        """sorted (key, value) Puts as one new run: newest of all, and one sequence number when its range overlaps the
        shard's (the oracle applies the rows as one batch of Puts)"""
        assert not self.mem
        # (the engine compares with every run's first and last key; the cases here overlap the shard's range or not)
        overlap = bool(self.written) and rows[0][0] <= max(self.written) and min(self.written) <= rows[-1][0]
        seq0 = self.s.latest_seq()
        assert self.s.ingest(rows) == 0
        assert self.s.latest_seq() == seq0 + (1 if overlap else 0)
        wb = WriteBatch()
        for k, v in rows:
            wb.put(k, v)
        assert self.o.apply(wb.data(), self.ts) == 0
        self.ts += 1
        self.seq_lag += len(rows) - (1 if overlap else 0)
        self.written |= {k for k, _ in rows}

    def _sorted(self, fn, full):
        """flush or compact; asserts the flush count and the sort the memtable took"""
        b = self.stats()
        n = b["memtable_entries"]
        assert n == len(self.mem)
        generic = n >= 2 and not radix_expected(self.mem)
        assert fn() == 0
        assert (self.o.compact() if full else self.o.flush()) == 0
        a = self.stats()
        assert a["memtable_entries"] == 0
        assert a["flushes"] - b["flushes"] == (1 if n else 0)
        assert a["flush_comparison_sorts"] - b["flush_comparison_sorts"] == int(generic), (n, generic)
        self.mem = []
        return b, a

    def flush(self):
        return self._sorted(self.s.flush, False)

    def compact(self):
        b, a = self._sorted(self.s.compact, True)
        assert a["n_runs"] <= 1
        return b, a

    def check(self):
        s, o = self.s, self.o
        assert s.latest_seq() == o.latest_seq() - self.seq_lag
        want = o.scan()
        assert s.scan() == want
        keys = sorted(self.written) + MISSING
        assert s.multi_get(keys) == o.multi_get(keys)
        k16 = [k for k in sorted(self.written) if len(k) == 16]
        if k16 and len(k16) == len(self.written):
            k16 += [b"zz-missing-key-0", b"\x00" * 16]
            stride = (max([256] + [len(v) for _, v in want]) + 15) & ~15
            assert fixed_get(self.eng, s, k16, stride) == o.multi_get(k16)
        assert not self.mem, "batched scans flush the memtable"
        batched_scans(self, want)
        return want


def scan_starts(p, want):
    """start keys of batched scans: the ends, written keys spread over the shard, a missing key"""
    ks = sorted(p.written)
    return [b"", b"\xff" * 20, b"zz-missing-key-0"] + ks[::max(1, len(ks) // 8)] + ks[-1:]


def expect_scans(want, starts, limit, reverse):
    """what forward scans from starts (reverse: from the last key <= start, descending) return"""
    keys = [k for k, _ in want]
    out = []
    for k in starts:
        if reverse:
            i = bisect.bisect_right(keys, k)
            out.append((OK, want[max(0, i - limit):i][::-1]))
        else:
            i = bisect.bisect_left(keys, k)
            out.append((OK, want[i:i + limit]))
    return out


def batched_scans(p, want, snapshot=None, limit=8):
    """forward and reverse batched scans (at a snapshot when given) against the oracle's scan.  With one run in the
    view, these are the reads that take the fixed-shape path of a RUN_ALL_PUT_FIXED run (k_read.cu: 16-byte-multiple
    keys, 8-byte-multiple values)"""
    starts = scan_starts(p, want)
    widest = max([0] + [len(k) + len(v) for k, v in want])
    stride = (limit * (8 + widest) + 7) & ~7
    for reverse in (False, True):
        if snapshot is None:
            fn = p.eng.multi_scan_reverse if reverse else p.eng.multi_scan
            got = fn([p.s.index] * len(starts), starts, limit, stride)
        else:
            fn = p.eng.multi_scan_reverse_at if reverse else p.eng.multi_scan_at
            got = fn([snapshot] * len(starts), starts, limit, stride)
        assert got == expect_scans(want, starts, limit, reverse), ("reverse" if reverse else "forward", snapshot)


def fixed_get(eng, s, keys, stride):
    """rsp_multi_get_fixed (16-byte keys) -> [(status, value | None)]"""
    n = len(keys)
    six = np.full(n, s.index, dtype=np.uint32)
    kb = np.frombuffer(b"".join(keys), dtype=np.uint8).copy()
    vals = np.zeros(n * stride, dtype=np.uint8)
    vlen = np.zeros(n, dtype=np.uint32)
    st = np.full(n, -1, dtype=np.int32)
    assert eng.multi_get_fixed(six, kb, 16, vals, stride, vlen, st) == OK
    assert INCOMPLETE not in st
    return [(int(st[i]), vals[i * stride:i * stride + int(vlen[i])].tobytes() if st[i] == OK else None)
            for i in range(n)]


@pytest.fixture
def pairs(eng, port_lib):
    """opens pairs for one test and closes them after it (flush_all flushes every open shard of the engine)"""
    made = []

    def make(**kw):
        made.append(Pair(eng, port_lib, **kw))
        return made[-1]
    yield make
    for p in made:
        p.close()


def k16(p):
    """a 16-byte key whose 8-byte prefix is p: distinct prefixes are distinct keys and the other way round"""
    return struct.pack(">QQ", p, (p * 0x9E3779B97F4A7C15) & (2 ** 64 - 1))


def with_versions(rng, keys, n, tag):
    """n entries over these distinct keys: each key once (a Put, some Deletes), the rest versions of a few hot keys
    (overwrites and Deletes), shuffled"""
    ops = [("del" if i % 7 == 3 else "put", k, b"%s-%d" % (tag, i)) for i, k in enumerate(keys)]
    hot = keys[:3] if len(keys) >= 3 else keys
    for i in range(n - len(keys)):
        k = rng.choice(hot) if i % 3 else rng.choice(keys)
        ops.append(("del" if i % 5 == 4 else "put", k, b"%s-v%d" % (tag, i)))
    rng.shuffle(ops)
    return ops


# ------------------------------------------------------------------------------------------------------------
# 1. the radix sort's pass counts: V varying prefix bits, P = ceil(V / 8) passes (even P starts in shared memory)
# ------------------------------------------------------------------------------------------------------------
BASE = 0x6B << 56  # the prefixes' fixed high bits (above bit 55)


@pytest.mark.parametrize("v", [0, 1, 8, 9, 16, 17, 24, 32, 40, 41, 48, 49])
def test_flush_sort_pass_counts(pairs, v):
    """Memtables of 2, 33 and 3000 entries whose prefixes vary in exactly V bits (min and max of the window included,
    the other prefixes drawn without replacement), versions of some keys on top: V = 0 is versions of one key (no
    pass), 48 is the widest width the radix sort takes, 49 goes to the comparison sort untouched"""
    rng = random.Random(1000 + v)
    for n in (2, 33, 3000):
        d = min(n if n == 2 else n - n // 4, 1 << v)
        pre = {BASE, BASE | ((1 << v) - 1)}
        while len(pre) < d:
            pre.add(BASE | rng.getrandbits(v))
        keys = [k16(q) for q in sorted(pre)]
        ops = with_versions(rng, keys, n, b"V%d" % v)
        assert (min(map(prefix_of, keys)) ^ max(map(prefix_of, keys))).bit_length() == v
        p = pairs()
        p.write(ops)
        assert radix_expected(p.mem) == (v <= 48)
        newest = dict((k, kind) for kind, k, _ in ops)
        live = sum(kind == "put" for kind in newest.values())
        _, a = p.flush()  # (the first flush of a shard is its bottom: tombstones dropped)
        assert (a["n_runs"], a["run_entries"]) == (int(live > 0), live), (v, n)
        p.check()


# ------------------------------------------------------------------------------------------------------------
# 2. the radix sort's capacity: FS_MAX_ITEMS, and one launch over memtables on both sides of it
# ------------------------------------------------------------------------------------------------------------
def radix_memtable(rng, n, tag, distinct=None):
    """n entries of 16-byte keys with distinct prefixes varying in 48 bits (radix-eligible up to FS_MAX_ITEMS)"""
    d = distinct or n - n // 8
    pre = {BASE, BASE | ((1 << 48) - 1)}
    while len(pre) < d:
        pre.add(BASE | rng.getrandbits(48))
    return with_versions(rng, [k16(q) for q in sorted(pre)], n, tag)


@pytest.mark.parametrize("n", [FS_MAX_ITEMS - 1, FS_MAX_ITEMS, FS_MAX_ITEMS + 1])
def test_flush_sort_capacity(pairs, n):
    """Radix-eligible memtables of FS_MAX_ITEMS - 1, FS_MAX_ITEMS and FS_MAX_ITEMS + 1 entries: the shared memory
    sized for the largest, the last one left to the comparison sort by its size alone"""
    rng = random.Random(n)
    p = pairs()
    p.write(radix_memtable(rng, n, b"cap"))
    assert p.stats()["memtable_entries"] == n
    assert radix_expected(p.mem) == (n <= FS_MAX_ITEMS)
    p.flush()
    p.check()


def test_flush_all_mixes_paths_in_one_launch(eng, pairs):
    """ONE flush_all over memtables of 24577 (comparison sort by size), 24576 (radix at full capacity), 40 entries and
    40 entries whose distinct keys share their prefix (radix, then handed over): one launch, one shared-memory size"""
    rng = random.Random(77)
    shapes = [radix_memtable(rng, FS_MAX_ITEMS + 1, b"a"), radix_memtable(rng, FS_MAX_ITEMS, b"b"),
              radix_memtable(rng, 40, b"c"),
              with_versions(rng, [b"user_profile_%04d" % i for i in range(30)], 40, b"d")]
    ps = []
    for ops in shapes:
        p = pairs()
        p.write(ops)
        ps.append(p)
    assert [radix_expected(p.mem) for p in ps] == [False, True, True, False]
    before = [p.stats() for p in ps]
    assert eng.flush_all() == 0
    for p, b in zip(ps, before):
        assert p.o.flush() == 0
        a = p.stats()
        assert (a["flushes"] - b["flushes"], a["memtable_entries"], a["n_runs"]) == (1, 0, 1)
        assert a["flush_comparison_sorts"] - b["flush_comparison_sorts"] == int(not radix_expected(p.mem))
        p.mem = []
        p.check()


# ------------------------------------------------------------------------------------------------------------
# 3. the comparison sort at production sizes: the global-memory strides of k_compact_sort
# ------------------------------------------------------------------------------------------------------------
SORT_CASES = [
    # (entries, how the memtable reaches the comparison sort, write buffer)
    (5000, "bits", 0), (5000, "shared", 0),  # n_pow2 8192: one global stride per stage
    (20000, "shared", 0),                      # 32768, after k_flush_sort reordered the items
    (30000, "bits", 64 << 20),                 # 32768 (over FS_MAX_ITEMS), the host shim's 64 MB write buffer
    (100000, "shared", 0),                     # 131072
]


@pytest.mark.parametrize("n,how,wb", SORT_CASES, ids=lambda x: str(x))
def test_comparison_sort_at_size(pairs, n, how, wb):
    rng = random.Random(n + len(how))
    if how == "bits":  # distinct random prefixes over 64 bits: V > 48, k_flush_sort leaves the items as filled
        pre = set()
        while len(pre) < n - n // 8:
            pre.add(rng.getrandbits(64))
        keys = [k16(q) for q in sorted(pre)]
    else:  # one 8-byte prefix per 16 distinct keys: k_flush_sort (up to FS_MAX_ITEMS) sorts, then finds them
        keys = [struct.pack(">QQ", BASE | (i // 16), i) for i in range(n - n // 8)]
    p = pairs(write_buffer_bytes=wb or (16 << 20))
    p.write(with_versions(rng, keys, n, b"cs"))
    assert p.stats()["memtable_entries"] == n and not radix_expected(p.mem)
    v = (min(map(prefix_of, keys)) ^ max(map(prefix_of, keys))).bit_length()
    assert (v > 48) == (how == "bits")
    p.flush()
    p.check()


# ------------------------------------------------------------------------------------------------------------
# 4. the merge path over nine sources: seven flushed runs, an ingested run, the memtable
# ------------------------------------------------------------------------------------------------------------
def mkey(i):
    return b"m%015d" % i


def nine_source_layout(rng, total, big_ingest):
    """per source (7 runs oldest first, the ingested run, the memtable): its keys.  One hot key has a version in every
    source; `total - 9` other keys, each in one source.  The hot key's nine versions sit across the merge tile boundary
    (2044 keys before it, or as many as there are) when there are two tiles or more."""
    n_keys = total - 8
    c = min(MERGE_TILE - 4, n_keys - 1) if total > MERGE_TILE else n_keys // 2
    hot = mkey(c)
    others = [mkey(i) for i in range(n_keys) if i != c]
    rng.shuffle(others)
    sizes = [total // 9] * 9
    for i in range(total - sum(sizes)):
        sizes[i] += 1
    if big_ingest:  # the ingested run alone holds more than a tile
        sizes = [(total - MERGE_TILE - 60) // 8] * 9
        sizes[7] = total - 8 * sizes[0]
        assert sizes[7] > MERGE_TILE
    srcs, at = [], 0
    for sz in sizes:
        srcs.append(sorted(others[at:at + sz - 1] + [hot]))
        at += sz - 1
    assert at == len(others) and sum(sizes) == total
    return hot, srcs


@pytest.mark.parametrize("total,big_ingest", [(2047, False), (2048, False), (2049, False), (4096, False),
                                              (4097, False), (4097, True)])
def test_nine_source_merge(pairs, total, big_ingest):
    rng = random.Random(total * 2 + big_ingest)
    hot, srcs = nine_source_layout(rng, total, big_ingest)
    p = pairs()
    for r, keys in enumerate(srcs[:7]):
        p.write([("put", k, b"r%d-%s" % (r, k[-4:])) for k in keys])
        _, a = p.flush()
        assert (a["n_runs"], a["compactions"]) == (r + 1, 0)
    p.ingest([(k, b"ing-%s" % k[-5:]) for k in srcs[7]])
    st = p.stats()
    assert (st["n_runs"], st["compactions"]) == (8, 0)
    # the memtable: the hot key's newest Put, and in place of one of its own keys a Delete of a key of the oldest run
    drop = next(k for k in srcs[8] if k != hot)
    victim = next(k for k in srcs[0] if k != hot)
    p.write([("del", victim, b"")] + [("put", k, b"mem-%s" % k[-4:]) for k in srcs[8] if k != drop])
    b = p.stats()
    assert b["n_runs"] == 8 and b["memtable_entries"] > 0
    assert b["run_entries"] + b["memtable_entries"] == total  # the items of the nine-source merge
    _, a = p.compact()
    assert (a["n_runs"], a["compactions"] - b["compactions"]) == (1, 1)
    assert a["run_entries"] == total - 10  # the hot key once; the Delete and its victim gone at the bottom
    p.check()


def test_tiered_flush_merges_a_subset(pairs):
    """A foreground flush at seven runs whose sizes grow more than 2x from the newest: tiered_set takes the memtable
    and the two newest runs only (4097 items, the hot key's versions across the tile boundary); then the full
    compaction"""
    rng = random.Random(99)
    hot = mkey(MERGE_TILE - 1)  # 2047 keys before it, its three versions at 2047 .. 2049
    others = [mkey(i) for i in range(4097 - 2) if mkey(i) != hot]
    rng.shuffle(others)
    thirds = [sorted(others[i::3] + [hot]) for i in range(3)]  # the newest run, the second newest, the memtable
    p = pairs()
    sizes = []
    for r in range(5):  # the five oldest runs: large values, far beyond twice what the flush gathers
        last = p.stats()["run_bytes"]
        p.write([("put", b"old%02d-%07d" % (r, i), bytes([65 + r]) * 600) for i in range(1500)])
        p.flush()
        sizes.append(p.stats()["run_bytes"] - last)
    for r in range(2):
        last = p.stats()["run_bytes"]
        p.write([("put", k, b"n%d" % r) for k in thirds[r]])
        p.flush()
        sizes.append(p.stats()["run_bytes"] - last)
    p.write([("put", k, b"mem") for k in thirds[2]])
    b = p.stats()
    assert (b["n_runs"], b["compactions"]) == (7, 0)
    # the precondition, restated from tiered_set (runs newest first, from the memtable's bytes, two runs at least): the
    # setup reaches a subset merge.  What checks the engine is (n_runs, compactions) after the flush below.
    newest_first = sizes[::-1]
    acc, take = b["memtable_bytes"], 0
    while take < 7 and (take < 2 or newest_first[take] <= 2 * acc):
        acc += newest_first[take]
        take += 1
    assert take == 2
    assert b["memtable_entries"] + sum(len(t) for t in thirds[:2]) == 4097
    _, a = p.flush()
    assert (a["n_runs"], a["compactions"] - b["compactions"]) == (6, 1)
    p.check()
    p.compact()
    p.check()


# ------------------------------------------------------------------------------------------------------------
# 5. sizing and write: output sizes, long groups of versions, 64 KB shapes, RUN_ALL_PUT_FIXED
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 31, 32, 33, 1023, 1024, 1025])
def test_output_sizes(pairs, k):
    """Runs of exactly k entries around the block index (32 entries per block) and the 1024-thread scan of
    k_compact_size: k written as a flush over an older run (not the bottom: tombstones kept), then k as the bottom of a
    full compaction (tombstones dropped)"""
    rng = random.Random(k)
    p = pairs()
    under = k16(BASE | (1 << 40))
    p.write([("put", under, b"under")])
    p.flush()
    t = k // 4
    keys = [k16(BASE | (i * 7919 + 3)) for i in range(k + k)]
    live, fresh = keys[:k - t], keys[k:]
    tombs = keys[k - t:k]
    ops = [("put", x, b"a%d" % i) for i, x in enumerate(live)] + [("del", x, b"") for x in tombs]
    ops += [("put", rng.choice(live), b"over%d" % i) for i in range(max(1, k // 3))]
    p.write(ops)
    _, a = p.flush()
    assert (a["n_runs"], a["run_entries"]) == (2, 1 + k)
    p.check()
    x = max(1, k // 8) if k > 1 else 1
    gone = live[:x]
    p.write([("del", y, b"") for y in gone + [under]] + [("put", y, b"f") for y in fresh[:x + t]])
    _, a = p.compact()
    assert (a["n_runs"], a["run_entries"]) == (1, k)
    p.check()


@pytest.mark.parametrize("merge_op", [okv.MERGE_NONE, okv.MERGE_COUNTER], ids=["versions", "counter"])
def test_one_key_over_2048_versions(pairs, merge_op):
    """One key with 2100 versions among other keys: its group crosses the per-thread scan chunks of k_compact_size in
    a flush, then the merge tile boundary in a compaction with a run beside the memtable"""
    rng = random.Random(5 + merge_op)
    hot = k16(BASE | 500)
    p = pairs(merge_op=merge_op)
    val = (lambda i: struct.pack("<q", i * 37 - 900)) if merge_op else (lambda i: b"v%d" % i)
    side = [k16(BASE | i) for i in range(1000) if i != 500]
    for rnd in range(2):
        ops = [("put", hot, val(10 ** 6))]
        for i in range(2100):
            if merge_op:
                ops.append(("put" if i % 700 == 300 else "merge", hot, val(i)))
            else:
                ops.append(("del" if i % 9 == 8 else "put", hot, val(i)))
        ops += [("put", x, val(rnd * 10000 + j)) for j, x in enumerate(side[rnd::2])]
        p.write(ops)
        if rnd == 0:
            _, a = p.flush()
            assert a["run_entries"] == 1 + len(side[0::2])
        else:
            b = p.stats()
            assert b["memtable_entries"] + b["run_entries"] > MERGE_TILE
            _, a = p.compact()
            assert a["run_entries"] == 1 + len(side)
        p.check()


@pytest.mark.parametrize("size", [0xffff, 0x10000, 0x10001])
def test_wide_keys_and_values(pairs, size):
    """Keys and values of 65535 / 65536 / 65537 bytes (the 16-bit shape cache of k_compact_size): wide keys beside
    short ones, and runs whose every entry is a Put of a 16-byte key and a value of that size"""
    wide = [bytes([0x61 + i]) * 8 + b"w" * (size - 8) for i in range(3)]
    assert {len(w) for w in wide} == {size}
    p = pairs()
    p.write([("put", w, b"wide-%d" % i) for i, w in enumerate(wide)] + [("put", b"short", b"s"), ("del", b"b", b"")])
    p.flush()
    p.check()
    p.write([("put", wide[0], b"x" * size), ("del", wide[1], b"")])
    p.compact()
    p.check()
    # every entry a Put of one shape (16-byte key, `size`-byte value): flushed, then compacted with an overwrite
    q = pairs()
    ks = [k16(BASE | (i * 131)) for i in range(4)]
    q.write([("put", x, bytes([0x30 + i]) * size) for i, x in enumerate(ks)])
    q.flush()
    q.check()
    q.write([("put", ks[1], bytes([0x39]) * size)])
    q.compact()
    q.check()


UNDER = k16(BASE | (1 << 40))  # the key of the older run under the flushed memtable


def fixed_runs():
    """(name, merge op, the memtable's ops, the older run's value): memtables whose sorted run sits on one side of
    RUN_ALL_PUT_FIXED while it keeps what a read can still observe (a snapshot of the memtable, a flush over an older
    run), and whose bottom-most run may sit on the other (tombstones dropped, base-less operands folded into Puts)"""
    keys = [k16(BASE | (i * 977)) for i in range(300)]
    puts = [("put", x, b"%024d" % i) for i, x in enumerate(keys)]
    longer = list(puts)
    longer[150] = ("put", keys[150], b"%025d" % 150)
    tomb = puts + [("del", UNDER, b"")]  # shadows the older run's key: a flush must keep it
    # empty values: a Delete has the Puts' key length, value length and units, only its type sets it apart
    tomb_empty = [("put", x, b"") for x in keys] + [("del", UNDER, b"")]
    ctr = [("put", x, struct.pack("<q", i)) for i, x in enumerate(keys)]
    ctr += [("merge", x, struct.pack("<q", 3 * i + 1)) for i, x in enumerate(keys[::2])]
    ops_only = ctr[:100] + [("merge", k16(BASE | 3), struct.pack("<q", 7)), ("merge", k16(BASE | 3), struct.pack("<q", 8))]
    v24, v8 = b"%024d" % 10 ** 9, struct.pack("<q", 5)
    return [("all_put_fixed", okv.MERGE_NONE, puts, v24), ("one_value_longer", okv.MERGE_NONE, longer, v24),
            ("tombstone_kept", okv.MERGE_NONE, tomb, v24), ("tombstone_empty_values", okv.MERGE_NONE, tomb_empty, b""),
            ("counter_folded", okv.MERGE_COUNTER, ctr, v8),
            ("counter_partial_merge", okv.MERGE_COUNTER, ops_only, v8)]


@pytest.mark.parametrize("case", fixed_runs(), ids=lambda c: c[0])
def test_fixed_shape_runs(pairs, case):
    """Runs on each side of RUN_ALL_PUT_FIXED, which sends batched scans of a view holding that one run to the
    fixed-shape copy: all Puts of one shape, one value a byte longer, a tombstone, counter operands folded to 8-byte
    Puts among 8-byte Puts, and two operands with no base (one Merge until the bottom folds them into a Put).

    - A snapshot of a memtable-only shard: its view is one run sorted without being the bottom (the tombstone and the
      Merge survive), read through forward and reverse batched scans at the snapshot.
    - The same memtable flushed over an older run: stats() shows every key kept (the tombstone, the Merge); then the
      full compaction (the bottom) leaves one run, read through batched scans, MultiGet and the iterator.

    This covers the flag set where it must not be (a wrong fixed-shape copy fails the comparison); for the base-less
    counter Merge the copy would return the same 8 bytes as the fold, so that case proves its shape through stats()
    only.  Whether the flag is set where it may be is not observable from outside: the generic scan returns the same
    records."""
    name, merge_op, ops, under_value = case
    m = pairs(merge_op=merge_op)
    m.write(ops)
    with m.s.snapshot() as snap:
        st = m.stats()
        assert (st["n_runs"], st["memtable_entries"], st["flushes"]) == (0, len(ops), 0)
        batched_scans(m, m.o.scan(), snapshot=snap)
    p = pairs(merge_op=merge_op)
    p.write([("put", UNDER, under_value)])
    p.flush()
    p.write(ops)
    b, a = p.flush()
    assert (a["n_runs"], a["run_entries"] - b["run_entries"]) == (2, len({k for _, k, _ in ops}))
    p.check()
    b, a = p.compact()
    assert (a["n_runs"], a["run_entries"]) == (1, len(p.o.scan()))
    p.check()
