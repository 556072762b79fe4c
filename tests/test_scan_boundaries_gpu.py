"""GPU: the batched range scans of k_read.cu (k_multi_scan) at the boundaries of each path it picks, against a plain model
(one run of Puts) or the oracle port (deletes, overwrites, merge operands).

k_multi_scan serves every range read: rsp_multi_scan, _bounded, _reverse, the _at snapshot forms, the _device forms on
a caller's stream, and every iterator page.  It picks its path from sizes and shapes the caller cannot see:

- the fixed-shape fast path: one run in the view, flagged RUN_ALL_PUT_FIXED, klen % 16 == 0, vlen % 8 == 0, and an
  8-byte aligned output pointer and stride.  Its Seek (run_lower_bound_warp) stages the block index in shared memory
  and counts prefixes 32 blocks at a time with ballots when 1 < n_blocks <= SCAN_STAGE_PFX, searches the index in
  global memory (run_lower_bound) above that, and searches no index for one block or an empty key;
- the general path: the lane-per-run k-way merge (a shuffle-min of 8-byte prefixes, a loop that settles prefix ties by
  full-key compares, version groups walked newest run first), with the end / low key checked against the prefix.

Which path ran is not observable from outside, so every case states its path from a model of the choice (scan_path)
and the shape stats() reports, and reads every fast-path run a second time on the general path (a stride one byte
longer, or a device output pointer 4 bytes off 8-byte alignment): both must equal the model."""
import bisect
import os
import random
import struct

import numpy as np
import pytest

import bounded_oracle as BO
from oracle import okv
from rocksplicator_b200.write_batch import WriteBatch

pytestmark = pytest.mark.gpu
EMUL = bool(os.environ.get("RSP_TEST_EMUL_LIB"))
if not EMUL:
    import torch

# ---- the engine's constants (kernels.h, k_read.cu)
BLOCK = 32         # RSP_BLOCK_ENTRIES: one block-index prefix per 32 entries
STAGE_PFX = 512    # SCAN_STAGE_PFX: the largest block index staged in shared memory
OK, INCOMPLETE = 0, 7


def scan_path(n_runs, run_entries, klen, vlen, all_put, out_align, stride):
    """the path k_multi_scan takes for a view of n_runs runs (a live memtable counts as one) holding run_entries
    entries, all Puts of klen / vlen bytes when all_put, with the output at out_align (mod 8) and this stride"""
    if n_runs != 1 or not all_put or klen % 16 or vlen % 8 or (out_align | stride) % 8:
        return "general"
    n_blocks = (run_entries + BLOCK - 1) // BLOCK
    if n_blocks <= 1:
        return "fixed/no-index"
    return "fixed/staged" if n_blocks <= STAGE_PFX else "fixed/global"


# ------------------------------------------------------------------------------------------------------------
# the model of one run of Puts
# ------------------------------------------------------------------------------------------------------------
class Model:
    """sorted live (key, value) records (a run of Puts, or the port's scan of a view): what every scan form returns,
    before the limit and the byte budget"""

    def __init__(self, rows):
        self.rows = rows
        self.keys = [k for k, _ in rows]

    def fwd(self, start, exclusive=False, end=None):
        """from start (None: the first key; exclusive: after it), stopping before end"""
        i = 0 if start is None else (bisect.bisect_right if exclusive else bisect.bisect_left)(self.keys, start)
        j = len(self.keys) if end is None else bisect.bisect_left(self.keys, end)
        return self.rows[i:j] if j > i else []

    def rev(self, start, exclusive=False, low=None):
        """descending from the last key <= start (< start when exclusive; None: the last key), down to low inclusive"""
        i = len(self.keys) if start is None else (bisect.bisect_left if exclusive else bisect.bisect_right)(self.keys,
                                                                                                           start)
        j = 0 if low is None else bisect.bisect_left(self.keys, low)
        return self.rows[j:i][::-1] if i > j else []


def budget(recs, max_entries, stride):
    """the first max_entries records, as many as fit in stride bytes of [u32 klen][u32 vlen][key][value] records:
    INCOMPLETE with the records that fit when the next one does not"""
    out, used = [], 0
    for k, v in recs[:max_entries]:
        used += 8 + len(k) + len(v)
        if used > stride:
            return (INCOMPLETE, out)
        out.append((k, v))
    return (OK, out)


# ------------------------------------------------------------------------------------------------------------
# shards
# ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng():
    """l0_compaction_trigger = 8 (the clamp): no background merge while a shard holds fewer than eight runs"""
    from rocksplicator_b200 import engine
    e = engine.Engine(0, l0_compaction_trigger=8)
    yield e
    e.close()


_n = [0]


@pytest.fixture
def shards(eng):
    """opens shards for one test and closes them after it"""
    made = []

    def make(merge_op=okv.MERGE_NONE):
        _n[0] += 1
        made.append(eng.open_shard("sb%05d" % _n[0], merge_op=merge_op))
        return made[-1]
    yield make
    for s in made:
        s.close()


def one_run(make, rows):
    """a shard holding rows as ONE run built by rsp_ingest_sorted (the ordinary flush kernels)"""
    s = make()
    assert s.ingest(rows) == 0
    st = s.stats()
    assert (st["n_runs"], st["run_entries"], st["memtable_entries"]) == (1, len(rows), 0)
    return s


# ------------------------------------------------------------------------------------------------------------
# key layouts: 16-byte keys, 8-byte big-endian prefix + 8-byte suffix
# ------------------------------------------------------------------------------------------------------------
EDGE_PFX = [0x00 << 56, (0x7f << 56) | 0x00ffffffffffff, 0x80 << 56, (0xff << 56) | 0xfe]  # high bytes 00 7f 80 ff


def prefixes(rng, m):
    """m distinct sorted 64-bit prefixes, the four high-byte edges among them when m >= 4"""
    pre = set(EDGE_PFX[:m] if m >= 4 else [0x80 << 56][:m])
    while len(pre) < m:
        pre.add(rng.getrandbits(64))
    return sorted(pre)


def suffix(j, g):
    """suffix j of g sharing one prefix: spread over 64 bits (bytes 9.. from 0x00 to 0xff)"""
    return struct.pack(">Q", j * ((2 ** 64 - 1) // max(1, g - 1)))


def group_plan(n):
    """(start, size) of the shared-prefix groups of an n-entry run: one starting mid-block, one over the ballot chunk
    edge (blocks 31 | 32, entry 1024), groups of 100 and 1100 entries, and one over blocks 511 | 512 (entry 16384)"""
    plan = [(13, 31), (100, 32), (1010, 33), (2000, 100), (5000, 1100), (16300, 85)]
    fit = [(a, g) for a, g in plan if a + g <= n]
    if not fit and n >= 31:
        fit = [(1, min(31, n - 1))]
    return fit


def layout_keys(n, layout, seed):
    """n sorted 16-byte keys: "distinct" (one key per prefix), "groups" (group_plan, distinct prefixes between), "one"
    (one prefix for the whole run)"""
    rng = random.Random(seed)
    if layout == "distinct":
        return [struct.pack(">QQ", p, (p * 0x9E3779B97F4A7C15) & (2 ** 64 - 1)) for p in prefixes(rng, n)]
    if layout == "one":
        return [struct.pack(">Q", 0x80 << 56) + suffix(j, n) for j in range(n)]
    slots, i, plan = [], 0, dict(group_plan(n))
    while i < n:  # a slot is one prefix: a group or a single key
        g = plan.get(i, 1)
        slots.append(g)
        i += g
    keys = []
    for p, g in zip(prefixes(rng, len(slots)), slots):
        keys += [struct.pack(">Q", p) + (suffix(j, g) if g > 1 else struct.pack(">Q", rng.getrandbits(64)))
                 for j in range(g)]
    assert len(keys) == n and keys == sorted(set(keys))
    return keys


def pred(k):
    """a key just below k: k's last byte decremented, then 0xff bytes (or k without its trailing zero byte)"""
    return k[:-1] if k[-1] == 0 else k[:-1] + bytes([k[-1] - 1]) + b"\xff" * 4


def sample_blocks(n):
    nb = (n + BLOCK - 1) // BLOCK
    return sorted({b for b in (0, 1, 30, 31, 32, 33, 63, 64, 510, 511, 512, nb - 1) if b < nb})


def probes_of(keys):
    """block-edge probes (first key, last key, just below the first, just above the last), short keys (1 to 7 bytes:
    a zero-padded prefix), a key's first 8 bytes, the empty key and a key above every key"""
    n = len(keys)
    out = []
    for b in sample_blocks(n):
        first, last = keys[b * BLOCK], keys[min(n, (b + 1) * BLOCK) - 1]
        out += [first, last, pred(first), last + b"\0"]
    mid = keys[n // 2]
    out += [mid[:w] for w in range(1, 8)] + [mid[:8], keys[-1][:8], b"", b"\xff" * 20]
    return sorted(set(out))


# ------------------------------------------------------------------------------------------------------------
# the device forms on a caller's stream
# ------------------------------------------------------------------------------------------------------------
def to_dev(arrays):
    if EMUL:
        return [a.copy() for a in arrays]
    d = [torch.from_numpy(a.copy()).cuda() for a in arrays]
    torch.cuda.synchronize()
    return d


def device_scan(eng, six, keys, max_entries, stride, ends=None, reverse=False, exclusive=False, misalign=0):
    """rsp_multi_scan_device / _bounded_device / _reverse_device over shard six (keys of one length; ends: the end or
    low keys, of one length), output at an address misalign bytes past an 8-byte boundary"""
    from rocksplicator_b200.engine import _scan_records
    n = len(keys)
    arrs = [np.full(n, six, np.uint32), np.frombuffer(b"".join(keys) + b"\0", np.uint8),
            np.frombuffer(b"".join(ends or []) + b"\0", np.uint8), np.zeros(n * stride + 8, np.uint8),
            np.zeros(n, np.uint32), np.full(n, -1, np.int32)]
    d = to_dev(arrs)
    p = [a.ctypes.data if EMUL else a.data_ptr() for a in d]
    assert p[3] % 8 == 0
    stream = eng.lib.rsp_engine_stream(eng.h) if EMUL else torch.cuda.Stream()
    sh = stream if EMUL else stream.cuda_stream
    klen, elen = len(keys[0]), len(ends[0]) if ends else 0
    out = p[3] + misalign
    if reverse:
        rc = eng.lib.rsp_multi_scan_reverse_device(eng.h, n, p[0], p[1], klen, 1 if exclusive else 0,
                                                   p[2] if ends else None, elen, max_entries, out, stride, p[4], p[5],
                                                   sh)
    elif ends:
        rc = eng.lib.rsp_multi_scan_bounded_device(eng.h, n, p[0], p[1], klen, p[2], elen, max_entries, out, stride,
                                                   p[4], p[5], sh)
    else:
        rc = eng.lib.rsp_multi_scan_device(eng.h, n, p[0], p[1], klen, max_entries, out, stride, p[4], p[5], sh)
    assert rc == 0
    if not EMUL:
        stream.synchronize()
        d = [t.cpu().numpy() for t in d]
    return _scan_records(d[3][misalign:], d[4], d[5], n, stride)


# ------------------------------------------------------------------------------------------------------------
# every form over one run of Puts, against the model
# ------------------------------------------------------------------------------------------------------------
def rotate(xs, k):
    return xs[k:] + xs[:k]


def check_all_forms(eng, s, m, probes, limits, stride, fast_path, device=True, general_limits=(1, 33)):
    """host, _at (a snapshot of the run) and _device forms over s, forward / bounded / reverse / from the extremes,
    each read on the path stated (fast_path) at every limit and, at general_limits, with a stride one byte longer or
    the output 4 bytes off, on the general path: every result equals the model"""
    st = s.stats()
    n, klen, vlen = st["run_entries"], len(m.keys[0]), len(m.rows[0][1])
    assert st["memtable_entries"] == 0
    assert scan_path(st["n_runs"], n, klen, vlen, True, 0, stride) == fast_path
    assert scan_path(st["n_runs"], n, klen, vlen, True, 0, stride + 1) == "general"
    assert scan_path(st["n_runs"], n, klen, vlen, True, 4, stride) == "general"
    starts = rotate(probes, len(probes) - 3)  # mostly below the end / above the low they go with
    highs = rotate(probes, 3)
    six = [s.index] * len(probes)
    d16 = [p for p in probes if len(p) == klen]
    with s.snapshot() as snap:
        snaps = [snap] * len(probes)
        for L in limits:
            for strd in (stride, stride + 1)[:2 if L in general_limits else 1]:
                def eq(got, want, what):
                    assert got == [budget(w, L, strd) for w in want], (what, L, strd, fast_path)
                eq(eng.multi_scan(six, probes, L, strd), [m.fwd(p) for p in probes], "forward")
                eq(eng.multi_scan(six, starts, L, strd, ends=probes),
                   [m.fwd(a, end=e) for a, e in zip(starts, probes)], "bounded")
                for x in (False, True):
                    eq(eng.multi_scan_reverse(six, probes, L, strd, exclusive=x), [m.rev(p, x) for p in probes],
                       ("reverse", x))
                    eq(eng.multi_scan_reverse(six, highs, L, strd, lows=probes, exclusive=x),
                       [m.rev(h, x, lo) for h, lo in zip(highs, probes)], ("reverse low", x))
                    eq(eng.multi_scan_at(snaps, probes, L, strd, exclusive=x), [m.fwd(p, x) for p in probes],
                       ("at", x))
                    eq(eng.multi_scan_reverse_at(snaps, probes, L, strd, exclusive=x, lows=starts),
                       [m.rev(p, x, lo) for p, lo in zip(probes, starts)], ("reverse at low", x))
                eq(eng.multi_scan_at(snaps[:1], None, L, strd), [m.fwd(None)], "at from the first")
                eq(eng.multi_scan_reverse(six[:1], None, L, strd), [m.rev(None)], "reverse from the last")
                eq(eng.multi_scan_reverse_at(snaps[:1], None, L, strd), [m.rev(None)], "reverse at from the last")
            if not (device and d16):
                continue
            dst = rotate(d16, len(d16) - 1)
            for mis in (0, 4)[:2 if L in general_limits else 1]:
                def deq(got, want, what):
                    assert got == [budget(w, L, stride) for w in want], (what, L, mis, fast_path)
                deq(device_scan(eng, s.index, d16, L, stride, misalign=mis), [m.fwd(p) for p in d16], "device")
                deq(device_scan(eng, s.index, dst, L, stride, ends=d16, misalign=mis),
                    [m.fwd(a, end=e) for a, e in zip(dst, d16)], "device bounded")
                for x in (False, True):
                    deq(device_scan(eng, s.index, d16, L, stride, ends=dst, reverse=True, exclusive=x, misalign=mis),
                        [m.rev(p, x, lo) for p, lo in zip(d16, dst)], ("device reverse", x))


# ------------------------------------------------------------------------------------------------------------
# A. the block index: one run of 16-byte keys and 64-byte values per size and key layout
# ------------------------------------------------------------------------------------------------------------
SIZES = [(1, "fixed/no-index"), (31, "fixed/no-index"), (32, "fixed/no-index"), (33, "fixed/staged"),
         (1023, "fixed/staged"), (1024, "fixed/staged"), (1025, "fixed/staged"), (1057, "fixed/staged"),
         (16383, "fixed/staged"), (16384, "fixed/staged"), (16385, "fixed/global"), (20000, "fixed/global")]
A_CASES = [(n, path, lay) for n, path in SIZES for lay in ("distinct", "groups", "one") if n > 1 or lay == "distinct"]
A_LIMITS = (1, 31, 32, 33, 128)
VLEN = 64


def value_of(i, vlen=VLEN):
    return (struct.pack("<I", i) * ((vlen + 3) // 4))[:vlen]


@pytest.mark.parametrize("n,path,layout", A_CASES, ids=lambda x: str(x))
def test_block_index_search(eng, shards, n, path, layout):
    """Runs of 1 / 2 / 32 / 33 / 34 / 512 / 513 / 625 blocks, their keys one per prefix, in shared-prefix groups placed
    mid-block and over blocks 31 | 32 and 511 | 512, or all under one prefix: every scan form from, to and down to
    block-edge keys, keys just outside them, short keys and the extremes, at limits around one ballot chunk"""
    keys = layout_keys(n, layout, n)
    rows = [(k, value_of(i)) for i, k in enumerate(keys)]
    s = one_run(shards, rows)
    if layout == "groups":
        assert any(a <= 1024 < a + g for a, g in group_plan(n)) == (n >= 1043)
        assert any(a <= 16384 < a + g for a, g in group_plan(n)) == (n >= 16385)
    check_all_forms(eng, s, Model(rows), probes_of(keys), A_LIMITS, 128 * (24 + VLEN), path)


# ------------------------------------------------------------------------------------------------------------
# B. fast-path eligibility and the byte budget
# ------------------------------------------------------------------------------------------------------------
def shaped_rows(n, klen, vlen, seed):
    """n sorted rows of klen-byte keys (distinct 8-byte prefixes when klen >= 8) and vlen-byte values"""
    rng = random.Random(seed)
    keys = [(struct.pack(">Q", p) + struct.pack(">Q", p ^ 0x5555) * 8)[:klen] for p in prefixes(rng, n)]
    return [(k, value_of(i, vlen)) for i, k in enumerate(keys)]


@pytest.mark.parametrize("klen", [16, 32, 48, 8, 15, 17, 24])
def test_fast_path_eligibility(eng, shards, klen):
    """One-run shards of 100 entries (4 blocks) for every key length x value length 0 / 8 / 24 / 64 (the fixed-shape
    copy) and 1 / 7 / 12 / 65 (never): 8- and 24-byte keys and 12-byte values are what a looser alignment test would
    send down the 8-byte word stream"""
    for vlen in (0, 8, 24, 64, 1, 7, 12, 65):
        rows = shaped_rows(100, klen, vlen, klen * 100 + vlen)
        s = one_run(shards, rows)
        keys = [k for k, _ in rows]
        stride = (33 * (8 + klen + vlen) + 7) & ~7
        eligible = klen % 16 == 0 and vlen % 8 == 0
        path = scan_path(1, 100, klen, vlen, True, 0, stride)
        assert path == ("fixed/staged" if eligible else "general")
        probes = sorted({keys[0], keys[31], keys[32], keys[63], keys[64], keys[-1], pred(keys[40]), keys[70] + b"\0",
                         keys[50][:3], b"", b"\xff" * 20})
        check_all_forms(eng, s, Model(rows), probes, (1, 33), stride, path)


def test_empty_key_run(eng, shards):
    """one entry, the empty key (klen 0: eligible, no index)"""
    rows = [(b"", value_of(7, 8))]
    s = one_run(shards, rows)
    check_all_forms(eng, s, Model(rows), [b"", b"\0", b"a", b"\xff" * 20], (1, 2), 64, "fixed/no-index",
                    device=False)


@pytest.mark.parametrize("n", [33, 1025, 16385])
def test_byte_budget(eng, shards, n):
    """strides of exactly k records (fast path), one byte short of k records and one byte short of one record (no
    record fits: INCOMPLETE with none), max_entries 0 and 1, forward and reverse"""
    rows = [(k, value_of(i)) for i, k in enumerate(layout_keys(n, "groups", n + 1))]
    s = one_run(shards, rows)
    m, keys = Model(rows), [k for k, _ in rows]
    rec = 8 + 16 + VLEN
    probes = sorted({keys[0], keys[n // 2], keys[min(n - 1, 1030)], keys[-1], pred(keys[BLOCK]), b""})
    six = [s.index] * len(probes)
    with s.snapshot() as snap:
        for k in (1, 5, 32):
            for stride in (k * rec, k * rec - 1, rec - 1):
                assert (scan_path(1, n, 16, VLEN, True, 0, stride) == "general") == (stride != k * rec)
                for L in (0, 1, k, 64):
                    want_f = [budget(m.fwd(p), L, stride) for p in probes]
                    want_r = [budget(m.rev(p), L, stride) for p in probes]
                    assert eng.multi_scan(six, probes, L, stride) == want_f, (k, stride, L)
                    assert eng.multi_scan_at([snap] * len(probes), probes, L, stride) == want_f, (k, stride, L)
                    assert eng.multi_scan_reverse(six, probes, L, stride) == want_r, (k, stride, L)
                    assert eng.multi_scan_reverse_at([snap] * len(probes), probes, L, stride) == want_r, (k, stride, L)
                    if stride == rec - 1 and L:
                        assert all(w == (INCOMPLETE, []) for w in want_f[:-1] + want_r[1:])


def steps(it, move, n):
    """the iterator's entry, then up to n moves while it stays valid"""
    got = []
    while it.valid() and len(got) <= n:
        got.append((it.key(), it.value()))
        if len(got) <= n:
            move()
    return got


@pytest.mark.parametrize("n", [33, 16385])
def test_iterator_pages(eng, shards, n):
    """Iterators over a 2-block and a 513-block run (pages of 16 growing to 1024 entries end at many offsets): full walks
    both ways, Seek / SeekForPrev at block-edge keys, and a walk whose upper bound lies inside a shared-prefix group"""
    rows = [(k, value_of(i)) for i, k in enumerate(layout_keys(n, "groups", n + 2))]
    s = one_run(shards, rows)
    m, keys = Model(rows), [k for k, _ in rows]
    assert scan_path(1, n, 16, VLEN, True, 0, 16 * (24 + VLEN)) == ("fixed/staged" if n == 33 else "fixed/global")
    it = s.iterator()
    it.seek_to_first()
    assert steps(it, it.next, n) == rows and it.status() == 0
    it.seek_to_last()
    assert steps(it, it.prev, n) == rows[::-1] and it.status() == 0
    for p in probes_of(keys):
        it.seek(p)
        assert steps(it, it.next, 40) == m.fwd(p)[:41], p
        it.seek_for_prev(p)
        assert steps(it, it.prev, 40) == m.rev(p)[:41], p
    it.close()
    a, g = group_plan(n)[-1]
    for ub in (keys[a + g // 2], keys[a + g // 2] + b"\0", keys[a][:8] + b"\x80"):
        for start in (keys[0], keys[max(0, a - 70)], keys[a]):
            it = s.iterator(upper_bound=ub)
            it.seek(start)
            assert steps(it, it.next, n) == m.fwd(start, end=ub) and it.status() == 0, (start, ub)
            it.close()


# ------------------------------------------------------------------------------------------------------------
# C. the general path at its lane and tie limits, against the oracle port
# ------------------------------------------------------------------------------------------------------------
def ops_batches(ops, per_batch=256):
    out = []
    for lo in range(0, len(ops), per_batch):
        wb = WriteBatch()
        for kind, k, v in ops[lo:lo + per_batch]:
            {"put": lambda: wb.put(k, v), "del": lambda: wb.delete(k), "merge": lambda: wb.merge(k, v)}[kind]()
        out.append(wb.data())
    return out


def write_both(eng, s, db, ops):
    batches = ops_batches(ops)
    st = eng.apply_many([s.index] * len(batches), batches)
    assert not st.any(), st
    for b in batches:
        assert db.apply(b, 0) == 0


C_LIMITS = (1, 7, 500)


def check_general_view(eng, db, probes, snap_e=None, snap_o=None, six=None):
    """forward, bounded and reverse scans (the _at forms at snap_e, or the host forms on shard six) against the port,
    at every limit and at strides that cut a record.  The port's forward scan of the whole view is read once: a forward
    scan is a slice of it, a reverse scan the slice [low, start] reversed"""
    port = Model(db.scan(snapshot=snap_o))
    n = len(probes)
    lows = rotate(probes, n - 5)
    ends = rotate(probes, 5)
    for L in C_LIMITS:
        for stride in (1 << 16, 301, 1001) if L == C_LIMITS[-1] else (1 << 16,):
            want_f = [budget(port.fwd(p), L, stride) for p in probes]
            want_b = [budget(port.fwd(a, end=e), L, stride) for a, e in zip(probes, ends)]
            for x in (False, True):
                want_r = [budget(port.rev(p, x, lo), L, stride) for p, lo in zip(probes, lows)]
                if snap_e is not None:
                    got_r = eng.multi_scan_reverse_at([snap_e] * n, probes, L, stride, lows=lows, exclusive=x)
                else:
                    got_r = eng.multi_scan_reverse([six] * n, probes, L, stride, lows=lows, exclusive=x)
                assert got_r == want_r, ("reverse", x, L, stride)
            if snap_e is not None:
                got_f = eng.multi_scan_at([snap_e] * n, probes, L, stride)
                got_b = eng.multi_scan_at([snap_e] * n, probes, L, stride, ends=ends)
            else:
                got_f = eng.multi_scan([six] * n, probes, L, stride)
                got_b = eng.multi_scan([six] * n, probes, L, stride, ends=ends)
            assert got_f == want_f, ("forward", L, stride)
            assert got_b == want_b, ("bounded", L, stride)


def walk_both(it_e, it_o, probes):
    """full walks both ways, and Seek / SeekForPrev at every probe followed by 12 moves: the engine's iterator and the
    port's visit the same (key, value, status) states"""
    def walk(it, first, back, n):
        first(it)
        out = [BO._state(it)]
        while it.valid() and len(out) <= n:
            it.prev() if back else it.next()
            out.append(BO._state(it))
        return out
    for back in (False, True):
        seek_end = (lambda i: i.seek_to_last()) if back else (lambda i: i.seek_to_first())
        assert walk(it_e, seek_end, back, 10 ** 6) == walk(it_o, seek_end, back, 10 ** 6), back
    for p in probes:
        for back in (False, True):
            sk = (lambda i: i.seek_for_prev(p)) if back else (lambda i: i.seek(p))
            assert walk(it_e, sk, back, 12) == walk(it_o, sk, back, 12), (p, back)


TIE_A, TIE_B = b"tie\x80\x00\xffAA", b"tie\x80\x00\xffBB"  # two 8-byte prefixes shared by 40 keys each
HOT = b"hot-key-in-every-source"
PAD = [b"pad", b"pad\0", b"pad\0\0\0\0\0", b"pad\0\0\0\0\0\0", b"pad\0\0\0\0\0x", b"pad\0\0\0\0\0\xff\xff"]


def eight_sources(rng):
    """per source (7 runs oldest first, then the memtable): its ops.  Key j of tie group A goes to source j % 8, of
    group B to source 7 - j % 8: whichever order the lanes hold the sources in, in one of the groups the lowest lane
    holding the prefix holds the largest head (forward) and in the other the smallest (reverse) — several rounds of the
    tie loop per key.  The hot key has a version in every source (a Put, merge operands, a tombstone, a Put, operands);
    the PAD keys share one prefix with the shorter "pad" padded with zero bytes."""
    src = [[] for _ in range(8)]
    for j in range(40):
        src[j % 8].append(("put", TIE_A + struct.pack(">Q", 1000 * j + 7), struct.pack("<q", j)))
        src[7 - j % 8].append(("put", TIE_B + struct.pack(">H", 500 * j), struct.pack("<q", -j)))
    hot = [("put", 10), ("merge", 3), ("merge", 4), ("del", 0), ("put", 20), ("merge", 5), ("merge", 6), ("merge", 7)]
    for i, (kind, v) in enumerate(hot):
        src[i].append((kind, HOT, struct.pack("<q", v)))
    for i, k in enumerate(PAD):
        src[(3 * i) % 8].append(("put", k, struct.pack("<q", 100 + i)))
        src[(3 * i + 5) % 8].append(("merge", k, struct.pack("<q", 1)))
    fill = [b"f%04d" % i for i in range(200)]
    for i in range(8):
        for k in rng.sample(fill, 30):
            r = rng.random()
            src[i].append(("del" if r < 0.2 else "merge" if r < 0.4 else "put", k, struct.pack("<q", rng.randrange(99))))
    for ops in src:
        seen = set()
        ops[:] = [op for op in ops if not (op[1] in seen or seen.add(op[1]))]  # one version per key and source
    return src


def tie_probes(db):
    keys = [k for k, _ in db.scan()]
    out = [b"", b"\xff" * 20, b"tie", TIE_A, TIE_B, TIE_A + b"\0", TIE_B + b"\xff" * 9, HOT, HOT + b"\0", HOT[:8]]
    out += PAD + [b"pad\0\0\0\0", b"pad\0\0\0\0\0\0\0"]
    out += [TIE_A + struct.pack(">Q", 1000 * j + 7) for j in (0, 1, 7, 8, 20, 39)]
    out += [TIE_A + struct.pack(">Q", 1000 * j + 8) for j in (0, 9, 38)]
    out += [TIE_B + struct.pack(">H", 500 * j) for j in (0, 1, 8, 15, 39)] + [TIE_B + struct.pack(">H", 500 * 9 + 1)]
    return sorted(set(out + keys[::23]))


@pytest.mark.parametrize("merge_op", [okv.MERGE_COUNTER, okv.MERGE_UINT64ADD], ids=["counter", "uint64add"])
def test_eight_lane_view(eng, shards, merge_op):
    """Seven flushed runs and a live memtable (eight lanes), read at a snapshot and by iterators: prefix ties across all
    eight sources settled over several rounds, one key with a version in every source, keys whose prefixes equal a
    shorter key's padded with zero bytes"""
    rng = random.Random(8 + merge_op)
    s = shards(merge_op)
    db = BO.BoundedOkv(BO.load_port(), merge_op=merge_op)
    src = eight_sources(rng)
    for r, ops in enumerate(src[:7]):
        write_both(eng, s, db, ops)
        assert s.flush() == 0 and db.flush() == 0
        assert (s.stats()["n_runs"], s.stats()["compactions"]) == (r + 1, 0)
    write_both(eng, s, db, src[7])
    st = s.stats()
    assert st["n_runs"] == 7 and st["memtable_entries"] > 0
    assert scan_path(st["n_runs"] + 1, st["run_entries"], 16, 8, False, 0, 1 << 16) == "general"
    probes = tie_probes(db)
    snap_e, snap_o = s.snapshot(), db.snapshot()
    later = [("put", TIE_A + struct.pack(">Q", 1000 * 3 + 7), b"late"), ("del", HOT, b""), ("put", b"pad\0", b"l")]
    write_both(eng, s, db, later)
    assert s.stats()["n_runs"] == 7
    check_general_view(eng, db, probes, snap_e, snap_o)
    for at in (False, True):
        ie = (snap_e if at else s).iterator()
        io = db.iterator(snap_o if at else None, None)
        walk_both(ie, io, probes[::2])
        ie.close()
        io.close()
    snap_e.release()
    snap_o.release()
    db.close()


@pytest.mark.parametrize("merge_op", [okv.MERGE_COUNTER, okv.MERGE_UINT64ADD], ids=["counter", "uint64add"])
def test_big_run_beside_small_runs(eng, shards, merge_op):
    """An ingested run of 17000 entries (532 blocks: each lane searches the index in global memory) under three small
    flushed runs: overwrites, deletes, merge operands and new keys inside its shared-prefix groups and at its block
    edges; scans start, end and stop inside the groups and at the block edges"""
    rng = random.Random(17 + merge_op)
    n = 17000
    keys = layout_keys(n, "groups", 3)
    rows = [(k, struct.pack("<q", i)) for i, k in enumerate(keys)]
    s = shards(merge_op)
    db = BO.BoundedOkv(BO.load_port(), merge_op=merge_op)
    assert s.ingest(rows) == 0
    wb = WriteBatch()
    for k, v in rows:
        wb.put(k, v)
    assert db.apply(wb.data(), 0) == 0
    edges = [b * BLOCK + d for b in sample_blocks(n) for d in (-1, 0, 1) if 0 <= b * BLOCK + d < n]
    inside = [a + j for a, g in group_plan(n) for j in (0, 1, g // 2, g - 1)]
    for r in range(3):
        ops = []
        for i in rng.sample(edges + inside, 20) + rng.sample(range(n), 40):
            kind = ("put", "del", "merge")[rng.randrange(3)]
            ops.append((kind, keys[i], struct.pack("<q", rng.randrange(-50, 50))))
        for a, g in group_plan(n):
            ops.append(("put", keys[a + g // 2][:8] + struct.pack(">Q", rng.getrandbits(64)),
                        struct.pack("<q", 1000 + r)))
        seen = set()
        ops = [op for op in ops if not (op[1] in seen or seen.add(op[1]))]
        write_both(eng, s, db, ops)
        assert s.flush() == 0 and db.flush() == 0
    st = s.stats()
    assert (st["n_runs"], st["memtable_entries"]) == (4, 0) and st["run_entries"] > n
    assert scan_path(st["n_runs"], st["run_entries"], 16, 8, False, 0, 1 << 16) == "general"
    assert (n + BLOCK - 1) // BLOCK > STAGE_PFX
    probes = sorted(set([keys[i] for i in edges[::3] + inside[::2]] + [pred(keys[i]) for i in inside[1::4]] +
                        [keys[i] + b"\0" for i in edges[1::6]] + [b"", b"\xff" * 20, keys[n // 2][:5]]))
    check_general_view(eng, db, probes, six=s.index)
    snap_e, snap_o = s.snapshot(), db.snapshot()
    check_general_view(eng, db, probes[::3], snap_e, snap_o)
    snap_e.release()
    snap_o.release()
    db.close()
