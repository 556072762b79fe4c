"""GPU: every point-lookup path at forced hash collisions, full buckets and wrapped probes, against the oracle port.

Random keys reach the hash tables' rare branches only by chance (a run-tag false positive about once per 60 000
lookups, a tag32 collision inside one memtable window at about 2**16 keys per memtable).  Here the key sets are built
with tests/hash_layout.py's mirror of the layout (pinned to format.cuh by tests/test_hash_layout_cpu.py):

  run index   R1 a full home bucket, R2 the same at the last bucket (the probe wraps to bucket 0), R3 tag false
              positives, R4 run tag 0, R5 the sizes where n_buckets and ord_bits change, R6 several runs
              (k_multi_get16m), R7 the entry-size and value-stride edges of the same kernels;
  memtable    M1 two keys with one tag32 in one window, M2 full windows (one wrapping at the end of the table), M3
              h >> 32 == 0 (stored as tag32 1) next to h >> 32 == 1, M4 a filter bit set by another key, M5 keys with
              one tag32 and one home slot written in the same tick by each tick builder.

Every scenario is read through rsp_multi_get_fixed's direct path, rsp_multi_get_device, Get and MultiGet through the
read combiner (16-byte keys, and mixed with one odd-length key), a device key buffer shifted by 8 bytes (the generic
kernel), a snapshot (MultiGet and Get at it), and, built again on a shard with the append operator, Get
(k_get_versions).  rsp_debug_last_pending shows which lookups the 16-byte-key kernel deferred: the tests assert that
the fast kernel itself serves the tag false positives and bucket overflows, and that the windows it cannot decide go
to the pending list."""
import os
import struct

import numpy as np
import pytest

import hash_layout as hl
from oracle import okv
from rocksplicator_b200.write_batch import WriteBatch

pytestmark = pytest.mark.gpu
EMUL = bool(os.environ.get("RSP_TEST_EMUL_LIB"))
if not EMUL:
    import torch

OK, NOT_FOUND, INVALID, INCOMPLETE = 0, 1, 4, 7
UNKNOWN_SHARD = 0xFFFFFFF0  # answers InvalidArgument: the read combiner hands the whole call to the direct path
WB_SMALL = 64 << 10   # memtable of 2048 slots
WB_TINY = 1 << 10     # memtable of 32 slots
MASK_SMALL = hl.mt_slot_cap(WB_SMALL) - 1
MASK_TINY = hl.mt_slot_cap(WB_TINY) - 1


@pytest.fixture(scope="module")
def eng():
    """every shard holds at most one run when it is read: k_multi_get16"""
    from rocksplicator_b200 import engine
    e = engine.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def engm():
    """shards with several runs (no background merge below eight): k_multi_get16m"""
    from rocksplicator_b200 import engine
    e = engine.Engine(0, l0_compaction_trigger=8)
    yield e
    e.close()


_n = [0]


def val(k, ver=0, n=64):
    """n bytes naming the key and the version"""
    return ((k.hex() + ".%d|" % ver).encode() * (n // 20 + 2))[:n]


class Pair:
    """an engine shard and an oracle DB fed the same batches"""

    def __init__(self, e, merge_op=okv.MERGE_NONE, **kw):
        _n[0] += 1
        self.e = e
        self.merge_op = merge_op
        self.s = e.open_shard("coll%05d" % _n[0], merge_op=merge_op, **kw)
        self.o = okv.Okv(okv.load_port(), merge_op=merge_op)

    def apply(self, batches):
        if not batches:
            return
        st = self.e.apply_many([self.s.index] * len(batches), batches, [7] * len(batches))
        assert not st.any(), st
        for b in batches:
            assert self.o.apply(b, 7) == 0

    def puts(self, kvs):
        self.apply([WriteBatch().put(k, v).data() for k, v in kvs])

    def ingest(self, kvs):
        kvs = sorted(kvs)
        assert self.s.ingest(kvs) == OK
        for k, v in kvs:
            assert self.o.apply(WriteBatch().put(k, v).data(), 0) == 0

    def flush(self):
        assert self.s.flush() == OK
        assert self.o.flush() == OK

    def compact(self):
        assert self.s.compact() == OK
        assert self.o.compact() == OK

    def close(self):
        self.s.close()
        self.o.close()


def build_run(p, kvs, how):
    """one run holding kvs (16-byte keys, Puts), built by a flush, by a merge of three flushed runs, or by ingest"""
    if how == "ingest":
        p.ingest(kvs)
    elif how == "flush":
        p.puts(kvs)
        p.flush()
    else:
        for part in (kvs[0::3], kvs[1::3], kvs[2::3]):
            p.puts(part)
            p.flush()
        p.compact()


def assert_layout(p, keys, entries, n_runs=1):
    st = p.s.stats()
    assert st["n_runs"] == n_runs and st["run_entries"] == entries and st["memtable_entries"] == 0, st
    return hl.run_layout(keys, entries)


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


def _answers(vals, vlen, st, n, stride):
    out = []
    for i in range(n):
        s = int(st[i])
        if s == OK:
            out.append((s, vals[i * stride:i * stride + int(vlen[i])].tobytes()))
        else:
            out.append((s, int(vlen[i]) if s == INCOMPLETE else None))
    return out


def want_get(o, keys, stride=None):
    res = o.multi_get(keys)
    return [(INCOMPLETE, len(v)) if stride is not None and st == OK and len(v) > stride else (st, v) for st, v in res]


def same(got, want, what):
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    if len(got) != len(want) or bad:
        i = bad[0] if bad else min(len(got), len(want))
        raise AssertionError("%s: %d of %d answers differ; first at %d: got %.200r, want %.200r" % (
            what, len(bad), len(want), i, got[i] if i < len(got) else None, want[i] if i < len(want) else None))


def pending(e):
    cap = 1 << 16
    buf = np.zeros(cap, dtype=np.uint32)
    n = e.debug_last_pending(buf)
    return sorted(buf[:min(n, cap)].tolist()) if n <= cap else None


def host_form(p, keys, stride):
    """rsp_multi_get_fixed on its direct path (one extra lookup on an unknown shard sends it there) -> answers,
    deferred positions among `keys`"""
    e = p.e
    n = len(keys) + 1
    six = np.array([p.s.index] * len(keys) + [UNKNOWN_SHARD], dtype=np.uint32)
    kb = np.frombuffer(b"".join(keys) + b"\xee" * 16, dtype=np.uint8).copy()
    vals = np.zeros(n * stride, dtype=np.uint8)
    vlen = np.zeros(n, dtype=np.uint32)
    st = np.full(n, -1, dtype=np.int32)
    assert e.multi_get_fixed(six, kb, 16, vals, stride, vlen, st) == OK
    assert st[-1] == INVALID
    pend = pending(e)
    assert pend[-1:] == [len(keys)], pend  # the unknown shard is always deferred
    return _answers(vals, vlen, st, len(keys), stride), pend[:-1]


def device_form(p, keys, stride, shift=0):
    """rsp_multi_get_device on the engine stream; shift=8 moves the 16-byte keys off their 16-byte alignment (the
    generic kernel) -> answers, deferred positions"""
    e = p.e
    n = len(keys)
    kb = np.frombuffer(b"\0" * shift + b"".join(keys) + b"\0" * 8, dtype=np.uint8)
    d = _dev([np.full(n, p.s.index, dtype=np.uint32), kb, np.zeros(n * stride, dtype=np.uint8),
              np.zeros(n, dtype=np.uint32), np.full(n, -1, dtype=np.int32)])
    pp = [_ptr(a) for a in d]
    assert e.lib.rsp_multi_get_device(e.h, n, pp[0], pp[1] + shift, 16, pp[2], stride, pp[3], pp[4], None) == OK
    pend = pending(e)
    _, _, vals, vlen, st = _host(d)
    return _answers(vals, vlen, st, n, stride), pend


def read_all(p, keys, deferred=None, not_deferred=None, stride=256, snapshot=True):
    """every read path against the oracle; deferred / not_deferred: positions in `keys` the 16-byte-key kernel must
    (not) send to the pending list, in both the host and the device form"""
    want = want_get(p.o, keys, stride)
    plain = want_get(p.o, keys)
    for what, (got, pend) in (("host form", host_form(p, keys, stride)), ("device form", device_form(p, keys, stride))):
        same(got, want, what)
        if deferred is not None:
            missing = sorted(set(deferred) - set(pend))
            assert not missing, "%s: lookups %s were not deferred (pending %s)" % (what, missing, pend[:20])
        if not_deferred is not None:
            extra = sorted(set(not_deferred) & set(pend))
            assert not extra, "%s: lookups %s were deferred" % (what, extra[:20])
    got, pend = device_form(p, keys, stride, shift=8)
    same(got, want, "device form, shifted keys")
    assert pend == []  # the generic kernel has no pending list
    same(p.e.multi_get([p.s.index] * len(keys), keys, stride), plain, "combiner multi_get")
    odd = b"odd-length-key"
    same(p.e.multi_get([p.s.index] * (len(keys) + 1), keys + [odd], stride), plain + [p.o.get(odd)],
         "combiner multi_get with an odd-length key")
    same([p.s.get(k) for k in keys], plain, "Get")
    if snapshot:
        with p.s.snapshot() as snap:
            same(snap.multi_get(keys, stride), plain, "snapshot multi_get")
            same([snap.get(k) for k in keys], plain, "snapshot get")


def twin_append(e, build, keys):
    """the same scenario on a shard with the append operator (host-folded: Get walks the versions with
    k_get_versions)"""
    p = Pair(e, merge_op=okv.MERGE_APPEND)
    build(p)
    same([p.s.get(k) for k in keys], want_get(p.o, keys), "append-operator Get")
    p.close()


def fillers(n, label):
    return [r.tobytes() for r in hl.candidates(label, 0, n)]


# ---- run index --------------------------------------------------------------------------------------------------
K_RUN = 64  # keys per run of the collision scenarios: 16 buckets, ord_bits 7


def _full_bucket_kvs(home, label):
    nb, _ = hl.run_layout(K_RUN, K_RUN)
    crowd = hl.find_run_home(home, nb, 20, label)
    stored = crowd[:13]
    misses = crowd[13:]
    rest = [k for k in fillers(K_RUN * 2, label + "f") if k not in crowd][:K_RUN - len(stored)]
    return [(k, val(k)) for k in stored + rest], misses


@pytest.mark.parametrize("how", ["flush", "merge", "ingest"])
@pytest.mark.parametrize("where", ["R1", "R2"])
def test_full_home_bucket(eng, how, where):
    """R1: 13 keys home to one bucket: five spill into the next one and push its own keys further.  R2: the same at the
    last bucket: spills and misses wrap to bucket 0."""
    nb, ob = hl.run_layout(K_RUN, K_RUN)
    home = 5 if where == "R1" else nb - 1
    kvs, misses = _full_bucket_kvs(home, "%s%s" % (where, how))
    p = Pair(eng)
    build_run(p, kvs, how)
    assert assert_layout(p, K_RUN, K_RUN) == (nb, ob)
    keys = [k for k, _ in kvs] + misses
    read_all(p, keys, not_deferred=range(len(keys)))
    twin_append(eng, lambda q: build_run(q, kvs, how), keys)
    p.close()


@pytest.mark.parametrize("how", ["flush", "merge", "ingest"])
def test_tag_false_positives(eng, how):
    """R3: misses with the (bucket, tag) of a stored key answer NotFound; stored keys sharing one (bucket, tag) each
    find their own value (enough pairs that both slot orders inside a bucket occur)"""
    nb, ob = hl.run_layout(K_RUN, K_RUN)
    pairs = hl.run_collision_pairs(nb, ob, 24)
    both = pairs[:16]     # both keys stored
    half = pairs[16:]     # only the first stored: the second is a miss behind a false positive
    stored = [k for a, b in both for k in (a, b)] + [a for a, _ in half]
    stored += fillers(K_RUN, "R3" + how)[:K_RUN - len(stored)]
    kvs = [(k, val(k)) for k in stored]
    p = Pair(eng)
    build_run(p, kvs, how)
    assert assert_layout(p, K_RUN, K_RUN) == (nb, ob)
    keys = [k for a, b in both for k in (a, b)] + [b for _, b in half] + [a for a, _ in half]
    read_all(p, keys, not_deferred=range(len(keys)))
    twin_append(eng, lambda q: build_run(q, kvs, how), keys)
    p.close()


def test_run_tag_zero(eng):
    """R4: keys whose h >> 32 is 0 or 1 have run tag 0 at any ord_bits: the slot word is just ordinal + 1"""
    e = hl.load_edges()
    special = e["hi0_16"] + e["hi1_16"]
    for how in ("flush", "ingest"):
        kvs = [(k, val(k)) for k in special + fillers(K_RUN - len(special), "R4" + how)]
        p = Pair(eng)
        build_run(p, kvs, how)
        nb, ob = assert_layout(p, K_RUN, K_RUN)
        assert all(int(hl.run_tag(hl.hash_key(k), ob)) == 0 for k in special)
        keys = special + [k for k, _ in kvs[len(special):]][:8] + fillers(8, "R4miss")
        read_all(p, keys, not_deferred=range(len(keys)))
        p.close()
    # an 8-byte key with h >> 32 == 0 in a run of mixed key lengths (the generic kernel)
    p = Pair(eng)
    kvs = [(k, val(k)) for k in e["hi0_8"]] + [(b"x%d" % i, b"v%d" % i) for i in range(9)]
    build_run(p, kvs, "flush")
    same(p.e.multi_get([p.s.index] * len(kvs), [k for k, _ in kvs]), want_get(p.o, [k for k, _ in kvs]), "8-byte")
    same([p.s.get(k) for k, _ in kvs], want_get(p.o, [k for k, _ in kvs]), "8-byte Get")
    p.close()


SIZES = [1, 4, 5, 8, 9, (1 << 12) - 1, 1 << 12, (1 << 12) + 1, (1 << 16) - 1, 1 << 16, (1 << 16) + 1]


@pytest.mark.parametrize("n", SIZES)
def test_run_sizes(eng, n):
    """R5: n_buckets from 1 to 2 and ord_bits across its boundaries; every key found, misses NotFound (with one bucket
    a miss probes the only bucket)"""
    keys = fillers(n, "R5n%d" % n)
    kvs = [(k, val(k)) for k in keys]
    p = Pair(eng)
    build_run(p, kvs, "ingest" if n > 9 else "flush")
    assert_layout(p, n, n)
    sample = keys if n <= 64 else keys[:32] + keys[-32:] + keys[n // 2:n // 2 + 32]
    q = sample + fillers(24, "R5miss%d" % n)
    read_all(p, q, not_deferred=range(len(q)))
    p.close()


@pytest.mark.parametrize("n", [3, 4, 5, 63, 64, 65])
def test_entries_outnumber_keys(eng, n):
    """R5: an append-operator shard keeps its operand stacks in the run, so ord_bits follows the entries and n_buckets
    the keys; the last key's version group ends at the last ordinal"""
    keys = sorted(fillers(n, "R5e%d" % n))
    p = Pair(eng, merge_op=okv.MERGE_APPEND)
    batches = [WriteBatch().put(k, val(k)).data() for k in keys]
    batches += [WriteBatch().merge(keys[-1], b"op%d" % j).data() for j in range(5)]
    batches += [WriteBatch().merge(keys[0], b"first").data()]
    p.apply(batches)
    p.flush()
    assert_layout(p, n, n + 6)
    q = keys + fillers(8, "R5emiss")
    same([p.s.get(k) for k in q], want_get(p.o, q), "append Get")
    same(p.e.multi_get([p.s.index] * len(q), q), want_get(p.o, q), "append multi_get")
    # the same shape with Puts stacked under the last key (plain shard): the fast kernel answers the newest version
    p2 = Pair(eng)
    p2.apply([WriteBatch().put(k, val(k)).data() for k in keys] + [WriteBatch().put(keys[-1], val(keys[-1], j)).data()
                                                                  for j in range(1, 4)])
    p2.flush()
    st = p2.s.stats()
    assert st["run_entries"] in (n, n + 3), st  # a flush keeps or drops the overwritten versions
    read_all(p2, q)
    p.close()
    p2.close()


def test_several_runs(engm):
    """R6 (k_multi_get16m): keys held only by the oldest run while the newer runs hold tag false positives and full
    home buckets on their probe path; the two newest runs hold Merges and Deletes of keys whose slots collide with
    those of older keys (each run's entries are uniform, so the fast kernel probes every one of them)"""
    nb, ob = hl.run_layout(K_RUN, K_RUN)
    pairs = hl.run_collision_pairs(nb, ob, 24, label="R6pair")
    old_keys = [a for a, _ in pairs[:12]]
    fp_keys = [b for _, b in pairs[:12]]
    del_pairs = pairs[12:18]
    mrg_pairs = pairs[18:24]
    homes = sorted(set(int(hl.run_home(hl.hash_key(k), nb)) for k in old_keys))[:2]
    crowd = [k for h in homes for k in hl.find_run_home(h, nb, 13, "R6crowd%d" % h)]
    p = Pair(engm, merge_op=okv.MERGE_UINT64ADD)
    # oldest run: the keys looked up, and the partners of the Delete / Merge pairs
    old = old_keys + [a for a, _ in del_pairs] + [a for a, _ in mrg_pairs] + [b for _, b in del_pairs + mrg_pairs]
    old += fillers(K_RUN, "R6o")[:K_RUN - len(old)]
    p.puts([(k, val(k)) for k in old])
    p.flush()
    # middle run: false positives of the old keys and two crowded home buckets
    mid = fp_keys + crowd
    mid += fillers(K_RUN, "R6m")[:K_RUN - len(mid)]
    p.puts([(k, val(k, 1)) for k in mid])
    p.flush()
    # two newer runs: Merges (64-byte operands: uniform entries, as a Put's) and Deletes of keys whose slots collide
    # with keys of the older runs
    mrg = [WriteBatch().merge(b, val(b, 3)).data() for _, b in mrg_pairs]
    p.apply(mrg + [WriteBatch().put(k, val(k, 2)).data() for k in fillers(K_RUN, "R6n")[:K_RUN - len(mrg)]])
    p.flush()
    dels = [WriteBatch().delete(b).data() for _, b in del_pairs]
    p.apply(dels + [WriteBatch().delete(k).data() for k in fillers(K_RUN, "R6d")[:K_RUN - len(dels)]])
    p.flush()
    st = p.s.stats()
    assert st["n_runs"] == 4 and st["run_entries"] == 4 * K_RUN, st
    keys = old_keys + [a for a, _ in del_pairs + mrg_pairs] + [b for _, b in del_pairs + mrg_pairs] + fillers(8, "R6miss")
    n_plain = len(old_keys) + len(del_pairs) + len(mrg_pairs)
    read_all(p, keys, not_deferred=range(n_plain), deferred=range(n_plain, n_plain + len(del_pairs) + len(mrg_pairs)))
    p.close()


def test_entry_size_and_stride_edges(eng):
    """R7: uniform entries of 254 units (vlen 4032, served by the fast kernel) and 255 units (vlen 4033: the
    descriptor's meta byte saturates, deferred); strides 96 and 97 around the BIG template; a stride below the value
    answers Incomplete with the size needed"""
    for vl, fast in ((4032, True), (4033, False)):
        keys = fillers(24, "R7u%d" % vl)
        p = Pair(eng)
        build_run(p, [(k, val(k, 0, vl)) for k in keys], "ingest")
        q = keys + fillers(4, "R7miss")
        if fast:
            read_all(p, q, not_deferred=range(len(q)), stride=4096)
        else:
            read_all(p, q, deferred=range(len(keys)), stride=4096)
        read_all(p, q, stride=4000, snapshot=False)  # Incomplete, vlen = the size needed
        p.close()
    for vl in (96, 97):
        keys = fillers(24, "R7v%d" % vl)
        p = Pair(eng)
        build_run(p, [(k, val(k, 0, vl)) for k in keys], "flush")
        q = keys + fillers(4, "R7vmiss")
        for stride in (96, 97, 112):
            read_all(p, q, stride=stride, snapshot=stride == 96)
        p.close()


# ---- memtable -------------------------------------------------------------------------------------------------------
def assert_memtable_only(p):
    st = p.s.stats()
    assert st["n_runs"] == 0 and st["memtable_entries"] > 0, st


def test_same_tag32_in_one_window(eng):
    """M1: two keys with one tag32 and one home slot (both in one window: the fast kernel cannot tell which is which
    and defers), and a miss with a stored key's tag32 in its window"""
    pairs = hl.mt_collision_pairs(MASK_SMALL, 10)
    both, half = pairs[:5], pairs[5:]
    p = Pair(eng, write_buffer_bytes=WB_SMALL)
    p.puts([(k, val(k)) for a, b in both for k in (a, b)] + [(a, val(a)) for a, _ in half])
    assert_memtable_only(p)
    keys = [k for a, b in both for k in (a, b)] + [b for _, b in half]
    read_all(p, keys, deferred=range(len(keys)))
    p.flush()
    read_all(p, keys, not_deferred=range(len(keys)))
    twin_append(eng, lambda q: (q.puts([(k, val(k)) for a, b in both for k in (a, b)] + [(a, val(a)) for a, _ in half])),
                keys)
    p.close()


@pytest.mark.parametrize("home", [100, MASK_SMALL - 3])
def test_full_window(eng, home):
    """M2: eight keys home to one slot, so a ninth lands behind a full window (deferred), and a miss there whose
    filter bit is set by a stored key is deferred too; the eight inside the window are served by the fast kernel.  At
    home = mask - 3 the window wraps to slot 0"""
    crowd = hl.find_mt_home(home, MASK_SMALL, 9, "M2h%d" % home)
    p = Pair(eng, write_buffer_bytes=WB_SMALL)
    p.puts([(k, val(k)) for k in crowd[:8]])
    p.puts([(crowd[8], val(crowd[8]))])  # a tick later: it lands behind the eight
    bits = set(int(hl.mt_filter_bit(hl.hash_key(k))) for k in crowd)
    miss = hl.find_keys("M2miss%d" % home, lambda h: (hl.mt_home(h, MASK_SMALL) == home) & np.isin(hl.mt_filter_bit(h), list(bits)), 1)
    keys = crowd + miss
    read_all(p, keys, deferred=[8, 9], not_deferred=range(8))
    twin_append(eng, lambda q: (q.puts([(k, val(k)) for k in crowd[:8]]), q.puts([(crowd[8], val(crowd[8]))])), keys)
    p.close()


def test_tag32_zero_and_one(eng):
    """M3: a key with h >> 32 == 0 (its tag32 is stored as 1) next to a key with h >> 32 == 1 in one window of a
    32-slot memtable; the first is deferred (two tag matches) to walk_memtable; again after a flush (run tag 0)"""
    e = hl.load_edges()
    best = None
    for z in e["hi0_16"]:
        for o in e["hi1_16"]:
            d = (int(hl.mt_home(hl.hash_key(o), MASK_TINY)) - int(hl.mt_home(hl.hash_key(z), MASK_TINY))) & MASK_TINY
            if d <= 5 and (best is None or d < best[0]):
                best = (d, z, o)
    assert best, "no tag-0 / tag-1 pair within one window at mask %d" % MASK_TINY
    d, z, o = best
    hz = int(hl.mt_home(hl.hash_key(z), MASK_TINY))
    gap = [hl.find_mt_home((hz + i) & MASK_TINY, MASK_TINY, 1, "M3g")[0] for i in range(1, d)]
    p = Pair(eng, write_buffer_bytes=WB_TINY)
    p.puts([(k, val(k, 0, 8)) for k in [z, o] + gap])
    assert_memtable_only(p)
    keys = [z, o] + gap + [e["hi0_16"][-1] if e["hi0_16"][-1] != z else e["hi0_16"][0]]
    read_all(p, keys, deferred=[0])
    p.flush()
    read_all(p, keys, not_deferred=range(len(keys)))
    # variable lengths: the 8-byte key with h >> 32 == 0, and the empty key next to an 8-byte key with its tag32 and
    # home slot (the generic kernel and walk_memtable)
    p2 = Pair(eng, write_buffer_bytes=WB_TINY)
    vk = e["hi0_8"][:1] + [b""] + e["empty_mate_8"]
    p2.puts([(k, b"v-" + k) for k in vk])
    same(p2.e.multi_get([p2.s.index] * len(vk), vk), want_get(p2.o, vk), "variable-length multi_get")
    same([p2.s.get(k) for k in vk], want_get(p2.o, vk), "variable-length Get")
    p2.flush()
    same([p2.s.get(k) for k in vk], want_get(p2.o, vk), "variable-length Get after a flush")
    p.close()
    p2.close()


@pytest.mark.parametrize("window", ["empty", "full"])
def test_filter_false_positive(eng, window):
    """M4: run keys whose memtable filter bit is set by a different memtable key: with an empty window the fast kernel
    goes on to the run itself; with a full window it defers"""
    run_keys = fillers(16, "M4r" + window)
    p = Pair(eng, write_buffer_bytes=WB_SMALL)
    build_run(p, [(k, val(k)) for k in run_keys], "ingest")
    mem = []
    for k in run_keys[:4]:
        h = hl.hash_key(k)
        mem += hl.find_filter_bit(int(hl.mt_filter_bit(h)), 1, "M4q%s" % k.hex()[-6:])
        if window == "full":
            mem += hl.find_mt_home(int(hl.mt_home(h, MASK_SMALL)), MASK_SMALL, 8, "M4w%s" % k.hex()[-6:])
    p.puts([(k, val(k, 1)) for k in mem])
    keys = run_keys[:4] + run_keys[4:8]
    if window == "empty":
        # (the memtable keys must not sit in the run keys' windows)
        for k in run_keys[:4]:
            hk = int(hl.mt_home(hl.hash_key(k), MASK_SMALL))
            assert all((int(hl.mt_home(hl.hash_key(m), MASK_SMALL)) - hk) & MASK_SMALL >= 8 for m in mem)
        read_all(p, keys, not_deferred=range(4))
    else:
        read_all(p, keys, deferred=range(4))
    p.close()


# ---- M5: colliding keys written in one tick -------------------------------------------------------------------------
def _interleaved(a, b, first_a):
    """Put / Merge / Delete versions of two keys, interleaved, one batch per version"""
    x, y = (a, b) if first_a else (b, a)
    ops = [("put", x, 1), ("put", y, 2), ("merge", x, 3), ("merge", y, 4), ("delete", y, 0), ("merge", x, 5),
           ("put", y, 6), ("merge", y, 7)]
    out = []
    for op, k, v in ops:
        wb = WriteBatch()
        if op == "put":
            wb.put(k, struct.pack("<Q", v))
        elif op == "merge":
            wb.merge(k, struct.pack("<Q", v))
        else:
            wb.delete(k)
        out.append(wb.data())
    return out


def _tick(e, groups):
    """one apply_many over {pair: batches}: the groups go to the engine as one tick"""
    six, bl = [], []
    for p, bs in groups:
        six += [p.s.index] * len(bs)
        bl += bs
    st = e.apply_many(six, bl, [7] * len(bl))
    assert not st.any(), st
    for p, bs in groups:
        for b in bs:
            assert p.o.apply(b, 7) == 0


@pytest.mark.parametrize("builder", ["fused64", "fused128", "chunks", "general"])
def test_colliding_keys_in_one_tick(eng, builder):
    """M5: keys with one tag32 and one home slot written in the same tick with interleaved versions, in both orders:
    link_into_table must compare the full keys, or one key's versions end up on the other's chain"""
    pairs = hl.mt_collision_pairs(MASK_SMALL, 10)
    n_shards = 1 if builder in ("fused64", "general") else (3 if builder == "chunks" else 2)
    ps = [Pair(eng, merge_op=okv.MERGE_UINT64ADD, write_buffer_bytes=WB_SMALL) for _ in range(n_shards)]
    groups, keys = [], []
    for si, p in enumerate(ps):
        mine = pairs[si * 3:(si + 1) * 3] if builder != "fused64" else pairs[:6]
        bs = []
        for j, (a, b) in enumerate(mine):
            bs += _interleaved(a, b, j % 2 == 0)
        keys.append([k for a, b in mine for k in (a, b)])
        if builder in ("fused128", "chunks"):  # groups longer than 64 (k_tick_fused<128> / k_tick_chunks) or 128
            extra = 100 if builder == "fused128" else 160
            bs += [WriteBatch().put(k, b"pad").data() for k in fillers(extra - len(bs), "M5pad%d" % si)]
        if builder == "general":  # a batch beyond 16 KB: the host stages the tick for the general kernels
            bs.insert(len(bs) // 2, WriteBatch().put(b"M5-big", b"B" * 20000).data())
        groups.append((p, bs))
    others = []
    if builder == "fused128":
        # k_tick_fused<128> runs a CTA per group when the groups alone fill the machine (4 per SM): one small group in
        # each of enough other shards
        others = [eng.open_shard("coll-fill%05d" % i, write_buffer_bytes=4096) for i in range(4 * 132)]
        six = [s.index for s in others]
        bl = [WriteBatch().put(b"f", b"%d" % i).data() for i in range(len(others))]
        all_six = six + [i for p, bs in groups for i in [p.s.index] * len(bs)]
        st = eng.apply_many(all_six, bl + [b for _, bs in groups for b in bs], [7] * len(all_six))
        assert not st.any(), st
        for p, bs in groups:
            for b in bs:
                assert p.o.apply(b, 7) == 0
    else:
        _tick(eng, groups)
    for p, ks in zip(ps, keys):
        q = ks + [b"M5-big"] if builder == "general" else ks
        same([p.s.get(k, cap=32768) for k in q], want_get(p.o, q), "Get")
        read_all(p, ks, stride=64)
        p.flush()
        read_all(p, ks, stride=64)
    for s in others:
        s.close()
    for p in ps:
        p.close()


def test_variable_length_colliding_keys_in_one_tick(eng):
    """M5: colliding keys of lengths 1, 7, 8, 9, 15 and 17 (one tag32, one home slot), and the empty key with an
    8-byte key of its tag32 and home slot at mask 31, written in one tick with interleaved versions"""
    pairs = hl.mt_collision_pairs(MASK_SMALL, 8, n=1 << 22, klens=(1, 7, 8, 9, 15, 17), label="M5v")
    p = Pair(eng, merge_op=okv.MERGE_UINT64ADD, write_buffer_bytes=WB_SMALL)
    bs = []
    for j, (a, b) in enumerate(pairs):
        bs += _interleaved(a, b, j % 2 == 0)
    _tick(eng, [(p, bs)])
    keys = [k for a, b in pairs for k in (a, b)]
    assert len(set(len(k) for k in keys)) > 1
    for stage in ("memtable", "run"):
        same(p.e.multi_get([p.s.index] * len(keys), keys), want_get(p.o, keys), "multi_get " + stage)
        same([p.s.get(k) for k in keys], want_get(p.o, keys), "Get " + stage)
        p.flush()
    e = hl.load_edges()
    pe = Pair(eng, merge_op=okv.MERGE_UINT64ADD, write_buffer_bytes=WB_TINY)
    mate = e["empty_mate_8"][0]
    _tick(eng, [(pe, _interleaved(b"", mate, True))])
    for stage in ("memtable", "run"):
        same([pe.s.get(k) for k in (b"", mate)], want_get(pe.o, [b"", mate]), "empty key " + stage)
        pe.flush()
    p.close()
    pe.close()


def test_debug_last_pending_reports_host_and_device_forms(eng):
    """rsp_debug_last_pending reports the last host-form or device-form MultiGet: its deferred count and positions
    (a Merge in the memtable is always deferred), and nothing after a call the generic kernel served"""
    p = Pair(eng, merge_op=okv.MERGE_UINT64ADD)
    keys = fillers(40, "dbgp")
    p.apply([WriteBatch().put(k, struct.pack("<Q", i)).data() for i, k in enumerate(keys)])
    p.flush()
    p.apply([WriteBatch().merge(k, struct.pack("<Q", 1)).data() for k in keys[5::7]])
    want = [i for i in range(len(keys)) if i % 7 == 5]
    got, pend = host_form(p, keys, 64)
    same(got, want_get(p.o, keys, 64), "host form")
    assert pend == want
    got, pend = device_form(p, keys, 64)
    same(got, want_get(p.o, keys, 64), "device form")
    assert pend == want
    got, pend = device_form(p, keys, 64, shift=8)
    assert pend == []
    p.close()
