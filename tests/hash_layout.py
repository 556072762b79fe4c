"""Host mirror of the engine's hash layout (test infrastructure, not a test).

The point lookups find a key through two hash tables (rocksplicator_b200/csrc/format.cuh):
  - a run's bucketised index: n_buckets 32-byte buckets of 8 u32 slots, slot = tag << ord_bits | ordinal + 1, home
    bucket ((u32)h * n_buckets) >> 32, tag (h >> 32) >> ord_bits, spilling into the next bucket (wrapping at the end);
  - a memtable's slot table: u64 slots, slot = tag32 << 32 | head + 1 with tag32 = hash_tag32(h) (0 is stored as 1),
    home (u32)h & mask, linear probing; the two-lane MultiGet kernels read the 8-slot window from the home slot.

This module restates the hash and those formulas in numpy (vectorised over many keys of one length) and offers
seeded, deterministic finders for keys that land on the branches a random key set reaches only by chance: a given
home, a shared (bucket, tag) or tag32, a shared memtable filter bit.  tests/test_hash_layout_cpu.py pins the mirror to
format.cuh itself.

Keys whose h >> 32 is 0 or 1 take about 2**32 hashes each; `python tests/hash_layout.py --generate` finds them with a
small brute-force C program (compiled with g++ into a temporary directory) and writes tests/golden/hash_edges.json.
"""
import functools
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
EDGES_JSON = os.path.join(HERE, "golden", "hash_edges.json")

U64 = np.uint64
MASK64 = (1 << 64) - 1
MT_FILTER_BITS = 65536


# ---- the hash (format.cuh: hash_init / hash_step / hash_final over zero-padded little-endian words) ----------------
def _init(klen):
    return U64((0x5EED0001D1B54A32 ^ ((klen * 0x9E3779B97F4A7C15) & MASK64)) & MASK64)


def _step(h, w):
    h = (h ^ w) * U64(0xff51afd7ed558ccd)
    return h ^ (h >> U64(32))


def _final(h):
    h = h ^ (h >> U64(33))
    h = h * U64(0xc4ceb9fe1a85ec53)
    return h ^ (h >> U64(29))


def hash_rows(keys):
    """keys: (N, klen) uint8, every row one key of length klen -> (N,) uint64 hashes"""
    keys = np.ascontiguousarray(keys, dtype=np.uint8)
    n, klen = keys.shape
    nw = (klen + 7) // 8
    padded = np.zeros((n, nw * 8), dtype=np.uint8)
    padded[:, :klen] = keys
    words = padded.view("<u8")
    with np.errstate(over="ignore"):
        h = np.full(n, _init(klen), dtype=U64)
        for i in range(nw):
            h = _step(h, words[:, i])
        return _final(h)


def hash_key(key):
    """one key (bytes) -> int"""
    return int(hash_rows(np.frombuffer(key, dtype=np.uint8).reshape(1, len(key)))[0]) if key else int(
        hash_rows(np.zeros((1, 0), dtype=np.uint8))[0])


def hash_keys(keys):
    """list of bytes (any lengths) -> (N,) uint64"""
    out = np.zeros(len(keys), dtype=U64)
    by_len = {}
    for i, k in enumerate(keys):
        by_len.setdefault(len(k), []).append(i)
    for klen, ix in by_len.items():
        rows = np.frombuffer(b"".join(keys[i] for i in ix), dtype=np.uint8).reshape(len(ix), klen)
        out[ix] = hash_rows(rows)
    return out


def hash_tag32(h):
    t = np.asarray(h, dtype=U64) >> U64(32)
    return np.where(t == 0, U64(1), t)


def mt_filter_bit(h):
    return (np.asarray(h, dtype=U64) >> U64(40)) & U64(MT_FILTER_BITS - 1)


# ---- run index layout (engine.cu: compact_plan sizes, k_compact.cu: k_compact_write places) ------------------------
def run_layout(keys, entries):
    """(n_buckets, ord_bits) of a run of `keys` user keys in `entries` entries"""
    n_buckets = max(1, (keys + 3) // 4)
    ord_bits = 1
    while (1 << ord_bits) <= entries:
        ord_bits += 1
    return n_buckets, ord_bits


def run_home(h, n_buckets):
    return ((np.asarray(h, dtype=U64) & U64(0xffffffff)) * U64(n_buckets)) >> U64(32)


def run_tag(h, ord_bits):
    return (np.asarray(h, dtype=U64) >> U64(32)) >> U64(ord_bits)


# ---- memtable layout (engine.cu: alloc_memtable) ----------------------------------------------------------------
def mt_slot_cap(write_buffer_bytes):
    """slots of a shard's first memtable (shard open), from ShardOpts.write_buffer_bytes (0 = 1 MiB)"""
    units = (write_buffer_bytes or (1 << 20)) // 16
    ents = units // 7
    want = max(16, ents * 2)
    cap = 1
    while cap < want:
        cap <<= 1
    return cap


def mt_home(h, mask):
    return np.asarray(h, dtype=U64) & U64(mask)


# ---- candidate keys -------------------------------------------------------------------------------------------
def candidates(label, start, count, klen=16):
    """(count, klen) uint8: `label` (ASCII, padded / cut to 8 bytes) then a little-endian counter from `start`.
    Deterministic: the same arguments give the same keys."""
    assert klen >= 1
    rows = np.zeros((count, 16), dtype=np.uint8)
    lab = np.frombuffer((label.encode() + b"________")[:8], dtype=np.uint8)
    rows[:, :8] = lab
    rows[:, 8:16] = np.arange(start, start + count, dtype="<u8").view(np.uint8).reshape(count, 8)
    if klen >= 16:
        return rows[:, :klen] if klen == 16 else np.concatenate([rows, np.zeros((count, klen - 16), np.uint8) + 0x2b], 1)
    # short keys: the counter bytes first, so that keys of one length stay distinct
    return np.ascontiguousarray(rows[:, 8:8 + klen] if klen <= 8 else np.concatenate([rows[:, :klen - 8], rows[:, 8:16]], 1))


def find_keys(label, pred, count, klen=16, batch=1 << 22, limit=1 << 28):
    """the first `count` candidates (in counter order) for which pred(h) holds -> list of bytes"""
    out = []
    start = 0
    while len(out) < count:
        if start >= limit:
            raise RuntimeError("hash_layout: %s found %d of %d keys" % (label, len(out), count))
        rows = candidates(label, start, batch, klen)
        h = hash_rows(rows)
        for i in np.nonzero(pred(h))[0][:count - len(out)]:
            out.append(rows[i].tobytes())
        start += batch
    return out


def find_run_home(bucket, n_buckets, count, label="rhome"):
    """keys whose home bucket in a run of n_buckets buckets is `bucket`"""
    return find_keys("%s%d" % (label, bucket), lambda h: run_home(h, n_buckets) == bucket, count)


def find_mt_home(slot, mask, count, label="mhome", klen=16):
    """keys whose home slot in a memtable of mask + 1 slots is `slot`"""
    return find_keys("%s%d" % (label, slot), lambda h: mt_home(h, mask) == slot, count, klen)


def find_filter_bit(bit, count, label="fbit"):
    """keys whose memtable filter bit is `bit`"""
    return find_keys("%s%d" % (label, bit), lambda h: mt_filter_bit(h) == bit, count)


def _pairs(label, sig, count, n, klens=(16,)):
    """groups of candidates with equal signature sig(h) (a uint64 array), birthday style over n candidates per key
    length; returns up to `count` pairs of distinct keys (a, b), deterministic"""
    rows, hs = [], []
    for klen in klens:
        r = candidates("%s%d" % (label, klen), 0, n, klen)
        rows.append(r)
        hs.append(hash_rows(r))
    s = np.concatenate([sig(h) for h in hs])
    src = np.concatenate([np.full(len(h), j, dtype=np.int32) for j, h in enumerate(hs)])
    idx = np.concatenate([np.arange(len(h)) for h in hs])
    order = np.argsort(s, kind="stable")
    ss = s[order]
    dup = np.nonzero(ss[1:] == ss[:-1])[0]
    out = []
    for d in dup:
        a, b = order[d], order[d + 1]
        ka = rows[src[a]][idx[a]].tobytes()
        kb = rows[src[b]][idx[b]].tobytes()
        if ka != kb:
            out.append((ka, kb))
        if len(out) == count:
            break
    if len(out) < count:
        raise RuntimeError("hash_layout: %s found %d of %d pairs" % (label, len(out), count))
    return out


@functools.lru_cache(maxsize=None)
def run_collision_pairs(n_buckets, ord_bits, count, n=1 << 18, label="rpair"):
    """pairs of 16-byte keys with equal (home bucket, run tag) in a run of that layout: each one's slot is a tag
    false positive for the other"""
    return _pairs(label, lambda h: (run_home(h, n_buckets) << U64(32 - ord_bits)) | run_tag(h, ord_bits), count, n)


@functools.lru_cache(maxsize=None)
def mt_collision_pairs(mask, count, n=1 << 24, klens=(16,), label="mpair"):
    """pairs of keys with equal tag32 AND equal home slot in a memtable of mask + 1 slots (keys of the lengths in
    klens; a pair may mix lengths)"""
    return _pairs(label, lambda h: (hash_tag32(h) << U64(32)) | mt_home(h, mask), count, n, klens)


def load_edges():
    with open(EDGES_JSON) as f:
        d = json.load(f)
    return {k: [bytes.fromhex(x) for x in v] for k, v in d.items() if isinstance(v, list)}


# ---- --generate: keys with h >> 32 == 0 / 1 (about 2**32 hashes each) ---------------------------------------------
_BRUTE_C = r"""
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <pthread.h>
#include <atomic>
static uint64_t init(uint32_t klen) { return 0x5EED0001D1B54A32ull ^ ((uint64_t)klen * 0x9E3779B97F4A7C15ull); }
static uint64_t step(uint64_t h, uint64_t w) { h = (h ^ w) * 0xff51afd7ed558ccdull; return h ^ (h >> 32); }
static uint64_t fin(uint64_t h) { h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ull; h ^= h >> 29; return h; }
// keys: klen 8 -> word0 = counter; klen 16 -> word0 = prefix, word1 = counter
// match: (h >> 32) == hi && (h & lo_mask) == lo
static uint32_t klen, hi, want; static uint64_t prefix, lo_mask, lo;
static std::atomic<uint64_t> next_blk{0}; static std::atomic<uint32_t> found{0};
static pthread_mutex_t mu = PTHREAD_MUTEX_INITIALIZER;
static uint64_t hits[64];
static void* worker(void*) {
  for (;;) {
    if (found.load() >= want) return 0;
    uint64_t b = next_blk.fetch_add(1);
    for (uint64_t c = b << 24; c < (b + 1) << 24; c++) {
      uint64_t h = init(klen);
      if (klen == 8) h = step(h, c); else { h = step(h, prefix); h = step(h, c); }
      h = fin(h);
      if ((uint32_t)(h >> 32) == hi && (h & lo_mask) == lo) {
        pthread_mutex_lock(&mu);
        uint32_t f = found.load();
        if (f < want) { hits[f] = c; found.store(f + 1); }
        pthread_mutex_unlock(&mu);
      }
    }
  }
}
int main(int argc, char** argv) {
  klen = atoi(argv[1]); prefix = strtoull(argv[2], 0, 16); hi = strtoul(argv[3], 0, 16);
  lo_mask = strtoull(argv[4], 0, 16); lo = strtoull(argv[5], 0, 16); want = atoi(argv[6]);
  int nt = atoi(argv[7]);
  pthread_t t[256];
  for (int i = 0; i < nt; i++) pthread_create(&t[i], 0, worker, 0);
  for (int i = 0; i < nt; i++) pthread_join(t[i], 0);
  for (uint32_t i = 0; i < want; i++) printf("%016llx\n", (unsigned long long)hits[i]);
  return 0;
}
"""


def _brute(exe, klen, prefix, hi, lo_mask, lo, want):
    out = subprocess.check_output([exe, str(klen), "%x" % prefix, "%x" % hi, "%x" % lo_mask, "%x" % lo, str(want),
                                   str(os.cpu_count() or 4)], text=True)
    keys = []
    for line in out.split():
        c = int(line, 16)
        k = c.to_bytes(8, "little") if klen == 8 else prefix.to_bytes(8, "little") + c.to_bytes(8, "little")
        keys.append(k)
    return sorted(keys)


def generate():
    with tempfile.TemporaryDirectory() as td:
        src, exe = os.path.join(td, "brute.cpp"), os.path.join(td, "brute")
        with open(src, "w") as f:
            f.write(_BRUTE_C)
        subprocess.check_call(["g++", "-O3", "-march=native", "-std=c++17", "-pthread", src, "-o", exe])
        prefix = int.from_bytes(b"hashedge", "little")
        h_empty = hash_key(b"")
        d = {
            "comment": "keys whose hash h (format.cuh) has h >> 32 == 0 (hash_tag32 stores it as 1) or == 1, and an "
                       "8-byte key with the empty key's tag32 and home slot at memtable mask 31; written by "
                       "python tests/hash_layout.py --generate",
            "hi0_16": [k.hex() for k in _brute(exe, 16, prefix, 0, 0, 0, 4)],
            "hi1_16": [k.hex() for k in _brute(exe, 16, prefix, 1, 0, 0, 4)],
            "hi0_8": [k.hex() for k in _brute(exe, 8, 0, 0, 0, 0, 2)],
            "empty_mate_8": [k.hex() for k in _brute(exe, 8, 0, h_empty >> 32, 31, h_empty & 31, 1)],
        }
    with open(EDGES_JSON, "w") as f:
        json.dump(d, f, indent=1)
        f.write("\n")
    print("wrote", EDGES_JSON)


if __name__ == "__main__":
    if "--generate" in sys.argv:
        generate()
    else:
        print(__doc__)
