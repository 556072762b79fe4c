"""CPU-only: tests/hash_layout.py's numpy mirror against format.cuh itself.

A small shim calls the header's host-callable hash_init / hash_step / hash_final / hash_tag32 / mt_filter_bit (built
with g++ against the CUDA emulation's cuda_runtime.h, into pytest's temporary directory).  The collision tests
(tests/test_lookup_collisions_gpu.py) build their key sets from the mirror, so a mirror that drifted from the header
would let them pass without reaching the branches they are about; this file catches that."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import hash_layout as hl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SHIM = r"""
#include <string.h>
#include "format.cuh"
using namespace rsp;
extern "C" {
uint64_t shim_hash(const uint8_t* k, uint32_t n) {
  uint64_t h = hash_init(n);
  for (uint32_t i = 0; i < (n + 7u) / 8u; i++) {
    uint64_t w = 0;
    memcpy(&w, k + 8u * i, n - 8u * i < 8u ? n - 8u * i : 8u);  // zero padded, little-endian
    h = hash_step(h, w);
  }
  return hash_final(h);
}
uint32_t shim_tag32(uint64_t h) { return hash_tag32(h); }
uint32_t shim_filter_bit(uint64_t h) { return mt_filter_bit(h); }
}
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("hash_shim")
    src, so = d / "shim.cpp", d / "libshim.so"
    src.write_text(SHIM)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-w",
                           "-I", os.path.join(ROOT, "tests", "emul", "include"),
                           "-I", os.path.join(ROOT, "rocksplicator_b200", "csrc"), str(src), "-o", str(so)])
    lib = C.CDLL(str(so))
    lib.shim_hash.restype = C.c_uint64
    lib.shim_hash.argtypes = [C.c_char_p, C.c_uint32]
    lib.shim_tag32.restype = C.c_uint32
    lib.shim_tag32.argtypes = [C.c_uint64]
    lib.shim_filter_bit.restype = C.c_uint32
    lib.shim_filter_bit.argtypes = [C.c_uint64]
    return lib


def check(shim, keys):
    hs = hl.hash_keys(keys)
    for k, h in zip(keys, hs):
        want = shim.shim_hash(k, len(k))
        assert int(h) == want, (k.hex(), int(h), want)
        assert hl.hash_key(k) == want
        assert int(hl.hash_tag32(h)) == shim.shim_tag32(want)
        assert int(hl.mt_filter_bit(h)) == shim.shim_filter_bit(want)


def test_random_keys_of_every_length(shim):
    rng = random.Random(5)
    keys = [rng.randbytes(n) for n in list(range(0, 65)) + [255, 256, 1000] for _ in range(8)]
    check(shim, keys)


def test_trailing_zero_bytes(shim):
    """zero padding: keys that differ only in trailing zero bytes hash apart (the length is in hash_init)"""
    base = b"abc\x00def"
    keys = [base + b"\x00" * z for z in range(0, 20)] + [b"\x00" * n for n in range(0, 20)]
    check(shim, keys)
    assert len(set(hl.hash_keys(keys).tolist())) == len(keys)


def test_candidates_and_finders_agree_with_the_header(shim):
    for klen in (1, 7, 8, 9, 15, 16, 17):
        rows = hl.candidates("cand", 3, 64, klen)
        keys = [r.tobytes() for r in rows]
        assert len(set(keys)) == len(keys) and all(len(k) == klen for k in keys)
        check(shim, keys)
    nb, ob = hl.run_layout(64, 64)
    assert (nb, ob) == (16, 7)
    for a, b in hl.run_collision_pairs(nb, ob, 4):
        ha, hb = shim.shim_hash(a, 16), shim.shim_hash(b, 16)
        assert a != b and ((ha & 0xffffffff) * nb) >> 32 == ((hb & 0xffffffff) * nb) >> 32
        assert (ha >> 32) >> ob == (hb >> 32) >> ob
    for k in hl.find_run_home(15, 16, 3):
        assert ((shim.shim_hash(k, 16) & 0xffffffff) * 16) >> 32 == 15
    for k in hl.find_mt_home(2044, 2047, 3):
        assert shim.shim_hash(k, 16) & 2047 == 2044
    for k in hl.find_filter_bit(1234, 2):
        assert shim.shim_filter_bit(shim.shim_hash(k, 16)) == 1234


def test_layout_formulas():
    # engine.cu: n_buckets = max(1, ceil(keys / 4)); ord_bits: the least b >= 1 with 2**b > entries
    assert hl.run_layout(1, 1) == (1, 1)
    assert hl.run_layout(4, 4) == (1, 3)
    assert hl.run_layout(5, 5) == (2, 3)
    assert hl.run_layout(4095, 4095) == (1024, 12)
    assert hl.run_layout(4096, 4096) == (1024, 13)
    assert hl.run_layout(65536, 65536) == (16384, 17)
    assert hl.run_layout(3, 100) == (1, 7)
    # engine.cu alloc_memtable: max(16, 2 * entries) slots rounded up to a power of two, entries = units / 7
    assert hl.mt_slot_cap(64 << 10) == 2048
    assert hl.mt_slot_cap(1 << 10) == 32
    assert hl.mt_slot_cap(0) == 1 << 15


def test_edge_keys_have_the_property_they_claim(shim):
    e = hl.load_edges()
    assert len(e["hi0_16"]) >= 2 and len(e["hi1_16"]) >= 2 and e["hi0_8"] and e["empty_mate_8"]
    for name, hi in (("hi0_16", 0), ("hi1_16", 1), ("hi0_8", 0)):
        for k in e[name]:
            h = shim.shim_hash(k, len(k))
            assert h >> 32 == hi, (name, k.hex())
            assert shim.shim_tag32(h) == 1  # stored as 1 in a memtable slot
            assert int(hl.hash_keys([k])[0]) == h
    he = shim.shim_hash(b"", 0)
    for k in e["empty_mate_8"]:
        h = shim.shim_hash(k, len(k))
        assert h >> 32 == he >> 32 and h & 31 == he & 31
