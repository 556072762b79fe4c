#!/usr/bin/env python
"""Ingestion rate of sorted files: rsp_ingest_sorted (normal) and rsp_ingest_sorted_behind (behind), both of which build
their run on the device from the sorted input.

    python tools/ingest_bench.py [--keys 1000000,10000000] [--values 16,64] [--reps 3]

Data: N 16-byte keys (big-endian indices, so already sorted) with V-byte random values, in host memory as the callers
pass them (pageable numpy arrays of keys, values and offsets).  Each repetition ingests the file into a fresh, empty
shard (normal) or behind 1000 Puts already in a fresh allow-ingest-behind shard (behind).  Timer: host clock around the
call, which uploads the input, runs the kernels on the engine stream and returns after they finished; so the rate
includes the host-to-device transfer of the input.  "compact_pass_ms" is the engine's device time of the compaction
passes that finish the run (CUDA events, rsp_last_kernel_ms("ingest")).  keys/s and GB/s use the median call time,
GB = (key + value bytes) / 1e9.  A sample of keys is read back through rsp_multi_get_fixed and checked.  Prints one JSON
line per (N, V, form), and the card's name and power limit read in the same run."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as ex:  # the numbers stand without it, but say so
        return "unknown (%s)" % ex


def make_file(n, vlen, seed):
    idx = np.arange(n, dtype=np.uint64)
    keys = np.zeros((n, 16), dtype=np.uint8)
    keys[:, 8:] = idx.astype(">u8").view(np.uint8).reshape(n, 8)  # bytes 0..7 zero: sorted by the index
    keys[:, 0] = ord("i")
    vals = np.random.default_rng(seed).integers(0, 256, size=(n, vlen), dtype=np.uint8)
    koff = np.arange(n + 1, dtype=np.uint64) * np.uint64(16)
    voff = np.arange(n + 1, dtype=np.uint64) * np.uint64(vlen)
    return keys.reshape(-1), vals.reshape(-1), koff, voff


def verify(eng, s, keys, vals, n, vlen):
    rng = np.random.default_rng(7)
    q = np.unique(rng.integers(0, n, size=min(n, 4096)))
    qk = np.ascontiguousarray(keys.reshape(n, 16)[q]).reshape(-1)
    out = np.zeros(len(q) * 64, dtype=np.uint8)
    vl = np.zeros(len(q), dtype=np.uint32)
    st = np.full(len(q), -1, dtype=np.int32)
    assert eng.multi_get_fixed(np.full(len(q), s.index, dtype=np.uint32), qk, 16, out, 64, vl, st) == 0
    assert (st == 0).all() and (vl == vlen).all()
    got = out.reshape(len(q), 64)[:, :vlen]
    assert np.array_equal(got, vals.reshape(n, vlen)[q]), "value mismatch"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", default="1000000,10000000")
    ap.add_argument("--values", default="16,64")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    from rocksplicator_b200 import engine
    from rocksplicator_b200.write_batch import WriteBatch
    eng = engine.Engine(0)
    print(json.dumps({"card": card()}), flush=True)
    ctr = [0]
    for n in [int(x) for x in a.keys.split(",")]:
        for vlen in [int(x) for x in a.values.split(",")]:
            keys, vals, koff, voff = make_file(n, vlen, n + vlen)
            kp, vp = C.cast(keys.ctypes.data, C.c_char_p), C.cast(vals.ctypes.data, C.c_char_p)
            for form in ("normal", "behind"):
                times, dev_ms = [], []
                for rep in range(a.reps + 1):  # the first call warms the arena and the pinned staging up
                    ctr[0] += 1
                    s = eng.open_shard("ing%05d" % ctr[0], allow_ingest_behind=form == "behind")
                    if form == "behind":
                        st = eng.apply_many([s.index] * 1000, [WriteBatch().put(b"u%015d" % i, b"v").data()
                                                               for i in range(1000)], [1] * 1000)
                        assert not st.any()
                    t0 = time.perf_counter()
                    if form == "behind":
                        rc = eng.lib.rsp_ingest_sorted_behind(s.h, n, kp, koff.ctypes.data, vp, voff.ctypes.data)
                    else:
                        rc = eng.lib.rsp_ingest_sorted(s.h, n, kp, koff.ctypes.data, vp, voff.ctypes.data, 1, None)
                    t = time.perf_counter() - t0
                    assert rc == 0, (rc, s.last_error)
                    if rep == a.reps:
                        verify(eng, s, keys, vals, n, vlen)
                    if rep:
                        times.append(t)
                        dev_ms.append(eng.last_kernel_ms("ingest"))
                    s.close()
                med = statistics.median(times)
                print(json.dumps({"form": form, "keys": n, "key_bytes": 16, "value_bytes": vlen,
                                  "call_ms": [round(x * 1e3, 2) for x in times],
                                  "keys_per_s": round(n / med), "GB_per_s": round(n * (16 + vlen) / med / 1e9, 3),
                                  "compact_pass_ms": [round(x, 2) for x in dev_ms], "timer": "host clock"}),
                      flush=True)
    eng.close()
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
