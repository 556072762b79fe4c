#!/usr/bin/env python
"""Reads and compactions on RSP_MERGE_STRING_APPEND shards (RocksDB's StringAppendOperator, folded on the device),
with the host-folded RSP_MERGE_APPEND on the same data as the before number.

    python tools/string_append_bench.py [--shards 1024] [--keys 64] [--lengths 1,4,16] [--reps 20]

Data: --shards shards of --keys 16-byte keys each; every key has a base Put and L 16-byte operands, L in --lengths.  The
base and the first third of the operands are flushed into one run, the next third into a second run, the rest stays in
the memtable.  Times, each with the timer it used ("timer" in the output):
  * rsp_multi_get_device lookups/s on string append (memtable + two runs), every answer checked: CUDA events on a caller
    stream, device-resident buffers;
  * the same keys on RSP_MERGE_APPEND through the host form rsp_multi_get (each merged key is a host round trip), as
    lookups/s over a smaller batch: host clock (the call makes host round trips and returns with host buffers);
  * rsp_multi_scan_device scans/s (Seek + 16 x Next) on string append after rsp_flush_all (the device form reads runs):
    CUDA events;
  * rsp_compact_all milliseconds, and the run entries before and after: host clock around the call, which runs its
    kernels on the engine's streams and returns after they finished (events on a caller stream would not see them).
Prints one JSON line per L, and the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def key_bytes(shard, i):
    return b"%08d%08d" % (shard, i)


def base_of(shard, i):
    return b"B%015d" % (shard * 100003 + i)


def operand(shard, i, j):
    return b"o%03d%012d" % (j, shard * 7919 + i)


def expected(shard, i, L):
    return b",".join([base_of(shard, i)] + [operand(shard, i, j) for j in range(L)])


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as ex:  # the numbers stand without it, but say so
        return "unknown (%s)" % ex


def load(eng, n_shards, n_keys, L, merge_op):
    from rocksplicator_b200 import engine
    from rocksplicator_b200.write_batch import WriteBatch
    shards = [eng.open_shard("sab%05d" % s, merge_op=merge_op,
                             merge_delim=b"," if merge_op == engine.MERGE_STRING_APPEND else None)
              for s in range(n_shards)]
    cuts = [0, L // 3, 2 * L // 3, L]
    for phase in range(3):
        batches = []
        for s in range(n_shards):
            wb = WriteBatch()
            for i in range(n_keys):
                k = key_bytes(s, i)
                if phase == 0:
                    wb.put(k, base_of(s, i))
                for j in range(cuts[phase], cuts[phase + 1]):
                    wb.merge(k, operand(s, i, j))
            batches.append(wb.data())
        st = eng.apply_many([sh.index for sh in shards], batches)
        assert (st == 0).all(), "apply"
        if phase < 2:
            assert eng.flush_all() == 0
    return shards


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shards", type=int, default=1024)
    ap.add_argument("--keys", type=int, default=64)
    ap.add_argument("--lengths", default="1,4,16")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--lookups", type=int, default=1 << 18)
    ap.add_argument("--host-lookups", type=int, default=4096)
    ap.add_argument("--scans", type=int, default=1 << 14)
    args = ap.parse_args()
    import torch
    from rocksplicator_b200 import engine
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this benchmark measures the GPU and has no CPU arm")
    print(json.dumps({"card": card()}), flush=True)
    rng = np.random.default_rng(7)
    S, K = args.shards, args.keys
    for L in [int(x) for x in args.lengths.split(",")]:
        res = {"L": L, "shards": S, "keys_per_shard": K}
        vmax = 16 + L * 17
        stride = (vmax + 15) & ~15
        # ---- string append: device-form MultiGet
        eng = engine.Engine(0, max_shards=S, l0_compaction_trigger=8)
        shards = load(eng, S, K, L, engine.MERGE_STRING_APPEND)
        n = args.lookups
        qs, qi = rng.integers(0, S, n), rng.integers(0, K, n)
        keys = np.frombuffer(b"".join(key_bytes(int(s), int(i)) for s, i in zip(qs, qi)), np.uint8)
        six = np.array([shards[int(s)].index for s in qs], np.uint32)
        d_six, d_keys = torch.from_numpy(six).cuda(), torch.from_numpy(keys.copy()).cuda()
        d_vals = torch.zeros(n * stride, dtype=torch.uint8, device="cuda")
        d_vlen = torch.zeros(n, dtype=torch.int32, device="cuda")
        d_st = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        stream = torch.cuda.Stream()

        def mg():
            assert eng.lib.rsp_multi_get_device(eng.h, n, d_six.data_ptr(), d_keys.data_ptr(), 16, d_vals.data_ptr(),
                                                stride, d_vlen.data_ptr(), d_st.data_ptr(), stream.cuda_stream) == 0

        def timed(fn, reps):
            for _ in range(3):
                fn()
            stream.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(reps):
                fn()
            e1.record(stream)
            e1.synchronize()
            return e0.elapsed_time(e1) / reps

        ms = timed(mg, args.reps)
        st, vlen, vals = d_st.cpu().numpy(), d_vlen.cpu().numpy(), d_vals.cpu().numpy()
        assert (st == 0).all(), "statuses"
        for q in rng.integers(0, n, 2048):
            assert vals[q * stride:q * stride + vlen[q]].tobytes() == expected(int(qs[q]), int(qi[q]), L), "value"
        res["string_append_multi_get_device"] = {"lookups_per_s": n / (ms * 1e-3), "ms": ms, "lookups": n,
                                                 "timer": "cuda_events"}
        # ---- scans (runs only: flush the memtables first)
        assert eng.flush_all() == 0
        ns, M = args.scans, 16
        rec = 8 + 16 + vmax
        sstride = (M * rec + 15) & ~15
        sq, si = rng.integers(0, S, ns), rng.integers(0, max(1, K - M), ns)
        skeys = np.frombuffer(b"".join(key_bytes(int(s), int(i)) for s, i in zip(sq, si)), np.uint8)
        d_ss = torch.from_numpy(np.array([shards[int(s)].index for s in sq], np.uint32)).cuda()
        d_sk = torch.from_numpy(skeys.copy()).cuda()
        d_out = torch.zeros(ns * sstride, dtype=torch.uint8, device="cuda")
        d_nout = torch.zeros(ns, dtype=torch.int32, device="cuda")
        d_sst = torch.full((ns,), -1, dtype=torch.int32, device="cuda")

        def sc():
            assert eng.lib.rsp_multi_scan_device(eng.h, ns, d_ss.data_ptr(), d_sk.data_ptr(), 16, M, d_out.data_ptr(),
                                                 sstride, d_nout.data_ptr(), d_sst.data_ptr(), stream.cuda_stream) == 0

        ms = timed(sc, args.reps)
        from rocksplicator_b200.engine import _scan_records
        out, nout, sst = d_out.cpu().numpy(), d_nout.cpu().numpy(), d_sst.cpu().numpy()
        recs = _scan_records(out, nout, sst, ns, sstride)
        for q in rng.integers(0, ns, 512):
            s, i = int(sq[q]), int(si[q])
            want = [(key_bytes(s, j), expected(s, j, L)) for j in range(i, min(K, i + M))]
            assert recs[q] == (0, want), "scan"
        res["string_append_scan_device"] = {"scans_per_s": ns / (ms * 1e-3), "ms": ms, "scans": ns, "entries": M,
                                            "timer": "cuda_events"}
        # ---- compaction
        before = sum(sh.stats()["run_entries"] for sh in shards)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        assert eng.compact_all() == 0
        torch.cuda.synchronize()
        cms = (time.perf_counter() - t0) * 1e3
        after = sum(sh.stats()["run_entries"] for sh in shards)
        assert after == S * K, "one Put per key after the full compaction"
        mg()
        stream.synchronize()
        st, vlen, vals = d_st.cpu().numpy(), d_vlen.cpu().numpy(), d_vals.cpu().numpy()
        for q in rng.integers(0, n, 512):
            assert st[q] == 0 and vals[q * stride:q * stride + vlen[q]].tobytes() == expected(int(qs[q]), int(qi[q]), L)
        res["compact_all"] = {"ms": cms, "run_entries_before": before, "run_entries_after": after, "timer": "host_clock"}
        eng.close()
        # ---- before: host-folded RSP_MERGE_APPEND (no delimiter), host-form MultiGet
        eng = engine.Engine(0, max_shards=S, l0_compaction_trigger=8)
        shards = load(eng, S, K, L, engine.MERGE_APPEND)
        hn = args.host_lookups
        hkeys = [key_bytes(int(qs[q]), int(qi[q])) for q in range(hn)]
        hsix = [shards[int(qs[q])].index for q in range(hn)]
        eng.multi_get(hsix[:64], hkeys[:64], stride=stride)  # warm-up
        t0 = time.perf_counter()
        got = eng.multi_get(hsix, hkeys, stride=stride)
        hms = (time.perf_counter() - t0) * 1e3
        for q in range(0, hn, 97):
            assert got[q] == (0, expected(int(qs[q]), int(qi[q]), L).replace(b",", b"")), "append value"
        res["append_host_multi_get"] = {"lookups_per_s": hn / (hms * 1e-3), "ms": hms, "lookups": hn, "timer": "host_clock"}
        eng.close()
        print(json.dumps(res), flush=True)
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
