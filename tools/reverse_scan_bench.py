"""Batched reverse scans (rsp_multi_scan_reverse_device) against forward scans on bench.py's config-2 state.

    python tools/reverse_scan_bench.py [--kv 10000000] [--shards 1024] [--steps 10] [--iter-only] [--out FILE]

Loads 1024 shards x 10 M KV (16 B keys / 64 B values) through the apply path and compacts them fully, then times with
CUDA events, device-resident, 16 384 scans per launch from random existing keys with max_entries = 128 (median of the
timed launches after the warm-up ones):
  - forward (rsp_multi_scan_device) against reverse from the same keys, on the fast path (one compacted run);
  - reverse with the low 8, 32 and 128 entries below the start;
  - forward against reverse after a flush without a merge (two runs per shard: the general path).
It also times one iterator's SeekForPrev + 1000 x Prev on the host clock (--iter-only: that case alone, which the
iterator API of earlier versions can run too).  Every launch's n_out and records, and every key the iterator returns,
are checked against the synthetic generator.  Prints one JSON line with the card's name and power limit read in the same
run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kv", type=int, default=10_000_000)
    ap.add_argument("--shards", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iter-only", action="store_true")
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    from rocksplicator_b200 import engine, synth
    if not torch.cuda.is_available():
        raise SystemExit("reverse_scan_bench.py: no CUDA device")
    lib = engine.load_library()
    eng = engine.Engine(0, max_shards=max(16384, args.shards))
    stream = torch.cuda.ExternalStream(lib.rsp_engine_stream(eng.h), device=torch.device("cuda", 0))
    S, NKV = args.shards, args.kv
    shards = [eng.open_shard("segment%05d" % i, write_buffer_bytes=2 << 20) for i in range(S)]
    six_of = np.array([s.index for s in shards], dtype=np.uint32)
    seed = synth.SEED_DATA
    CH = 1 << 20

    def load(step):
        for lo in range(0, NKV, CH * step):
            idx = np.arange(lo, min(NKV, lo + CH * step), step, dtype=np.uint64)
            sh = (idx % np.uint64(S)).astype(np.int64)
            b = synth.single_put_batches(synth.keys16(seed, idx), synth.values(seed, sh, idx, 0), 1000 + idx)
            off = np.arange(idx.size + 1, dtype=np.uint64) * np.uint64(b.shape[1])
            assert not eng.apply_packed(six_of[sh], b.reshape(-1), off, 1000 + idx).any()

    load(1)
    assert eng.compact_all() == 0

    NSC, LSC, REC = 16384, 128, 8 + 16 + 64
    K, W = args.steps, args.warmup
    n_in_shard = np.array([len(range(s, NKV, S)) for s in range(S)], dtype=np.int64)
    res = {"card": card(), "shards": S, "kv": NKV, "scans_per_launch": NSC, "max_entries": LSC, "steps": K}

    # ---- one iterator: SeekForPrev + 1000 x Prev (host clock: every fetch ends in a stream synchronisation)
    sh0, j0, n_prev = 0, n_in_shard[0] - 1 - 37, 1000
    it_keys = synth.keys16(seed, ((j0 - np.arange(n_prev + 1)) * S + sh0).astype(np.uint64))
    ms = []
    for k in range(W + K):
        it = shards[sh0].iterator()
        t0 = time.perf_counter()
        it.seek_for_prev(it_keys[0].tobytes())
        got = [it.key()]
        for _ in range(n_prev):
            it.prev()
            got.append(it.key())
        t1 = time.perf_counter()
        it.close()
        assert got == [r.tobytes() for r in it_keys], "iterator keys"
        if k >= W:
            ms.append((t1 - t0) * 1e3)
    res["iter_seek_for_prev_1000_prev_ms"] = {"median": float(np.median(ms)), "min": float(np.min(ms)),
                                              "max": float(np.max(ms))}
    if args.iter_only:
        eng.close()
        return emit(res, args.out)

    rng = np.random.default_rng(synth.SEED_QUERY)
    sc_idx = [rng.integers(0, NKV, size=NSC, dtype=np.uint64) for _ in range(2)]
    sh_of = [(qi % np.uint64(S)).astype(np.int64) for qi in sc_idx]
    with torch.cuda.stream(stream):
        d_sk = [torch.from_numpy(synth.keys16(seed, qi).reshape(-1)).cuda() for qi in sc_idx]
        d_ss = [torch.from_numpy(six_of[s].astype(np.int32)).cuda() for s in sh_of]
        d_out = torch.empty(NSC * LSC * REC, dtype=torch.uint8, device="cuda")
        d_nout = torch.empty(NSC, dtype=torch.int32, device="cuda")
        d_st = torch.empty(NSC, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    sp = C.c_void_p(stream.cuda_stream)

    def check(i, reverse, dist):
        """n_out and every record of the last launch on set i against the generator"""
        qi, sh = sc_idx[i], sh_of[i]
        j0 = (qi // np.uint64(S)).astype(np.int64)
        avail = j0 + 1 if reverse else n_in_shard[sh] - j0
        want_n = np.minimum(np.minimum(LSC, dist), avail)
        assert int(d_st.count_nonzero().item()) == 0, "scan status"
        n_out = d_nout.cpu().numpy()
        assert np.array_equal(n_out, want_n), "n_out"
        out = d_out.cpu().numpy().reshape(NSC, LSC, REC)
        q, r = np.nonzero(np.arange(LSC)[None, :] < want_n[:, None])
        idx = (((j0[q] - r) if reverse else (j0[q] + r)) * S + sh[q]).astype(np.uint64)
        got = out[q, r]
        assert (got[:, 0] == 16).all() and (got[:, 4] == 64).all(), "record header"
        assert np.array_equal(got[:, 8:24], synth.keys16(seed, idx)), "scan keys"
        assert np.array_equal(got[:, 24:], synth.values(seed, sh[q], idx, 0)), "scan values"
        return int(want_n.sum())

    def timed(reverse, dist=None):
        if not reverse:
            launch = lambda i: lib.rsp_multi_scan_device(  # noqa: E731
                eng.h, NSC, d_ss[i].data_ptr(), d_sk[i].data_ptr(), 16, LSC, d_out.data_ptr(), LSC * REC,
                d_nout.data_ptr(), d_st.data_ptr(), sp)
        else:
            d_lo = [None, None]
            if dist is not None:
                # low: the key dist - 1 entries below the start in its shard (below the shard's first key: all zeros)
                d_lo = []
                for qi, sh in zip(sc_idx, sh_of):
                    j_lo = (qi // np.uint64(S)).astype(np.int64) - (dist - 1)
                    lo = synth.keys16(seed, (np.maximum(j_lo, 0) * S + sh).astype(np.uint64))
                    lo[j_lo < 0] = 0
                    with torch.cuda.stream(stream):
                        d_lo.append(torch.from_numpy(np.ascontiguousarray(lo).reshape(-1)).cuda())
                torch.cuda.synchronize()
            launch = lambda i: lib.rsp_multi_scan_reverse_device(  # noqa: E731
                eng.h, NSC, d_ss[i].data_ptr(), d_sk[i].data_ptr(), 16, 0,
                d_lo[i].data_ptr() if d_lo[i] is not None else None, 16, LSC, d_out.data_ptr(), LSC * REC,
                d_nout.data_ptr(), d_st.data_ptr(), sp)
        for i in range(W):
            assert launch(i % 2) == 0
        torch.cuda.synchronize()
        ms, entries = [], 0
        for k in range(K):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            assert launch(k % 2) == 0
            b.record(stream)
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b))
            entries = check(k % 2, reverse, LSC if dist is None else dist)
        m = float(np.median(ms))
        return {"scans_per_s": NSC / (m * 1e-3), "entries_per_s": entries / (m * 1e-3), "entries_per_launch": entries,
                "ms_median": m, "ms_min": float(np.min(ms)), "ms_max": float(np.max(ms))}

    res["fast_forward_128"] = timed(False)
    res["fast_reverse_128"] = timed(True)
    for dist in (8, 32, 128):
        res["fast_reverse_low_%d" % dist] = timed(True, dist)
    # a flush without a merge: every 17th key again (same value, newer sequence) in a second run per shard
    load(17)
    assert eng.flush_all() == 0
    res["runs_per_shard"] = shards[0].stats()["n_runs"]
    res["general_forward_128"] = timed(False)
    res["general_reverse_128"] = timed(True)
    eng.close()
    emit(res, args.out)


def emit(res, out):
    line = json.dumps(res)
    print(line)
    if out:
        with open(out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
