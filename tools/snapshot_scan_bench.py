"""Batched scans at snapshots (rsp_multi_scan_at_device, rsp_multi_scan_reverse_at_device) against the same scans at the
latest state (rsp_multi_scan_device, rsp_multi_scan_reverse_device) on bench.py's config-2 state.

    python tools/snapshot_scan_bench.py [--kv 10000000] [--shards 1024] [--steps 10] [--warmup 3] [--out FILE]

Loads 1024 shards x 10 M KV (16 B keys / 64 B values) through the apply path, compacts them fully and takes one snapshot
per shard, then times with CUDA events, device-resident, 16 384 scans per launch from random existing keys with
max_entries = 128 (median of the timed launches after the warm-up ones):
  - forward and reverse at the snapshots against the latest state, on the fast path (one compacted run);
  - at the snapshots, forward with the end and reverse with the low 8, 32 and 128 entries away from the start;
  - two-run views: snapshots taken anew with 50 updates per shard in the memtables (the memtable's private run and the
    compacted run: the general path).
Every launch's n_out and records are checked against the synthetic generator.  Prints one JSON line with the card's name
and power limit read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

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
    ap.add_argument("--updates", type=int, default=50, help="updates per shard in the memtables of the two-run views")
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    from rocksplicator_b200 import engine, synth
    if not torch.cuda.is_available():
        raise SystemExit("snapshot_scan_bench.py: no CUDA device")
    lib = engine.load_library()
    eng = engine.Engine(0, max_shards=max(16384, args.shards))
    stream = torch.cuda.ExternalStream(lib.rsp_engine_stream(eng.h), device=torch.device("cuda", 0))
    S, NKV = args.shards, args.kv
    shards = [eng.open_shard("segment%05d" % i, write_buffer_bytes=2 << 20) for i in range(S)]
    six_of = np.array([s.index for s in shards], dtype=np.uint32)
    seed = synth.SEED_DATA
    CH = 1 << 20

    def load(idx_all):
        for lo in range(0, idx_all.size, CH):
            idx = idx_all[lo:lo + CH]
            sh = (idx % np.uint64(S)).astype(np.int64)
            b = synth.single_put_batches(synth.keys16(seed, idx), synth.values(seed, sh, idx, 0), 1000 + idx)
            off = np.arange(idx.size + 1, dtype=np.uint64) * np.uint64(b.shape[1])
            assert not eng.apply_packed(six_of[sh], b.reshape(-1), off, 1000 + idx).any()

    load(np.arange(NKV, dtype=np.uint64))
    assert eng.compact_all() == 0
    snaps = [s.snapshot() for s in shards]

    NSC, LSC, REC = 16384, 128, 8 + 16 + 64
    K, W = args.steps, args.warmup
    n_in_shard = np.array([len(range(s, NKV, S)) for s in range(S)], dtype=np.int64)
    res = {"card": card(), "shards": S, "kv": NKV, "scans_per_launch": NSC, "max_entries": LSC, "steps": K}

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

    def slots():
        slot_of = np.array([s.slot for s in snaps], dtype=np.int32)
        with torch.cuda.stream(stream):
            d = [torch.from_numpy(slot_of[s]).cuda() for s in sh_of]
        torch.cuda.synchronize()
        return d

    d_slot = slots()

    def bound_keys(dist, reverse):
        """the key dist entries after the start (forward end, exclusive: past the shard's last key, all 0xff) or dist - 1
        below it (reverse low, inclusive: below the shard's first key, all zeros), per scan of each set"""
        out = []
        for qi, sh in zip(sc_idx, sh_of):
            j = (qi // np.uint64(S)).astype(np.int64) + (-(dist - 1) if reverse else dist)
            ok = (j >= 0) & (j < n_in_shard[sh])
            k = synth.keys16(seed, (np.clip(j, 0, n_in_shard[sh] - 1) * S + sh).astype(np.uint64))
            k[~ok] = 0 if reverse else 0xff
            with torch.cuda.stream(stream):
                out.append(torch.from_numpy(np.ascontiguousarray(k).reshape(-1)).cuda())
        torch.cuda.synchronize()
        return out

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

    def timed(reverse, at, dist=None):
        d_b = bound_keys(dist, reverse) if dist is not None else [None, None]
        sel = d_slot if at else d_ss
        if at:
            fn = lib.rsp_multi_scan_reverse_at_device if reverse else lib.rsp_multi_scan_at_device
            launch = lambda i: fn(  # noqa: E731
                eng.h, NSC, sel[i].data_ptr(), d_sk[i].data_ptr(), 16, 0,
                d_b[i].data_ptr() if d_b[i] is not None else None, 16, LSC, d_out.data_ptr(), LSC * REC,
                d_nout.data_ptr(), d_st.data_ptr(), sp)
        elif reverse:
            launch = lambda i: lib.rsp_multi_scan_reverse_device(  # noqa: E731
                eng.h, NSC, sel[i].data_ptr(), d_sk[i].data_ptr(), 16, 0,
                d_b[i].data_ptr() if d_b[i] is not None else None, 16, LSC, d_out.data_ptr(), LSC * REC,
                d_nout.data_ptr(), d_st.data_ptr(), sp)
        else:
            assert dist is None
            launch = lambda i: lib.rsp_multi_scan_device(  # noqa: E731
                eng.h, NSC, sel[i].data_ptr(), d_sk[i].data_ptr(), 16, LSC, d_out.data_ptr(), LSC * REC,
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

    # the latest state and the snapshots alternate, so that drift over the session falls on both
    for rnd in range(2):
        for name, rev, at in (("latest_forward", False, False), ("snapshot_forward", False, True),
                              ("latest_reverse", True, False), ("snapshot_reverse", True, True)):
            res.setdefault("fast_" + name + "_128", []).append(timed(rev, at))
    for dist in (8, 32, 128):
        res["fast_snapshot_forward_end_%d" % dist] = timed(False, True, dist)
        res["fast_snapshot_reverse_low_%d" % dist] = timed(True, True, dist)
    # two-run views: `updates` existing keys per shard again (same value, newer sequence) in the memtables, then one
    # snapshot per shard anew
    step = max(1, NKV // (S * args.updates))
    load(np.arange(0, NKV, step, dtype=np.uint64)[:S * args.updates])
    for s in snaps:
        s.release()
    snaps = [s.snapshot() for s in shards]
    d_slot = slots()
    res["two_run_memtable_entries_shard0"] = shards[0].stats()["memtable_entries"]
    res["two_run_forward_128"] = timed(False, True)
    res["two_run_reverse_128"] = timed(True, True)
    for s in snaps:
        s.release()
    eng.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
