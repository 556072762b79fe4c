"""Batched scans with an end key (rsp_multi_scan_bounded_device) on bench.py's config-2 state.

    python tools/bounded_scan_bench.py [--kv 10000000] [--shards 1024] [--steps 10] [--out FILE]

Loads 1024 shards x 10 M KV (16 B keys / 64 B values) through the apply path and compacts them fully, then times with
CUDA events, device-resident, 16 384 scans per launch from random existing keys with max_entries = 128:
  - bounded, with the end key 8, 32 and 128 entries past the start (in the start's shard);
  - unbounded (rsp_multi_scan_device), which is what a caller who wants [start, end) runs today before cutting the
    128 entries at the end key on the host.
Every launch's n_out and records are checked against the synthetic generator.  Prints one JSON line with the median of
the timed launches per case, and the card's name and power limit read in the same run.
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
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    from rocksplicator_b200 import engine, synth
    if not torch.cuda.is_available():
        raise SystemExit("bounded_scan_bench.py: no CUDA device")
    lib = engine.load_library()
    eng = engine.Engine(0, max_shards=max(16384, args.shards))
    stream = torch.cuda.ExternalStream(lib.rsp_engine_stream(eng.h), device=torch.device("cuda", 0))
    S, NKV = args.shards, args.kv
    shards = [eng.open_shard("segment%05d" % i, write_buffer_bytes=2 << 20) for i in range(S)]
    six_of = np.array([s.index for s in shards], dtype=np.uint32)
    seed = synth.SEED_DATA
    CH = 1 << 20
    for lo in range(0, NKV, CH):
        idx = np.arange(lo, min(NKV, lo + CH), dtype=np.uint64)
        sh = (idx % np.uint64(S)).astype(np.int64)
        b = synth.single_put_batches(synth.keys16(seed, idx), synth.values(seed, sh, idx, 0), 1000 + idx)
        off = np.arange(idx.size + 1, dtype=np.uint64) * np.uint64(b.shape[1])
        assert not eng.apply_packed(six_of[sh], b.reshape(-1), off, 1000 + idx).any()
    assert eng.compact_all() == 0

    NSC, LSC, REC = 16384, 128, 8 + 16 + 64
    K, W = args.steps, args.warmup
    rng = np.random.default_rng(synth.SEED_QUERY)
    sc_idx = [rng.integers(0, NKV, size=NSC, dtype=np.uint64) for _ in range(2)]
    sh_of = [(qi % np.uint64(S)).astype(np.int64) for qi in sc_idx]
    n_in_shard = np.array([len(range(s, NKV, S)) for s in range(S)], dtype=np.int64)
    with torch.cuda.stream(stream):
        d_sk = [torch.from_numpy(synth.keys16(seed, qi).reshape(-1)).cuda() for qi in sc_idx]
        d_ss = [torch.from_numpy(six_of[s].astype(np.int32)).cuda() for s in sh_of]
        d_out = torch.empty(NSC * LSC * REC, dtype=torch.uint8, device="cuda")
        d_nout = torch.empty(NSC, dtype=torch.int32, device="cuda")
        d_st = torch.empty(NSC, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    sp = C.c_void_p(stream.cuda_stream)

    def check(i, dist):
        """n_out and every record of the last launch on set i against the generator"""
        qi, sh = sc_idx[i], sh_of[i]
        j0 = (qi // np.uint64(S)).astype(np.int64)
        want_n = np.minimum(np.minimum(LSC, dist), n_in_shard[sh] - j0)
        assert int(d_st.count_nonzero().item()) == 0, "scan status"
        n_out = d_nout.cpu().numpy()
        assert np.array_equal(n_out, want_n), "n_out"
        out = d_out.cpu().numpy().reshape(NSC, LSC, REC)
        q, r = np.nonzero(np.arange(LSC)[None, :] < want_n[:, None])
        idx = ((j0[q] + r) * S + sh[q]).astype(np.uint64)
        got = out[q, r]
        assert (got[:, 0] == 16).all() and (got[:, 4] == 64).all(), "record header"
        assert np.array_equal(got[:, 8:24], synth.keys16(seed, idx)), "scan keys"
        assert np.array_equal(got[:, 24:], synth.values(seed, sh[q], idx, 0)), "scan values"
        return int(want_n.sum())

    def timed(dist):
        if dist is None:
            launch = lambda i: lib.rsp_multi_scan_device(  # noqa: E731
                eng.h, NSC, d_ss[i].data_ptr(), d_sk[i].data_ptr(), 16, LSC, d_out.data_ptr(), LSC * REC,
                d_nout.data_ptr(), d_st.data_ptr(), sp)
        else:
            # end key: the key `dist` entries past the start in its shard (past the shard's last key: one beyond it)
            d_ek = []
            for qi, sh in zip(sc_idx, sh_of):
                j_end = (qi // np.uint64(S)).astype(np.int64) + dist
                e = synth.keys16(seed, (np.minimum(j_end, n_in_shard[sh] - 1) * S + sh).astype(np.uint64))
                beyond = j_end >= n_in_shard[sh]
                e[beyond] = 0xff
                with torch.cuda.stream(stream):
                    d_ek.append(torch.from_numpy(np.ascontiguousarray(e).reshape(-1)).cuda())
            torch.cuda.synchronize()
            launch = lambda i: lib.rsp_multi_scan_bounded_device(  # noqa: E731
                eng.h, NSC, d_ss[i].data_ptr(), d_sk[i].data_ptr(), 16, d_ek[i].data_ptr(), 16, LSC, d_out.data_ptr(),
                LSC * REC, d_nout.data_ptr(), d_st.data_ptr(), sp)
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
            entries = check(k % 2, LSC if dist is None else dist)
        m = float(np.median(ms))
        return {"scans_per_s": NSC / (m * 1e-3), "entries_per_s": entries / (m * 1e-3), "entries_per_launch": entries,
                "ms_median": m, "ms_min": float(np.min(ms)), "ms_max": float(np.max(ms))}

    res = {"card": card(), "shards": S, "kv": NKV, "scans_per_launch": NSC, "max_entries": LSC, "steps": K}
    res["unbounded_128"] = timed(None)
    for dist in (8, 32, 128):
        res["bounded_%d" % dist] = timed(dist)
    eng.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
