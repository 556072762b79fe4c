"""Point lookups at snapshots (k_multi_get_at) on bench.py's config-2 state, beside the main MultiGet of the same session.

    python tools/snapshot_bench.py [--kv 10000000] [--shards 1024] [--steps 10] [--out FILE]

Loads 1024 shards x 10 M KV (16 B keys / 64 B values) through the apply path and compacts them fully, then measures with
CUDA events, device-resident, 8.4 M uniform lookups per launch:
  - rsp_multi_get_device (the main MultiGet);
  - rsp_multi_get_at_device at one snapshot per shard (each view: the one compacted run);
  - the same after one apply tick of --tick updates per shard sat in the memtables when the snapshots were taken (each
    view: the memtable's private run + the compacted run);
and the host latency of rsp_snapshot_create with an empty memtable and with that tick in it.  Every timed launch's
values are checked against the values the load and the tick wrote.  Prints one JSON line, with the card's name and
power limit read in the same run.
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
    ap.add_argument("--mg-batches", type=int, default=2048)
    ap.add_argument("--tick", type=int, default=50, help="updates per shard in the memtables of the two-run case")
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    from rocksplicator_b200 import engine, synth
    if not torch.cuda.is_available():
        raise SystemExit("snapshot_bench.py: no CUDA device")
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

    Q = args.mg_batches * 4096
    K, W = args.steps, args.warmup
    rng = np.random.default_rng(synth.SEED_QUERY)
    q_idx = [rng.integers(0, NKV, size=Q, dtype=np.uint64) for _ in range(2)]
    with torch.cuda.stream(stream):
        d_keys = [torch.from_numpy(synth.keys16(seed, qi).reshape(-1)).cuda() for qi in q_idx]
        d_six = [torch.from_numpy(six_of[(qi % np.uint64(S)).astype(np.int64)].astype(np.int32)).cuda() for qi in q_idx]
        d_vals = torch.empty(Q * 64, dtype=torch.uint8, device="cuda")
        d_vlen = torch.empty(Q, dtype=torch.int32, device="cuda")
        d_st = torch.empty(Q, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    sp = C.c_void_p(stream.cuda_stream)

    def timed(launch, want_of):
        for i in range(W):
            launch(i % 2)
        torch.cuda.synchronize()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(K)]
        for k in range(K):
            ev[k][0].record(stream)
            launch(k % 2)
            ev[k][1].record(stream)
        torch.cuda.synchronize()
        ms = [a.elapsed_time(b) for a, b in ev]
        last = q_idx[(K - 1) % 2]
        assert int(d_st.count_nonzero().item()) == 0 and int((d_vlen != 64).count_nonzero().item()) == 0
        assert np.array_equal(d_vals.cpu().numpy().reshape(Q, 64), want_of(last)), "values differ from the expectation"
        return {"lookups_per_s": Q / (float(np.median(ms)) / 1e3), "ms_median": float(np.median(ms)),
                "ms_min": float(np.min(ms)), "ms_max": float(np.max(ms))}

    base = lambda qi: synth.values(seed, (qi % np.uint64(S)).astype(np.int64), qi, 0)  # noqa: E731
    res = {"card": card(), "shards": S, "kv": NKV, "lookups_per_launch": Q, "steps": K}
    res["multi_get"] = timed(lambda i: lib.rsp_multi_get_device(eng.h, Q, d_six[i].data_ptr(), d_keys[i].data_ptr(), 16,
                                                                d_vals.data_ptr(), 64, d_vlen.data_ptr(), d_st.data_ptr(), sp),
                             base)

    def snapshot_all():
        snaps, ms = [], []
        for s in shards:
            t = time.perf_counter()
            snaps.append(s.snapshot())
            ms.append((time.perf_counter() - t) * 1e3)
        slot_of = np.zeros(int(six_of.max()) + 1, dtype=np.uint32)
        for s, sn in zip(shards, snaps):
            slot_of[s.index] = sn.slot
        with torch.cuda.stream(stream):
            d_slot = [torch.from_numpy(slot_of[six_of[(qi % np.uint64(S)).astype(np.int64)]].astype(np.int32)).cuda()
                      for qi in q_idx]
        torch.cuda.synchronize()
        return snaps, d_slot, {"ms_median": float(np.median(ms)), "ms_p99": float(np.percentile(ms, 99))}

    def at(d_slot):
        return lambda i: lib.rsp_multi_get_at_device(eng.h, Q, d_slot[i].data_ptr(), d_keys[i].data_ptr(), 16,
                                                     d_vals.data_ptr(), 64, d_vlen.data_ptr(), d_st.data_ptr(), sp)

    snaps, d_slot, res["create_empty_memtable"] = snapshot_all()
    res["multi_get_at_one_run"] = timed(at(d_slot), base)
    for sn in snaps:
        sn.release()
    # one tick of updates per shard (keys 0 .. S*tick-1, version 1) stays in the memtables
    U = S * args.tick
    idx = np.arange(U, dtype=np.uint64)
    sh = (idx % np.uint64(S)).astype(np.int64)
    b = synth.single_put_batches(synth.keys16(seed, idx), synth.values(seed, sh, idx, 1), 2000 + idx)
    off = np.arange(U + 1, dtype=np.uint64) * np.uint64(b.shape[1])
    assert not eng.apply_packed(six_of[sh], b.reshape(-1), off, 2000 + idx).any()
    res["memtable_entries_per_shard"] = shards[0].stats()["memtable_entries"]

    def updated(qi):
        want = base(qi)
        new = qi < np.uint64(U)
        want[new] = synth.values(seed, (qi[new] % np.uint64(S)).astype(np.int64), qi[new], 1)
        return want
    snaps, d_slot, res["create_full_memtable"] = snapshot_all()
    res["multi_get_at_two_runs"] = timed(at(d_slot), updated)
    for sn in snaps:
        sn.release()
    eng.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
