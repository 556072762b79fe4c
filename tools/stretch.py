"""Config-2 stretch point (SURVEY §8d): a per-shard count near what fits — 48 GB of entries (96 B a key) resident on one
80 GB H100, beside the hash index, entry offsets and arena slack — loaded through the apply path,
compacted, then the same uniform MultiGet as bench.py (device-resident, CUDA events), every value of the last launch
checked.  Shows whether the roofline fraction survives TLB / L2 pressure.

    python tools/stretch.py [--kv 500000000] [--shards 1024] > stretch.json
"""
import argparse, ctypes as C, json, os, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from rocksplicator_b200 import engine, synth

ap = argparse.ArgumentParser()
ap.add_argument("--kv", type=int, default=500_000_000)
ap.add_argument("--shards", type=int, default=1024)
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
args = ap.parse_args()
S, NKV, K, W, Q = args.shards, args.kv, args.steps, args.warmup, 2048 * 4096
lib = engine.load_library()
eng = engine.Engine(0, max_shards=max(2048, S))  # (default 1 GiB arena slabs: near the HBM limit a large slab is what fails first)
shards = [eng.open_shard("segment%05d" % i, write_buffer_bytes=16 << 20) for i in range(S)]
six_of = np.array([s.index for s in shards], dtype=np.uint32)
seed = synth.SEED_DATA
t0 = time.perf_counter()
CH = 1 << 23
# the wire batches are generated on the GPU (synth.torch_single_put_batches == the numpy generator, bit for bit) in
# shard-grouped order, copied to pinned memory and handed to the packed tick: the host only moves bytes
dev = torch.device("cuda", 0)
pin_b = torch.empty((CH, 105), dtype=torch.uint8).pin_memory()
pin_i = torch.empty(CH, dtype=torch.int64).pin_memory()
six_t = torch.from_numpy(six_of.astype(np.int64)).to(dev)
for lo in range(0, NKV, CH):
    n = min(NKV, lo + CH) - lo
    idx = torch.arange(lo, lo + n, dtype=torch.int64, device=dev)
    sh = idx % S
    sh_sorted, order = torch.sort(sh, stable=True)  # grouped by shard: the packed / fused tick
    idx_o = idx[order]
    b = synth.torch_single_put_batches(seed, sh_sorted, idx_o, 0, idx_o + 1000)
    pin_b[:n].copy_(b, non_blocking=True)
    pin_i[:n].copy_(idx_o, non_blocking=True)
    six_o = six_t[sh_sorted].to(torch.int32).cpu().numpy().astype(np.uint32)
    torch.cuda.synchronize()
    off = np.arange(n + 1, dtype=np.uint64) * np.uint64(105)
    st = eng.apply_packed(six_o, pin_b[:n].numpy().reshape(-1), off, (pin_i[:n].numpy() + 1000).astype(np.uint64))
    assert not st.any(), "load failed"
    if (lo // CH) % 16 == 0:
        print("loaded %d M in %.0f s" % (lo >> 20, time.perf_counter() - t0), file=sys.stderr, flush=True)
t_load = time.perf_counter() - t0
def mem_report(tag):
    a = (C.c_uint64 * 4)()
    lib.rsp_debug_arena(eng.h, a)
    free_b, total_b = torch.cuda.mem_get_info()
    st_ = [s.stats() for s in shards]
    print("%s: runs %.1f GB in %d runs (max %d per shard), memtables %.1f GB | arena handed out %.1f GB, reserved %.1f GB, %.0f K blocks, free inside %.1f GB | device used %.1f GB (torch %.1f GB)" % (
        tag, sum(x["run_bytes"] for x in st_) / 1e9, sum(x["n_runs"] for x in st_), max(x["n_runs"] for x in st_), sum(x["memtable_bytes"] for x in st_) / 1e9,
        a[0] / 1e9, a[1] / 1e9, a[2] / 1e3, a[3] / 1e9, (total_b - free_b) / 1e9, torch.cuda.memory_reserved() / 1e9), file=sys.stderr, flush=True)
mem_report("after the load")
del pin_b, b, idx, sh, sh_sorted, order, idx_o
torch.cuda.empty_cache()
t1 = time.perf_counter()
rc_c = eng.compact_all()
mem_report("after compact_all (rc %d)" % rc_c)
assert rc_c == 0
t_compact = time.perf_counter() - t1
assert sum(s.latest_seq() for s in shards) == NKV
stats = [s.stats() for s in shards]
run_bytes = sum(x["run_bytes"] for x in stats)
stream = torch.cuda.ExternalStream(lib.rsp_engine_stream(eng.h))
rng = np.random.default_rng(synth.SEED_QUERY)
with torch.cuda.stream(stream):
    qs = [rng.integers(0, NKV, size=Q, dtype=np.uint64) for _ in range(W + K)]
    d_keys = [torch.from_numpy(synth.keys16(seed, q).reshape(-1)).cuda() for q in qs]
    d_six = [torch.from_numpy(six_of[(q % np.uint64(S)).astype(np.int64)].astype(np.int32)).cuda() for q in qs]
    d_vals = torch.empty(Q * 64, dtype=torch.uint8, device="cuda")
    d_vlen = torch.empty(Q, dtype=torch.int32, device="cuda")
    d_st = torch.empty(Q, dtype=torch.int32, device="cuda")
sp = C.c_void_p(stream.cuda_stream)
def mg(i):
    assert lib.rsp_multi_get_device(eng.h, Q, d_six[i].data_ptr(), d_keys[i].data_ptr(), 16, d_vals.data_ptr(), 64, d_vlen.data_ptr(), d_st.data_ptr(), sp) == 0
for i in range(W):
    mg(i)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(stream)
for k in range(K):
    mg(W + k)
e1.record(stream)
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / K
assert int(d_st.count_nonzero().item()) == 0
last = qs[W + K - 1]
assert np.array_equal(d_vals.cpu().numpy().reshape(Q, 64), synth.values(seed, (last % np.uint64(S)).astype(np.int64), last, 0)), "parity"
free, total = torch.cuda.mem_get_info()
peak = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists("MEASURED_PEAKS.json") else 6570.3
print(json.dumps({"what": "config-2 stretch point: %d shards x %d KV (16 B / 64 B) resident on one H100, uniform MultiGet of %d lookups per launch, values of the last launch checked" % (S, NKV, Q),
                  "run_bytes": run_bytes, "device_bytes_in_use": total - free, "load_s": t_load, "load_applies_per_s": NKV / t_load, "compact_s": t_compact,
                  "ms_per_launch": ms, "lookups_per_s": Q / ms * 1e3, "hbm_frac_of_peak_algorithmic": 168 * Q / (ms * 1e-3) / 1e9 / peak, "peak_gbs": peak}))
eng.close()
