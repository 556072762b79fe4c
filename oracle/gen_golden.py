"""Generate tests/golden/*.json from the reference's OWN RocksDB binary (oracle/_ref).

Run where oracle/_ref could be built (the reference's source tree at oracle/Makefile's REF):
    python -m oracle.gen_golden
The fixtures pin the oracle port (tests/test_oracle_golden.py, tests/test_sst_cpu.py) and the CUDA engine
(tests/test_parity_gpu.py, tests/test_zz_ingest_gpu.py) to outputs of the reference itself, so that the tests need
neither the reference nor its binary.
TEST INFRASTRUCTURE ONLY.
"""
import json
import os
import struct
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import okv  # noqa: E402
from streams import corrupt_cases, random_stream  # noqa: E402
from rocksplicator_b200.write_batch import WriteBatch  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
MERGES = {"none": okv.MERGE_NONE, "counter": okv.MERGE_COUNTER, "uint64add": okv.MERGE_UINT64ADD,
          "append": okv.MERGE_APPEND}


def snapshot(db, keys):
    """Everything the read path can observe: seq, per-key Get, MultiGet (with duplicates + a miss),
    forward scan, backward scan, a few Seeks."""
    probe = list(keys) + [b"zz-missing"] + list(keys[:3])
    it = db.iterator()
    it.seek_to_last()
    rev = []
    while it.valid():
        rev.append([it.key().hex(), it.value().hex()])
        it.prev()
    seeks = []
    for k in list(keys[:8]) + [b"", b"\x00", b"m", b"\xff\xff"]:
        it.seek(k)
        seeks.append([k.hex(), [it.key().hex(), it.value().hex()] if it.valid() else None])
    st = it.status()
    it.close()
    return {
        "seq": db.latest_seq(),
        "get": [[k.hex(), rc, v.hex() if v is not None else None] for k in probe for rc, v in [db.get(k)]],
        "multi_get": [[rc, v.hex() if v is not None else None] for rc, v in db.multi_get(probe)],
        "scan": [[k.hex(), v.hex()] for k, v in db.scan()],
        "rscan": rev,
        "seek": seeks,
        "iter_status": st,
    }


def gen_streams(ref):
    cases = []
    for merge in ("counter", "append", "uint64add", "none"):
        for seed in range(3):
            bad = merge == "counter" and seed == 2
            keys, stream = random_stream(1000 + 17 * seed + MERGES[merge], 60, n_keys=24,
                                         merge=None if merge == "none" else ("counter" if merge == "uint64add" else merge),
                                         bad_operands=bad)
            db = okv.Okv(ref, merge_op=MERGES[merge])
            steps = []
            for i, (b, ts) in enumerate(stream):
                rc = db.apply(b, ts)
                steps.append({"batch": b.hex(), "ts": ts, "rc": rc, "seq": db.latest_seq()})
                if i == 29 and not bad:
                    db.flush()
            mid = None
            if not bad:
                db.compact()
            final = snapshot(db, keys)
            db.close()
            cases.append({"name": f"{merge}-{seed}", "merge": merge, "keys": [k.hex() for k in keys],
                          "steps": steps, "final": final, "mid": mid})
    return cases


def gen_corrupt(ref):
    out = []
    pre = WriteBatch().put(b"pre", b"x").data()
    for name, b in corrupt_cases():
        db = okv.Okv(ref, merge_op=okv.MERGE_UINT64ADD)
        assert db.apply(pre, 1) == 0
        rc = db.apply(b, 0x1122334455667788)
        msg = db.last_error
        seq = db.latest_seq()
        rc2 = db.apply(pre, 2)  # the error latch (SURVEY §9 row 20)
        out.append({"name": name, "batch": b.hex(), "rc": rc, "msg": msg, "seq": seq, "rc_after": rc2,
                    "msg_after": db.last_error, "seq_after": db.latest_seq(),
                    "scan": [[k.hex(), v.hex()] for k, v in db.scan()]})
        db.close()
    return out


def gen_known_answers(ref):
    """SURVEY §9 rows 1-13 replayed on the binary (known-answer table)."""
    u64 = lambda x: struct.pack("<Q", x)  # noqa: E731
    rows = []
    db = okv.Okv(ref, merge_op=okv.MERGE_UINT64ADD)
    rows.append(["fresh_seq", db.latest_seq()])
    b = WriteBatch().put(b"k1", b"v1").delete(b"k2").merge(b"c", u64(5)).put_log_data(u64(1234)).set_sequence(999)
    rows.append(["row2_rc", db.apply(b.data(), 5)])
    rows.append(["row2_seq", db.latest_seq()])
    rows.append(["row3_rc", db.apply(WriteBatch().put_log_data(u64(1)).data(), 5)])
    rows.append(["row3_seq", db.latest_seq()])
    rows.append(["row4_rc", db.apply(bytes(12), 5)])
    rows.append(["row4_seq", db.latest_seq()])
    db.apply(WriteBatch().merge(b"c", u64(7)).data(), 5)
    rows.append(["row5_get_c", db.get(b"c")[1].hex()])
    db.apply(WriteBatch().merge(b"k1", u64(1)).data(), 5)
    rows.append(["row6_get_k1", db.get(b"k1")[1].hex()])
    db.apply(WriteBatch().put(b"z", u64(100)).delete(b"z").merge(b"z", u64(3)).merge(b"z", u64(4)).data(), 5)
    rows.append(["row7_seq", db.latest_seq()])
    rows.append(["row7_get_z", db.get(b"z")[1].hex()])
    db.apply(WriteBatch().put(b"x", b"1").put(b"x", b"2").delete(b"x").put(b"x", b"3").delete(b"y").data(), 5)
    rows.append(["row8_seq", db.latest_seq()])
    rows.append(["row8_get_x", db.get(b"x")[1].hex()])
    rows.append(["row8_get_y_rc", db.get(b"y")[0]])
    db.apply(WriteBatch().put(b"", b"").put(b"ev", b"").data(), 5)
    rows.append(["row9_get_empty", list(db.get(b""))[0], db.get(b"")[1].hex()])
    rows.append(["row10_scan", [[k.hex(), v.hex()] for k, v in db.scan()]])
    rows.append(["row10_seek_k", [[k.hex(), v.hex()] for k, v in db.scan(start=b"k", limit=1)]])
    rows.append(["row11_multi_get", [[rc, v.hex() if v is not None else None]
                                     for rc, v in db.multi_get([b"c", b"zz", b"c", b"k2", b"ev", b""])]])
    db.flush()
    rows.append(["row12_scan_after_flush", [[k.hex(), v.hex()] for k, v in db.scan()]])
    rows.append(["row12_seq", db.latest_seq()])
    db.apply(WriteBatch().single_delete(b"ev").data(), 5)
    rows.append(["row18_seq", db.latest_seq()])
    rows.append(["row18_get_ev_rc", db.get(b"ev")[0]])
    db.close()
    db = okv.Okv(ref, merge_op=okv.MERGE_NONE)
    rows.append(["row13_write_rc", db.apply(WriteBatch().merge(b"m", b"1").data(), 5)])
    rows.append(["row13_seq", db.latest_seq()])
    rc, _ = db.get(b"m")
    rows.append(["row13_get_rc", rc, db.last_error])
    db.close()
    return rows


LIVE_STREAMS = [(okv.MERGE_COUNTER, "counter", 91), (okv.MERGE_COUNTER, "counter", 92),
                (okv.MERGE_APPEND, "append", 91), (okv.MERGE_APPEND, "append", 92)]
FUZZ_SEEDS = range(200, 212)
CORRUPT_FUZZ_SEEDS = range(0, 25)
SST_READ_CASES = ((1, 11), (50, 12), (4000, 13))     # tests/test_sst_cpu.py: files the reference writes
SST_INGEST_CASES = ((1, 21), (200, 22), (5000, 23))  # tests/test_sst_cpu.py: files written here, ingested by the reference


def live_trace(lib, mop, mname, seed, flush):
    """One random stream through one DB, then every read.  The reference's run flushes after batch 40 and compacts at
    the end; the port's run does neither (its reads must not depend on where the data lives)."""
    keys, stream = random_stream(seed + mop, 80, merge=mname)
    db = okv.Okv(lib, merge_op=mop)
    out = []
    for i, (bt, ts) in enumerate(stream):
        out.append(db.apply(bt, ts))
        if flush and i == 40:
            db.flush()
    if flush:
        db.compact()
    out += [db.latest_seq(), [db.get(k) for k in keys], db.multi_get(keys), db.scan()]
    db.close()
    return out


def sst_base(kv):
    """what a reference-written SST file is delta-encoded against (tests/golden_util.py)"""
    return b"".join(k + v for k, v in kv)


def _ref_extras(ref_lib):
    """the SST entry points of the driver over the reference's binary (oracle/ref_driver.c)"""
    import ctypes as C
    ref_lib.okv_write_sst.restype = C.c_int
    ref_lib.okv_write_sst.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_void_p, C.c_char_p, C.c_void_p, C.c_char_p, C.c_size_t]
    ref_lib.okv_ingest_sst.restype = C.c_int
    ref_lib.okv_ingest_sst.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_char_p, C.c_size_t]
    return ref_lib


def gen_reference_runs(ref):
    """The reference's side of the differential tests: fingerprints of what its binary returned (golden_util.digest),
    and the SST files its SstFileWriter wrote (delta-encoded, tests/golden/ref_sst_<n>.delta)."""
    import ctypes as C
    import tempfile

    import golden_util as G
    from oracle.fuzz_corrupt_port_vs_ref import outcomes
    from oracle.fuzz_port_vs_ref import trace
    from rocksplicator_b200 import sst
    from test_sst_cpu import _kv
    out = {"live_streams": {"%s-%d" % (m, s): G.digest(live_trace(ref, mop, m, s, True)) for mop, m, s in LIVE_STREAMS}}
    live_corrupt = []
    for name, bt in corrupt_cases():
        db = okv.Okv(ref, merge_op=okv.MERGE_UINT64ADD)
        live_corrupt.append([name, db.apply(bt, 7), db.last_error, db.latest_seq()])
        db.close()
    out["live_corrupt"] = live_corrupt
    out["fuzz"] = {str(s): G.digest(trace(ref, s)) for s in FUZZ_SEEDS}
    out["corrupt_fuzz"] = {str(s): [[o[1], G.digest(o)] for o in outcomes(s, lambda mop: okv.Okv(ref, merge_op=mop))]
                           for s in CORRUPT_FUZZ_SEEDS}
    lib = _ref_extras(ref)
    tmp = tempfile.mkdtemp()
    out["sst_written_by_reference"] = {}
    for n, seed in SST_READ_CASES:
        kv = _kv(n, seed, max_v=2000)
        koff = [0]
        voff = [0]
        for k, v in kv:
            koff.append(koff[-1] + len(k))
            voff.append(voff[-1] + len(v))
        path = os.path.join(tmp, "ref%d.sst" % n)
        err = C.create_string_buffer(256)
        rc = lib.okv_write_sst(path.encode(), len(kv), b"".join(k for k, _ in kv) + b"\0", (C.c_uint64 * len(koff))(*koff),
                               b"".join(v for _, v in kv) + b"\0", (C.c_uint64 * len(voff))(*voff), err, 256)
        assert rc == 0, err.value
        data = open(path, "rb").read()
        delta = G.delta_encode(data, sst_base(kv))
        assert G.delta_decode(delta, sst_base(kv)) == data
        with open(os.path.join(OUT, "ref_sst_%d.delta" % n), "wb") as f:
            f.write(delta)
        out["sst_written_by_reference"][str(n)] = G.sha256(data)
    out["sst_ingest"] = {}
    for n, seed in SST_INGEST_CASES:
        kv = _kv(n, seed, max_v=1500)
        kv2 = [(k, b"second:" + v[:5]) for k, v in kv[::3]]
        r = {}
        db = okv.Okv(lib)
        for tag, rows in (("", kv), ("2", kv2)):
            data = sst.write_sst(rows)
            path = os.path.join(tmp, "ours%d%s.sst" % (n, tag))
            open(path, "wb").write(data)
            err = C.create_string_buffer(256)
            r["file" + tag] = G.sha256(data)
            r["rc" + tag] = lib.okv_ingest_sst(db.h, path.encode(), 1, err, 256)
            r["seq" + tag] = db.latest_seq()
            r["scan" + tag] = G.digest(db.scan())
            r["file%s_after" % tag] = G.sha256(open(path, "rb").read())
            if not tag:
                r["gets"] = G.digest([db.get(k) for k, _ in kv[:: max(1, len(kv) // 50)]])
        db.close()
        out["sst_ingest"][str(n)] = r
    out["gpu_ingest"] = gen_ingest(lib, tmp)
    return out


def gen_ingest(lib, tmp):
    """The reference's side of tests/test_zz_ingest_gpu.py::test_ingest_sequence_rules_and_contents, step for step:
    ["ingest", file hash, allow, rc], ["apply", batch hash, rc], ["check", latest seq, contents fingerprint]."""
    import ctypes as C

    import golden_util as G
    from rocksplicator_b200 import sst
    from test_zz_ingest_gpu import _kv
    db = okv.Okv(lib)
    ev = []

    def ingest(kv, allow=True):
        data = sst.write_sst(kv)
        path = os.path.join(tmp, "ingest%d.sst" % len(ev))
        open(path, "wb").write(data)
        err = C.create_string_buffer(256)
        ev.append(["ingest", G.sha256(data), allow, lib.okv_ingest_sst(db.h, path.encode(), 1 if allow else 0, err, 256)])

    def apply(data):
        ev.append(["apply", G.sha256(data), db.apply(data, 1234)])

    def check():
        ev.append(["check", db.latest_seq(), G.digest(db.scan())])

    f1 = _kv(3000, 1, lo=0, hi=1 << 20)
    ingest(f1)
    check()
    apply(WriteBatch().put(f1[10][0], b"overwritten").delete(f1[11][0]).put(b"k-new", b"v").data())
    check()
    f2 = _kv(500, 2, lo=1 << 28, hi=1 << 29)
    ingest(f2)
    check()
    f3 = sorted(dict([(k, b"third:" + v[:4]) for k, v in f1[::7]] + [(f1[11][0], b"back")]).items())
    ingest(f3)
    check()
    ingest([(f1[5][0], b"refused")], allow=False)
    check()
    apply(WriteBatch().put(f3[0][0], b"after").delete(f2[0][0]).data())
    check()
    check()  # (after the engine's full compaction)
    check()  # (after the engine refused two unsorted files)
    db.close()
    return ev


def main():
    if not okv.ref_available():
        raise SystemExit("oracle/_ref not built: run `make -C oracle ref` with the reference's source tree at REF")
    ref = okv.load_ref()
    os.makedirs(OUT, exist_ok=True)
    for name, data in (("streams.json", gen_streams(ref)), ("corrupt.json", gen_corrupt(ref)),
                       ("known_answers.json", gen_known_answers(ref)), ("reference_runs.json", gen_reference_runs(ref))):
        with open(os.path.join(OUT, name), "w") as f:
            json.dump({"generator": "oracle/gen_golden.py", "source": "rocksdb_admin/tests/librocksdb.so.5.4",
                       "cases": data}, f, separators=(",", ":"))
        print(name, os.path.getsize(os.path.join(OUT, name)), "bytes")


if __name__ == "__main__":
    main()
