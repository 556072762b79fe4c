"""SST interchange on the host (SURVEY §8f rank 2), CPU only.
  * the reference's golden file rocksdb_admin/tests/old_sst_data.sst (copied byte-for-byte to tests/golden/: a 978-byte
    test fixture, Snappy-compressed block) must read as key0..key9 -> value0..value9 (sst_binary.cpp:43-58);
  * files written by the reference's own SstFileWriter (librocksdb.so.5.4, stored under tests/golden/) must read back
    exactly;
  * files written by OUR writer must be those the reference's DB::IngestExternalFile accepted and scanned back exactly,
    with the sequence-number rule of rocksdb_assumption_test.cpp:248-262 (ingest into an empty DB: seq stays 0)."""
import os
import random
import tempfile

import pytest

import golden_util as G
from rocksplicator_b200 import sst

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "old_sst_data.sst")


def test_golden_old_sst_data():
    entries, props = sst.read_sst(open(GOLDEN, "rb").read())
    assert [(k, t, v) for k, _, t, v in entries] == [(b"key%d" % i, 1, b"value%d" % i) for i in range(10)]
    assert props["num_entries"] == 10
    assert all(seq == 0 for _, seq, _, _ in entries)


def test_rejects_garbage():
    with pytest.raises(ValueError):
        sst.read_sst(b"not an sst file at all, but long enough to have a footer ...............")
    data = bytearray(open(GOLDEN, "rb").read())
    data[10] ^= 0xFF  # flip a byte inside the first data block: the CRC32C must catch it
    with pytest.raises(ValueError):
        sst.read_sst(bytes(data))


def _kv(n, seed, max_v=300):
    rng = random.Random(seed)
    keys = sorted({bytes(rng.getrandbits(8) for _ in range(rng.randint(1, 40))) for _ in range(n)})
    return [(k, bytes(rng.getrandbits(8) for _ in range(rng.choice([0, 1, 8, 64, max_v])))) for k in keys]


def test_roundtrip_own_writer_reader():
    for n, seed in ((1, 1), (10, 2), (3000, 3)):
        kv = _kv(n, seed)
        entries, props = sst.read_sst(sst.write_sst(kv, block_size=512 if n > 100 else 4096))
        assert [(k, v) for k, _, _, v in entries] == kv
        assert props["external_version"] == 2 and props["num_entries"] == len(kv)
    with pytest.raises(ValueError):
        sst.write_sst([(b"b", b"1"), (b"a", b"2")])  # "Keys must be added in order"


def test_reads_files_written_by_the_reference():
    """files the reference's SstFileWriter wrote for these key / value sets, stored as deltas against the sets"""
    from oracle import gen_golden
    want = G.load("reference_runs.json")["sst_written_by_reference"]
    for n, seed in gen_golden.SST_READ_CASES:
        kv = _kv(n, seed, max_v=2000)
        with open(os.path.join(G.GOLDEN, "ref_sst_%d.delta" % n), "rb") as f:
            data = G.delta_decode(f.read(), gen_golden.sst_base(kv))
        assert G.sha256(data) == want[str(n)], n
        entries, props = sst.read_sst(data)
        assert [(k, t, v) for k, _, t, v in entries] == [(k, 1, v) for k, v in kv]
        assert props["external_version"] == 2 and props["global_seqno"] == 0 and props["num_entries"] == len(kv)


def test_reference_ingests_files_written_here():
    """the files written here are byte for byte those the reference ingested when the fixtures were made, and what it
    read back from them was this test's expectation"""
    from oracle import gen_golden
    want = G.load("reference_runs.json")["sst_ingest"]
    for n, seed in gen_golden.SST_INGEST_CASES:
        w = want[str(n)]
        kv = _kv(n, seed, max_v=1500)
        assert G.sha256(sst.write_sst(kv)) == w["file"], n
        assert w["rc"] == 0
        assert w["seq"] == 0  # ingest into an empty DB does not consume sequence numbers
        assert w["scan"] == G.digest(kv)
        assert w["gets"] == G.digest([(0, v) for _, v in kv[:: max(1, len(kv) // 50)]])
        # an overlapping second ingest is given global sequence number last+1 (rocksdb_assumption_test.cpp:272-283)
        kv2 = [(k, b"second:" + v[:5]) for k, v in kv[::3]]
        data2 = sst.write_sst(kv2)
        assert G.sha256(data2) == w["file2"], n
        assert w["rc2"] == 0 and w["seq2"] == 1
        want_kv = dict(kv)
        want_kv.update(kv2)
        assert w["scan2"] == G.digest(sorted(want_kv.items()))
        # (move_files = false: RocksDB stamps the sequence number into ITS copy; the file written here is untouched)
        assert w["file2_after"] == w["file2"]
        entries, props = sst.read_sst(data2)
        assert props["global_seqno"] == 0 and [(k, v) for k, _, _, v in entries] == kv2


def test_shard_file_helpers_host_half():
    """sst.export_file / sst.ingest_file around a stand-in shard: the file goes through the real writer and reader"""
    class Standin:
        def __init__(self, kv=()): self.kv = list(kv)
        def ingest(self, kv, allow_global_seqno=True): self.kv = list(kv); return 0
        def scan(self): return self.kv
    kv = _kv(300, 31)
    tmp = tempfile.mkdtemp(dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    path = os.path.join(tmp, "shard.sst")
    assert sst.export_file(Standin(kv), path) == len(kv)
    dst = Standin()
    assert sst.ingest_file(dst, path) == 0 and dst.kv == kv
    # the reference's own golden file (SstFileWriter output, Snappy block) loads the same way
    assert sst.ingest_file(dst, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "old_sst_data.sst")) == 0
    assert dst.kv == [(b"key%d" % i, b"value%d" % i) for i in range(10)]
