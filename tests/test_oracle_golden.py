"""Pins the oracle port (oracle/kv_oracle.c) to the reference:
  1. known-answer table measured on the reference's shipped librocksdb.so.5.4 (SURVEY.md §9),
  2. tests/golden/*.json generated from that binary by oracle/gen_golden.py,
  3. differential runs (random streams, fuzzed streams, mutated batches) against the binary's results on the same
     inputs, stored in tests/golden/reference_runs.json.
CPU only.
"""
import struct

import pytest

import golden_util as G
from oracle import okv
from rocksplicator_b200.write_batch import WriteBatch
from streams import corrupt_cases, random_stream

u64 = lambda x: struct.pack("<Q", x)  # noqa: E731


def test_wire_format_sample():
    # SURVEY §9 "Wire format (confirmed byte-for-byte)" and §8 a6 probe sample
    b = WriteBatch().put(b"k1", b"v1").delete(b"k2").merge(b"c", u64(5)).put_log_data(u64(1234))
    assert b.data().hex() == ("0000000000000000" "03000000" "01026b31027631" "00026b32"
                              "020163080500000000000000" "0308d204000000000000")
    assert WriteBatch().put(b"key", b"value").data().hex() == "00000000000000000100000001036b65790576616c7565"
    assert WriteBatch().put(b"k" * 300, b"").data()[13:15] == bytes([0xAC, 0x02])


def test_port_known_answers(port_lib):
    """§9 rows 1-13/18 — the expectations are the committed outputs of the reference binary."""
    want = {r[0]: r[1:] for r in G.load("known_answers.json")}
    db = okv.Okv(port_lib, merge_op=okv.MERGE_UINT64ADD)
    assert [db.latest_seq()] == want["fresh_seq"]
    b = WriteBatch().put(b"k1", b"v1").delete(b"k2").merge(b"c", u64(5)).put_log_data(u64(1234)).set_sequence(999)
    assert [db.apply(b.data(), 5)] == want["row2_rc"]
    assert [db.latest_seq()] == want["row2_seq"] == [3]
    assert [db.apply(WriteBatch().put_log_data(u64(1)).data(), 5)] == want["row3_rc"]
    assert [db.latest_seq()] == want["row3_seq"]
    assert [db.apply(bytes(12), 5)] == want["row4_rc"]
    assert [db.latest_seq()] == want["row4_seq"]
    db.apply(WriteBatch().merge(b"c", u64(7)).data(), 5)
    assert [db.get(b"c")[1].hex()] == want["row5_get_c"]
    db.apply(WriteBatch().merge(b"k1", u64(1)).data(), 5)
    assert [db.get(b"k1")[1].hex()] == want["row6_get_k1"]
    db.apply(WriteBatch().put(b"z", u64(100)).delete(b"z").merge(b"z", u64(3)).merge(b"z", u64(4)).data(), 5)
    assert [db.latest_seq()] == want["row7_seq"]
    assert [db.get(b"z")[1].hex()] == want["row7_get_z"]
    db.apply(WriteBatch().put(b"x", b"1").put(b"x", b"2").delete(b"x").put(b"x", b"3").delete(b"y").data(), 5)
    assert [db.latest_seq()] == want["row8_seq"]
    assert [db.get(b"x")[1].hex()] == want["row8_get_x"]
    assert [db.get(b"y")[0]] == want["row8_get_y_rc"]
    db.apply(WriteBatch().put(b"", b"").put(b"ev", b"").data(), 5)
    assert [db.get(b"")[0], db.get(b"")[1].hex()] == want["row9_get_empty"]
    assert [[[k.hex(), v.hex()] for k, v in db.scan()]] == want["row10_scan"]
    assert [[[k.hex(), v.hex()] for k, v in db.scan(start=b"k", limit=1)]] == want["row10_seek_k"]
    mg = [[rc, v.hex() if v is not None else None] for rc, v in db.multi_get([b"c", b"zz", b"c", b"k2", b"ev", b""])]
    assert [mg] == want["row11_multi_get"]
    db.flush()
    assert [[[k.hex(), v.hex()] for k, v in db.scan()]] == want["row12_scan_after_flush"]
    assert [db.latest_seq()] == want["row12_seq"]
    db.apply(WriteBatch().single_delete(b"ev").data(), 5)
    assert [db.latest_seq()] == want["row18_seq"]
    assert [db.get(b"ev")[0]] == want["row18_get_ev_rc"]
    db.close()
    db = okv.Okv(port_lib, merge_op=okv.MERGE_NONE)
    assert [db.apply(WriteBatch().merge(b"m", b"1").data(), 5)] == want["row13_write_rc"]
    assert [db.latest_seq()] == want["row13_seq"]
    rc, _ = db.get(b"m")
    assert [rc, db.last_error] == want["row13_get_rc"]
    db.close()


@pytest.mark.parametrize("case", G.load("streams.json"), ids=lambda c: c["name"])
def test_port_golden_streams(port_lib, case):
    db = okv.Okv(port_lib, merge_op=G.MERGE_IDS[case["merge"]])
    G.replay_stream_case(db, case)
    db.close()


def test_port_golden_corrupt(port_lib):
    pre = WriteBatch().put(b"pre", b"x").data()
    for c in G.load("corrupt.json"):
        db = okv.Okv(port_lib, merge_op=okv.MERGE_UINT64ADD)
        assert db.apply(pre, 1) == 0
        assert db.apply(bytes.fromhex(c["batch"]), 0x1122334455667788) == c["rc"], c["name"]
        assert db.last_error == c["msg"], c["name"]
        assert db.latest_seq() == c["seq"], c["name"]
        assert db.apply(pre, 2) == c["rc_after"], c["name"]
        assert db.last_error == c["msg_after"], c["name"]
        assert db.latest_seq() == c["seq_after"], c["name"]
        assert [[k.hex(), v.hex()] for k, v in db.scan()] == c["scan"], c["name"]
        db.close()


def test_replicator_test_vectors(port_lib):
    """rocksdb_replicator/tests/rocksdb_replicator_test.cpp:146-208: 100 batches x 2 Puts -> follower seq
    200 and every key reads back; rocksdb_assumption_test.cpp:136-187: Put/Delete/Merge +1, batch of n +n."""
    db = okv.Okv(port_lib, merge_op=okv.MERGE_APPEND)
    for i in range(100):
        s = str(i).encode()
        wb = WriteBatch().put(s + b"key", s + b"value").put(s + b"key2", s + b"value2")
        assert db.apply(wb.data(), i) == 0
        assert db.latest_seq() == 2 * (i + 1)
    for i in range(100):
        s = str(i).encode()
        assert db.get(s + b"key") == (0, s + b"value")
        assert db.get(s + b"key2") == (0, s + b"value2")
    seq = db.latest_seq()
    db.apply(WriteBatch().delete(b"a").put(b"b", b"1").put(b"c", b"2").merge(b"b", b"3").data(), 0)
    assert db.latest_seq() == seq + 4
    assert db.get(b"b") == (0, b"13")
    db.close()


def test_port_vs_reference_live(port_lib):
    """Differential: fresh random streams (not in the stream fixtures) through the port, against what the reference's
    binary returned for the same streams (tests/golden/reference_runs.json, oracle/gen_golden.py)."""
    from oracle import gen_golden
    want = G.load("reference_runs.json")
    for mop, mname, seed in gen_golden.LIVE_STREAMS:
        got = gen_golden.live_trace(port_lib, mop, mname, seed, flush=False)
        assert G.digest(got) == want["live_streams"]["%s-%d" % (mname, seed)], (mname, seed)
    cases = corrupt_cases()
    assert [name for name, _ in cases] == [w[0] for w in want["live_corrupt"]]
    for (name, bt), w in zip(cases, want["live_corrupt"]):
        a = okv.Okv(port_lib, merge_op=okv.MERGE_UINT64ADD)
        assert [name, a.apply(bt, 7), a.last_error, a.latest_seq()] == w, name
        a.close()


def test_port_vs_reference_fuzz(port_lib):
    """oracle/fuzz_port_vs_ref.py on a few seeds: flush/compaction at random points, MultiGet, iterator walks; the
    reference's traces of the same seeds are stored as fingerprints."""
    from oracle import fuzz_port_vs_ref, gen_golden
    want = G.load("reference_runs.json")["fuzz"]
    assert sorted(int(s) for s in want) == list(gen_golden.FUZZ_SEEDS)
    diverged = [s for s in gen_golden.FUZZ_SEEDS if G.digest(fuzz_port_vs_ref.trace(port_lib, s)) != want[str(s)]]
    assert not diverged, diverged


def test_port_vs_reference_corruption_fuzz(port_lib):
    """oracle/fuzz_corrupt_port_vs_ref.py on a few seeds: mutated batches, error class + text + latch + contents"""
    from oracle import fuzz_corrupt_port_vs_ref as fz
    from oracle import gen_golden
    want = G.load("reference_runs.json")["corrupt_fuzz"]
    assert sorted(int(s) for s in want) == list(gen_golden.CORRUPT_FUZZ_SEEDS)
    bad = []
    for seed in gen_golden.CORRUPT_FUZZ_SEEDS:
        got = fz.outcomes(seed, lambda mop: okv.Okv(port_lib, merge_op=mop))
        assert len(got) == len(want[str(seed)])
        for i, (ra, (rb_rc, rb_digest)) in enumerate(zip(got, want[str(seed)])):
            if G.digest(ra) != rb_digest and not fz.is_known_deviation(ra, rb_rc):
                bad.append((seed, i, ra[1], rb_rc, ra[2]))
    assert not bad, bad[:5]
