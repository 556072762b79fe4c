"""CPU-only: the oracle port's reverse walks (tests/reverse_oracle.py: SeekForPrev / SeekToLast + Prev down to a low, as
rsp_multi_scan_reverse states them) against what the reference's RocksDB binary answered on the recorded edge cases
(tests/golden/reverse_scans.json), and against the live binary on random streams when oracle/_ref is built."""
import random

import pytest

import bounded_oracle as BO
import golden_util as G
import reverse_oracle as RO
from oracle import okv
from rocksplicator_b200.write_batch import WriteBatch

CASES = G.load("reverse_scans.json")


@pytest.mark.parametrize("name", RO.case_names())
def test_port_reverse_walks_match_reference(name):
    assert RO.run_on_oracle(RO.load_port(), name) == CASES[name]


def test_expected_scan_separates_excluded_and_low_statuses():
    """the port pins what the binary's sticky status hides: a failing merge on an excluded start key or below the low
    raises nothing in the scan; one among the keys taken does"""
    db = BO.BoundedOkv(BO.load_port(), merge_op=okv.MERGE_COUNTER)
    for k in (b"a", b"c", b"e"):
        assert db.apply(WriteBatch().put(k, k.upper()).data(), 0) == 0
    for k in (b"b", b"d"):
        assert db.apply(WriteBatch().put(k, b"abc").data(), 0) == 0
        assert db.apply(WriteBatch().merge(k, (5).to_bytes(8, "little")).data(), 0) == 0

    def scan(key, exclusive, low):
        it = db.iterator()
        w = RO.reverse_walk(it, key, exclusive, low, 100)
        it.close()
        return RO.expected_scan(w)

    st, recs = scan(b"d", 1, b"c")  # d excluded, b below the low
    assert st == 0 and recs == [(b"c", b"C")]
    st, recs = scan(b"d", 0, b"c")  # d taken
    assert st != 0 and recs == [(b"d", b""), (b"c", b"C")]
    st, recs = scan(b"e", 0, b"c")  # d taken after a good key
    assert st != 0 and [k for k, _ in recs] == [b"e", b"d", b"c"]
    db.close()


def _random_run(lib, seed, merge):
    """a random stream with flushes and compactions; reverse walks from random starts down to random lows"""
    rng = random.Random(seed)
    keys = [b"k%02d" % i for i in range(0, 40, 2)]
    db = BO.BoundedOkv(lib, merge_op=merge)
    out = []
    try:
        for step in range(6):
            for _ in range(25):
                k, r = rng.choice(keys), rng.random()
                wb = WriteBatch()
                if r < 0.5:
                    wb.put(k, b"v%d" % rng.randrange(1000))
                elif r < 0.7:
                    wb.delete(k)
                else:
                    wb.merge(k, rng.randrange(1 << 32).to_bytes(8, "little"))
                assert db.apply(wb.data(), 0) == 0
            if step % 3 == 1:
                assert db.flush() == 0
            elif step % 3 == 2:
                assert db.compact() == 0
            for _ in range(12):
                start = None if rng.random() < 0.1 else b"k%02d" % rng.randrange(42)
                low = None if rng.random() < 0.3 else b"k%02d" % rng.randrange(42) + (b"0" if rng.random() < 0.3 else b"")
                it = db.iterator()
                out.append(RO.reverse_walk(it, start, rng.randrange(2), low, rng.choice((1, 3, 100))))
                it.close()
    finally:
        db.close()
    return out


@pytest.mark.skipif(not okv.ref_available(), reason="oracle/_ref is not built (the golden cases above still run)")
@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("merge", [okv.MERGE_UINT64ADD, okv.MERGE_APPEND])
def test_port_matches_live_reference_on_random_streams(seed, merge):
    assert _random_run(BO.load_port(), seed, merge) == _random_run(BO.load_ref(), seed, merge)
