"""CPU-only: the oracle port's bounded iterators (tests/bounded_oracle.py: ReadOptions::iterate_upper_bound and
SeekForPrev) against what the reference's RocksDB binary answered on the recorded edge cases
(tests/golden/bounded_scans.json), and against the live binary on random streams when oracle/_ref is built."""
import random

import pytest

import bounded_oracle as BO
import golden_util as G
from oracle import okv
from rocksplicator_b200.write_batch import WriteBatch

CASES = G.load("bounded_scans.json")


@pytest.mark.parametrize("name", BO.case_names())
def test_port_bounded_iterators_match_reference(name):
    assert BO.run_on_oracle(BO.load_port(), name) == CASES[name]


def test_port_bounded_scan_helper():
    db = BO.BoundedOkv(BO.load_port())
    for k in (b"a1", b"a2", b"b1", b"b2", b"c"):
        assert db.apply(WriteBatch().put(k, k.upper()).data(), 0) == 0
    assert db.scan(start=b"a", end=b"b") == [(b"a1", b"A1"), (b"a2", b"A2")]
    assert db.scan(end=b"b2") == [(b"a1", b"A1"), (b"a2", b"A2"), (b"b1", b"B1")]
    assert db.scan(start=b"b", end=b"b") == []
    db.close()


def _random_run(lib, seed, merge):
    """a random stream with flushes and compactions; bounded move lists at random bounds -> every state seen"""
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
                bound = None if rng.random() < 0.1 else b"k%02d" % rng.randrange(42) + (b"0" if rng.random() < 0.3 else b"")
                it = db.iterator(upper_bound=bound)
                got = []
                for _ in range(8):
                    m = rng.randrange(6)
                    if m == 0:
                        it.seek_to_first()
                    elif m == 1:
                        it.seek_to_last()
                    elif m == 2:
                        it.seek(b"k%02d" % rng.randrange(42))
                    elif m == 3:
                        it.seek_for_prev(b"k%02d" % rng.randrange(42))
                    elif it.valid():
                        it.next() if m == 4 else it.prev()
                    got.append(BO._state(it))
                it.close()
                out.append((bound, got))
    finally:
        db.close()
    return out


@pytest.mark.skipif(not okv.ref_available(), reason="oracle/_ref is not built (the golden cases above still run)")
@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("merge", [okv.MERGE_UINT64ADD, okv.MERGE_APPEND])
def test_port_matches_live_reference_on_random_streams(seed, merge):
    assert _random_run(BO.load_port(), seed, merge) == _random_run(BO.load_ref(), seed, merge)
