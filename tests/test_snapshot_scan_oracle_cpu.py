"""CPU-only: the oracle port's walks at snapshots (tests/snapshot_scan_oracle.py: forward with an end, reverse with a low,
as rsp_multi_scan_at and rsp_multi_scan_reverse_at state them) against what the reference's RocksDB binary answered on
the recorded edge cases (tests/golden/snapshot_scans.json), and against the live binary on random streams with snapshots
taken at random points when oracle/_ref is built."""
import random

import pytest

import bounded_oracle as BO
import golden_util as G
import snapshot_scan_oracle as SS
from oracle import okv
from rocksplicator_b200.write_batch import WriteBatch

CASES = G.load("snapshot_scans.json")


@pytest.mark.parametrize("name", SS.case_names())
def test_port_snapshot_walks_match_reference(name):
    assert SS.run_on_oracle(SS.load_port(), name) == CASES[name]


def test_fixture_covers_every_snapshot_of_every_layout():
    for name in SS.case_names():
        layout = name.split("-", 1)[1]
        snaps = [s[1:] for s in SS.LAYOUTS[layout] if s[0] == "S"]
        assert sorted(CASES[name]) == sorted(snaps), name
        for sn in snaps:
            assert sorted(CASES[name][sn]) == sorted(SS.walk_tag(w) for w in SS.walks(layout)), (name, sn)


def _random_run(lib, seed, merge):
    """a random stream with flushes and compactions and snapshots taken at random points; every snapshot is walked at
    the end, forward to random ends and backward to random lows"""
    rng = random.Random(seed)
    keys = [b"k%02d" % i for i in range(0, 40, 2)]
    db = BO.BoundedOkv(lib, merge_op=merge)
    snaps, out = [], []
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
                if rng.random() < 0.04:
                    snaps.append(db.snapshot())
            if step % 3 == 1:
                assert db.flush() == 0
            elif step % 3 == 2:
                assert db.compact() == 0
        for snap in snaps:
            for _ in range(6):
                d = rng.choice("fr")
                start = None if rng.random() < 0.1 else b"k%02d" % rng.randrange(42)
                bound = None if rng.random() < 0.3 else b"k%02d" % rng.randrange(42) + (b"0" if rng.random() < 0.3 else b"")
                w = (d, start, rng.randrange(2), bound, rng.choice((1, 3, 100)))
                out.append(SS.run_walk(lambda ub: db.iterator(snap, ub), w))
        for snap in snaps:
            snap.release()
    finally:
        db.close()
    return out


@pytest.mark.skipif(not okv.ref_available(), reason="oracle/_ref is not built (the golden cases above still run)")
@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("merge", [okv.MERGE_UINT64ADD, okv.MERGE_APPEND])
def test_port_matches_live_reference_on_random_streams(seed, merge):
    assert _random_run(BO.load_port(), seed, merge) == _random_run(BO.load_ref(), seed, merge)
