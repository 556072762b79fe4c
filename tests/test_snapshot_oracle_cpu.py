"""CPU-only: the oracle port's snapshot reads (tests/snapshot_oracle.py: okv_snapshot_create, okv_get_at, okv_multi_get_at,
okv_iter_create_at) against what the reference's RocksDB binary answered on the same scenarios
(tests/golden/snapshots.json)."""
import pytest

import golden_util as G
import snapshot_oracle as SO
import snapshot_streams as S

CASES = G.load("snapshots.json")


@pytest.mark.parametrize("merge,seed", S.STREAM_CASES, ids=lambda x: str(x))
def test_port_snapshot_streams_match_reference(merge, seed):
    db = SO.SnapOkv(SO.load_port(), merge_op=S.MERGES[merge])
    got = S.run_stream(S.OkvSide(db), merge, seed, G.digest)
    db.close()
    assert got == CASES["streams"]["%s-%d" % (merge, seed)]


def test_port_snapshot_seq_and_isolation():
    from rocksplicator_b200.write_batch import WriteBatch
    db = SO.SnapOkv(SO.load_port())
    assert db.apply(WriteBatch().put(b"a", b"1").data(), 1) == 0
    s = db.snapshot()
    assert s.seq == db.latest_seq() == 1
    assert db.apply(WriteBatch().put(b"a", b"2").delete(b"a").put(b"b", b"3").data(), 1) == 0
    assert db.get(b"a", snapshot=s) == (0, b"1") and db.get(b"a") == (1, None)
    assert db.multi_get([b"a", b"b"], snapshot=s) == [(0, b"1"), (1, None)]
    assert db.scan(snapshot=s) == [(b"a", b"1")]
    s.release()
    db.close()
