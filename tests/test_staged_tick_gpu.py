"""A tick of >= 1024 batches grouped by shard that also holds batches too large for the fused kernels: the host stages it
(the follower's LogData(timestamp) record is copied behind each batch) and the general kernels run it.  Bit-exact
against the oracle port, with the same input as tests/test_parity_gpu.py's test_packed_tick_virtual_trailer plus the
large batches."""
import random
import struct

import pytest

from oracle import okv
from rocksplicator_b200.write_batch import WriteBatch, varint32
from streams import bench_key, bench_value

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from rocksplicator_b200 import engine
    e = engine.Engine(0)
    yield e
    e.close()


def test_grouped_tick_with_large_batches_is_staged(eng, port_lib):
    """Each shard's group holds a batch of 20 000 bytes (in shard b after the batch whose last value legally SWALLOWS
    the first bytes of the LogData record), next to small batches, merges and corrupt batches that latch shard c."""
    a, b, c = (eng.open_shard("stg%d" % i, merge_op=okv.MERGE_COUNTER) for i in range(3))
    oa, ob, oc = (okv.Okv(port_lib, merge_op=okv.MERGE_COUNTER) for _ in range(3))
    rng = random.Random(77)
    six, batches, ts = [], [], []

    def add(sh, data, t):
        six.append(sh.index)
        batches.append(data)
        ts.append(t)

    def add_big(sh, key, t):
        add(sh, WriteBatch().put(key, rng.randbytes(20_000)).put(key + b"+", b"after").data(), t)

    for i in range(700):
        wb = WriteBatch().put(bench_key(5, i), bench_value(5, 0, i, 0))
        if i % 7 == 0:
            wb.merge(b"ctr", struct.pack("<q", i))
        add(a, wb.data(), 1000 + i)
        if i == 400:
            add_big(a, b"big-a", 1000 + i)
    swallow_ts = int.from_bytes(bytes([0x41] + [0x0D] * 7), "little")
    for i in range(400):
        if i == 200:
            v = b"tail-swallows-"
            raw = bytes(8) + struct.pack("<I", 1) + b"\x01" + varint32(3) + b"swk" + varint32(len(v) + 3) + v
            swallow_at = len(batches)
            add(b, raw, swallow_ts)
        else:
            add(b, WriteBatch().put(b"k%d" % (i % 50), bytes(rng.getrandbits(8) for _ in range(rng.choice([0, 5, 64, 200])))).data(), 5 + i)
        if i == 300:
            add_big(b, b"big-b", 5 + i)
    good = WriteBatch().put(b"x", b"1").data()
    for i in range(300):
        if i == 100:
            add_big(c, b"big-c", 9)
        if i == 250:
            add(c, good[:-1], 9)        # truncated: latches shard c
        else:
            add(c, WriteBatch().put(b"c%d" % i, b"v").delete(b"c%d" % (i - 1)).data(), 9)
    assert len(batches) >= 1024 and max(map(len, batches)) >= 20_000
    st = eng.apply_many(six, batches, ts)
    want = []
    for ix, bt, t in zip(six, batches, ts):
        o = oa if ix == a.index else (ob if ix == b.index else oc)
        want.append(o.apply(bt, t))
    assert list(st) == want
    assert want[swallow_at] == 0 and want[-1] != 0
    for s, o in ((a, oa), (b, ob), (c, oc)):
        assert s.latest_seq() == o.latest_seq()
        assert s.scan() == o.scan()
    assert b.get(b"swk") == ob.get(b"swk") == (0, b"tail-swallows-" + bytes([0x03, 0x08, 0x41]))
    assert b.get(b"big-b+") == ob.get(b"big-b+") == (0, b"after")
    assert c.last_error == oc.last_error
    for s in (a, b, c):
        s.close()
