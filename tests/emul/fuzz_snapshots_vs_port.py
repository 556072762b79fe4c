"""TEST INFRASTRUCTURE ONLY — the engine's snapshot reads against the oracle port's on seeded random streams:
snapshots are taken and released at random points while batches, flushes, compactions and background merges go on,
and every live snapshot is read (Get, cross-shard MultiGet, forward and backward walks) against the port's snapshot at
the same sequence number.

    python tests/emul/fuzz_snapshots_vs_port.py FIRST LAST      (RSP_TEST_EMUL_LIB selects the library)
"""
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import okv  # noqa: E402
from snapshot_oracle import SnapOkv, load_port  # noqa: E402
from rocksplicator_b200 import engine  # noqa: E402
from streams import random_stream  # noqa: E402


def walk(it, backward=False):
    out = []
    it.seek_to_last() if backward else it.seek_to_first()
    while it.valid():
        out.append((it.key(), it.value(), it.status()))
        it.prev() if backward else it.next()
    it.close()
    return out


def one_seed(eng, port, seed):
    rng = random.Random(seed * 131 + 7)
    mop, mname = rng.choice([(okv.MERGE_COUNTER, "counter"), (okv.MERGE_APPEND, "append"),
                             (okv.MERGE_UINT64ADD, "counter"), (okv.MERGE_NONE, None)])
    n_shards = rng.choice([1, 2, 3])
    keys, stream = random_stream(20000 + seed, rng.randint(30, 150), n_keys=rng.choice([6, 20, 60]), merge=mname,
                                 max_ops=rng.choice([2, 6, 12]), bad_operands=mop == okv.MERGE_COUNTER and rng.random() < 0.2)
    shards = [eng.open_shard("fs%d_%d" % (seed, i), merge_op=mop, write_buffer_bytes=rng.choice([0, 4096]))
              for i in range(n_shards)]
    ports = [SnapOkv(port, merge_op=mop) for _ in range(n_shards)]
    live = []  # (shard, engine snapshot, port snapshot)
    try:
        for bt, ts in stream:
            x = rng.randrange(n_shards)
            assert shards[x].apply(bt, ts) == ports[x].apply(bt, ts), (seed, "apply")
            r = rng.random()
            if r < 0.12:
                es, ps = shards[x].snapshot(), ports[x].snapshot()
                assert es.seq == ps.seq, (seed, "seq")
                live.append((x, es, ps))
            elif r < 0.18:
                shards[x].flush()
            elif r < 0.21:
                shards[x].compact()
            elif r < 0.26 and live:
                _, es, ps = live.pop(rng.randrange(len(live)))
                es.release(), ps.release()
        probe = keys + [b"zz-missing"]
        for x, es, ps in live:
            assert [es.get(k) for k in probe] == [ports[x].get(k, snapshot=ps) for k in probe], (seed, "get")
            assert walk(es.iterator()) == walk(ports[x].iterator(ps)), (seed, "walk")
            assert walk(es.iterator(), True) == walk(ports[x].iterator(ps), True), (seed, "walk back")
        if live:
            pick = [(rng.randrange(len(live)), rng.choice(probe)) for _ in range(100)]
            got = eng.multi_get_at([live[j][1] for j, _ in pick], [k for _, k in pick], stride=rng.choice([16, 256]))
            assert got == [ports[live[j][0]].get(k, snapshot=live[j][2]) for j, k in pick], (seed, "multi_get_at")
    finally:
        for _, es, ps in live:
            es.release(), ps.release()
        for s in shards:
            s.close()
        for p in ports:
            p.close()


def run(first, last, lib_path):
    engine.SO_PATH = lib_path
    port = load_port()
    eng = engine.Engine(0, arena_bytes=1 << 24, l0_compaction_trigger=2)
    bad = 0
    for seed in range(first, last):
        try:
            one_seed(eng, port, seed)
        except AssertionError as ex:
            bad += 1
            print("DIVERGE seed", seed, str(ex)[:400])
    eng.close()
    return bad


if __name__ == "__main__":
    lib = os.environ.get("RSP_TEST_EMUL_LIB", os.path.join(ROOT, "tests", "emul", "build", "librsp_b200_emul.so"))
    first, last = (int(sys.argv[1]), int(sys.argv[2])) if len(sys.argv) > 2 else (0, 40)
    print("done bad=", run(first, last, lib))
