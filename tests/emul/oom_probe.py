"""Out-of-device-memory behaviour on the emulation (RSP_EMUL_DEVICE_BYTES caps the emulated device): applies are refused
with an IO error once the device is full, nothing that was acknowledged is lost or changed, closing shards gives memory
back and applies go on.  Run by tests/test_emul_cpu.py; no GPU equivalent (a GPU shared with other work is not driven
out of memory on purpose)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import okv
from rocksplicator_b200 import engine
from rocksplicator_b200.write_batch import WriteBatch
from streams import bench_key, bench_value

engine.SO_PATH = os.environ.get("RSP_TEST_EMUL_LIB", os.path.join(os.path.dirname(os.path.abspath(__file__)), "build", "librsp_b200_emul.so"))
okv.build(ref=False)
port = okv.load_port()
eng = engine.Engine(0, max_shards=64, arena_bytes=1 << 20)
S = 6
shards = [eng.open_shard("oom%05d" % i, write_buffer_bytes=256 << 10) for i in range(S)]
oracles = [okv.Okv(port) for _ in range(S)]
acked = [0] * S
refused = 0
first_refusal_round = None
for rnd in range(400):
    six, batches, ts, who = [], [], [], []
    for j in range(S):
        for i in range(40):
            k = bench_key(3, (rnd * 40 + i) * 8 + j)
            six.append(shards[j].index); batches.append(WriteBatch().put(k, bench_value(3, j, rnd * 40 + i, 0)).data()); ts.append(rnd); who.append(j)
    st = eng.apply_many(six, batches, ts)
    for j, b, t, code in zip(who, batches, ts, st):
        if code == 0:
            assert oracles[j].apply(b, t) == 0
            acked[j] += 1
        else:
            refused += 1
    if refused and first_refusal_round is None:
        first_refusal_round = rnd
    if first_refusal_round is not None and rnd > first_refusal_round + 3:
        break
assert refused > 0, "the cap was never reached: lower RSP_EMUL_DEVICE_BYTES"
# everything acknowledged is there, bit for bit, and the sequence numbers agree
for j in range(S):
    assert shards[j].latest_seq() == oracles[j].latest_seq(), (j, shards[j].latest_seq(), oracles[j].latest_seq())
    assert shards[j].scan() == oracles[j].scan(), j
# give memory back: close half of the shards; the others take applies again
for j in range(S // 2):
    shards[j].close()
more = 0
for rnd in range(400, 420):
    six, batches, ts, who = [], [], [], []
    for j in range(S // 2, S):
        for i in range(10):
            k = bench_key(3, (rnd * 40 + i) * 8 + j)
            six.append(shards[j].index); batches.append(WriteBatch().put(k, bench_value(3, j, rnd * 40 + i, 1)).data()); ts.append(rnd); who.append(j)
    st = eng.apply_many(six, batches, ts)
    for j, b, t, code in zip(who, batches, ts, st):
        if code == 0:
            assert oracles[j].apply(b, t) == 0
            more += 1
assert more > 0, "no apply succeeded after memory was given back"
for j in range(S // 2, S):
    assert shards[j].latest_seq() == oracles[j].latest_seq()
    assert shards[j].scan() == oracles[j].scan(), j
print("OOM PROBE OK: %d acknowledged before the first refusal (round %d), %d refused, %d applied after shards were closed" % (sum(acked), first_refusal_round, refused, more))
eng.close()
