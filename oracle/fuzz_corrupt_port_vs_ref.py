"""Differential fuzzer for malformed WriteBatches: random mutations (byte flips, truncation, garbage tails, count and
tag edits) of valid batches through the oracle port and the reference's RocksDB — return code, error text, sequence
number, the latch on the next write, and the resulting contents must agree.  Test infrastructure only.
`python oracle/fuzz_corrupt_port_vs_ref.py FIRST LAST`."""
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import okv  # noqa: E402
from streams import random_stream  # noqa: E402


def mutate(rng, bt):
    b = bytearray(bt)
    r = rng.random()
    if r < 0.25 and len(b) > 0:
        for _ in range(rng.randint(1, 3)):
            b[rng.randrange(len(b))] = rng.getrandbits(8)
    elif r < 0.45:
        b = b[:rng.randrange(len(b) + 1)]
    elif r < 0.6:
        b += bytes(rng.getrandbits(8) for _ in range(rng.randint(1, 12)))
    elif r < 0.75 and len(b) >= 12:
        b[8:12] = (rng.choice([0, 1, 2, 255, 2 ** 32 - 1]) if rng.random() < 0.5 else rng.getrandbits(32)).to_bytes(4, "little")
    elif len(b) > 12:
        b[rng.randrange(12, len(b))] = rng.choice([0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 0x80, 0xff])
    return bytes(b)


def cases(seed, n=40):
    rng = random.Random(seed)
    mname = rng.choice(["counter", None, "append"])
    _, stream = random_stream(4000 + seed, n, n_keys=8, merge=mname, max_ops=rng.choice([1, 3, 6]))
    mop = {"counter": okv.MERGE_UINT64ADD, None: okv.MERGE_NONE, "append": okv.MERGE_APPEND}[mname]
    return mop, [(mutate(rng, bt), ts) for bt, ts in stream]


def outcome(db, pre, bt, ts):
    out = [db.apply(pre, 1)]
    out += [db.apply(bt, ts), db.last_error, db.latest_seq()]
    out += [db.apply(pre, 2), db.latest_seq()]  # the latch
    out.append(db.scan())
    return out


def outcomes(seed, make_db):
    """outcome() of every mutated batch of `seed`, each in a fresh DB from make_db(merge_op)"""
    from rocksplicator_b200.write_batch import WriteBatch
    pre = WriteBatch().put(b"pre", b"x").data()
    mop, cs = cases(seed)
    out = []
    for bt, ts in cs:
        db = make_db(mop)
        out.append(outcome(db, pre, bt, ts))
        db.close()
    return out


def is_known_deviation(ra, rb_rc):
    """a well-formed range deletion: refused here, applied by RocksDB (DESIGN.md section 9)"""
    return ra[1] == 3 and rb_rc == 0 and "outside the replicated hot path" in ra[2]


def run(first, last, a_lib=None, b_lib=None, make_a=None):
    a_lib = a_lib or okv.load_port()
    b_lib = b_lib or okv.load_ref()
    make_a = make_a or (lambda mop: okv.Okv(a_lib, merge_op=mop))
    bad = known = 0
    for seed in range(first, last):
        ras, rbs = outcomes(seed, make_a), outcomes(seed, lambda mop: okv.Okv(b_lib, merge_op=mop))
        for i, (ra, rb) in enumerate(zip(ras, rbs)):
            if ra != rb and is_known_deviation(ra, rb[1]):
                known += 1
            elif ra != rb:
                bad += 1
                print("DIVERGE seed", seed, "case", i, [x for x in zip(ra, rb) if x[0] != x[1]][:2])
    if known:
        print("known deviation (well-formed DeleteRange refused):", known)
    return bad


if __name__ == "__main__":
    print("done bad=", run(int(sys.argv[1]), int(sys.argv[2])))
