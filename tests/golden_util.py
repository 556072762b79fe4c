"""Replay helpers shared by the oracle tests and the GPU parity tests.

A "db" is anything with the Okv method set: apply(batch, ts) -> rc, latest_seq(), get(k) -> (rc, v),
multi_get(keys) -> [(rc, v)], scan(start=None, limit=None), iterator() (seek/seek_to_last/next/prev/
valid/key/value/status/close), flush(), compact(), last_error.
"""
import hashlib
import json
import os
import zlib

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MERGE_IDS = {"none": 0, "counter": 1, "uint64add": 2, "append": 3}


def load(name):
    with open(os.path.join(GOLDEN, name)) as f:
        return json.load(f)["cases"]


def sha256(data):
    return hashlib.sha256(data).hexdigest()


def digest(obj):
    """fingerprint of a result made of ints, strings, bytes, None, tuples and lists (what the oracle returns)"""
    return sha256(repr(obj).encode())[:32]


# A file the reference wrote is stored as a delta against `base`, bytes the test can regenerate (the keys and values the
# file holds): [varint literal length][literal bytes][varint copy offset][varint copy length] ..., zlib-compressed.
def _varint(x):
    out = bytearray()
    while x >= 0x80:
        out.append(x & 0x7F | 0x80)
        x >>= 7
    out.append(x)
    return bytes(out)


def _read_varint(buf, p):
    x = shift = 0
    while True:
        b = buf[p]
        p += 1
        x |= (b & 0x7F) << shift
        shift += 7
        if b < 0x80:
            return x, p


def delta_encode(target, base, w=8):
    index = {}
    for i in range(len(base) - w, -1, -1):
        index[base[i:i + w]] = i
    out, lit, p, last = bytearray(), bytearray(), 0, 0
    while p < len(target):
        j = last if target[p:p + w] == base[last:last + w] else index.get(target[p:p + w], -1)
        if j < 0 or p + w > len(target):
            lit.append(target[p])
            p += 1
            continue
        n = w
        while p + n < len(target) and j + n < len(base) and target[p + n] == base[j + n]:
            n += 1
        out += _varint(len(lit)) + lit + _varint(j) + _varint(n)
        lit = bytearray()
        p, last = p + n, j + n
    out += _varint(len(lit)) + lit + _varint(0) + _varint(0)
    return zlib.compress(bytes(out), 9)


def delta_decode(delta, base):
    buf, p, out = zlib.decompress(delta), 0, bytearray()
    while p < len(buf):
        n, p = _read_varint(buf, p)
        out += buf[p:p + n]
        p += n
        j, p = _read_varint(buf, p)
        n, p = _read_varint(buf, p)
        out += base[j:j + n]
    return bytes(out)


def unhex(x):
    return None if x is None else bytes.fromhex(x)


def check_snapshot(db, keys, snap, tag=""):
    probe = list(keys) + [b"zz-missing"] + list(keys[:3])
    assert db.latest_seq() == snap["seq"], tag
    for (khex, rc, vhex), k in zip(snap["get"], probe):
        assert bytes.fromhex(khex) == k
        got = db.get(k)
        assert got == (rc, unhex(vhex)), (tag, "get", khex, got, rc, vhex)
    got = db.multi_get(probe)
    want = [(rc, unhex(v)) for rc, v in snap["multi_get"]]
    assert got == want, (tag, "multi_get")
    want_scan = [(bytes.fromhex(k), bytes.fromhex(v)) for k, v in snap["scan"]]
    assert db.scan() == want_scan, (tag, "scan")
    it = db.iterator()
    it.seek_to_last()
    rev = []
    while it.valid():
        rev.append((it.key(), it.value()))
        it.prev()
    assert rev == [(bytes.fromhex(k), bytes.fromhex(v)) for k, v in snap["rscan"]], (tag, "rscan")
    for khex, want in snap["seek"]:
        it.seek(bytes.fromhex(khex))
        if want is None:
            assert not it.valid(), (tag, "seek", khex)
        else:
            assert it.valid(), (tag, "seek", khex)
            assert (it.key(), it.value()) == (bytes.fromhex(want[0]), bytes.fromhex(want[1])), (tag, "seek", khex)
    assert it.status() == snap["iter_status"], (tag, "iter_status")
    it.close()


def replay_stream_case(db, case, flush_at=29, do_flush=True):
    keys = [bytes.fromhex(k) for k in case["keys"]]
    bad = case["name"] == "counter-2"  # malformed counter operands: the reference run did not flush
    for i, st in enumerate(case["steps"]):
        rc = db.apply(bytes.fromhex(st["batch"]), st["ts"])
        assert rc == st["rc"], (case["name"], i, rc, st["rc"], getattr(db, "last_error", ""))
        assert db.latest_seq() == st["seq"], (case["name"], i)
        if do_flush and i == flush_at and not bad:
            db.flush()
    if do_flush and not bad:
        db.compact()
    check_snapshot(db, keys, case["final"], case["name"])
