"""A plain model of a shard with RocksDB's StringAppendOperator: every version of every key, in sequence order, and
the operator's rule applied at read time.  Merge(existing, operand) = operand when there is no existing value (nothing,
a Delete or a SingleDelete below), existing + delim + operand otherwise; operands fold oldest first; a Put of b"" is an
existing value.  delim is one byte or None (plain concatenation)."""
import bisect

from rocksplicator_b200.write_batch import WriteBatch

PUT, DEL, SDEL, MERGE = "put", "del", "sdel", "merge"


def batch_of(ops):
    """[(kind, key, value)] -> WriteBatch bytes"""
    wb = WriteBatch()
    for kind, k, v in ops:
        if kind == PUT:
            wb.put(k, v)
        elif kind == DEL:
            wb.delete(k)
        elif kind == SDEL:
            wb.single_delete(k)
        else:
            wb.merge(k, v)
    return wb.data()


class Model:
    def __init__(self, delim=b","):
        self.delim = delim
        self.seq = 0
        self.versions = {}  # key -> [(seq, kind, value)], oldest first

    def apply(self, ops):
        for kind, k, v in ops:
            self.seq += 1
            self.versions.setdefault(k, []).append((self.seq, kind, v))

    def get(self, key, seq=None):
        """the value of key at seq (None: latest), or None when the key is not there"""
        seq = self.seq if seq is None else seq
        ops = []
        base = None
        for s, kind, v in reversed(self.versions.get(key, [])):
            if s > seq:
                continue
            if kind == MERGE:
                ops.append(v)
                continue
            if kind == PUT:
                base = v
            break
        if not ops:
            return base
        out = base
        for o in reversed(ops):
            if out is None:
                out = o
            else:
                out = out + (self.delim or b"") + o
        return out

    def items(self, seq=None):
        """[(key, value)] of the live keys at seq, in key order"""
        out = []
        for k in sorted(self.versions):
            v = self.get(k, seq)
            if v is not None:
                out.append((k, v))
        return out

    def scan(self, seq=None, start=None, end=None, limit=None, reverse=False, exclusive=False):
        """forward: keys >= start (> start when exclusive) and < end; reverse: keys <= start (< start when exclusive)
        and >= end (the low), descending"""
        it = self.items(seq)
        keys = [k for k, _ in it]
        if not reverse:
            lo = 0 if start is None else (bisect.bisect_right(keys, start) if exclusive else bisect.bisect_left(keys, start))
            sel = [kv for kv in it[lo:] if end is None or kv[0] < end]
        else:
            hi = len(keys) if start is None else (bisect.bisect_left(keys, start) if exclusive else bisect.bisect_right(keys, start))
            sel = [kv for kv in reversed(it[:hi]) if end is None or kv[0] >= end]
        return sel if limit is None else sel[:limit]
