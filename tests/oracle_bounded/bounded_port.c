/*
 * bounded_port.c — bounded iterators on the oracle port (TEST INFRASTRUCTURE, not product code).
 *
 * tests/oracle_snapshots/snapshot_port.c (the port with snapshot reads), compiled into this translation unit as it is,
 * plus ReadOptions::iterate_upper_bound and Iterator::SeekForPrev as RocksDB 5.4's DBIter runs them:
 *   - the forward moves (Seek, SeekToFirst, Next) stop at the first internal entry whose user key is >= the bound,
 *     before its type is looked at: keys at or beyond the bound are never merged, and a failing merge there sets no
 *     status;
 *   - SeekToLast under a bound is SeekForPrev(bound), then Prev when that landed on the bound itself;
 *   - SeekForPrev and Prev do not look at the bound.
 * tests/golden/bounded_scans.json, recorded from librocksdb.so.5.4 through bounded_ref.c, pins these rules.
 * Built by tests/bounded_oracle.py into a library that exports oracle/okv.h, the snapshot calls and the calls below.
 */
#include "../oracle_snapshots/snapshot_port.c"

/* a bounded iterator: okv_iter_valid / key / value / status / prev take it as it is (base is its first member) */
typedef struct okv_biter {
  okv_iter base;
  int has_bound;
  buf_t bound;
} okv_biter;

okv_iter* okv_iter_create_bounded(okv_db* db, const okv_snapshot* s, const uint8_t* bound, size_t blen);
void okv_iter_destroy_bounded(okv_iter* it);
void okv_biter_seek_to_first(okv_iter* it);
void okv_biter_seek_to_last(okv_iter* it);
void okv_biter_seek(okv_iter* it, const uint8_t* key, size_t klen);
void okv_biter_next(okv_iter* it);
void okv_iter_seek_for_prev(okv_iter* it, const uint8_t* key, size_t klen);

/* s == NULL: the latest state; bound == NULL: no bound (an empty bound is a bound) */
okv_iter* okv_iter_create_bounded(okv_db* db, const okv_snapshot* s, const uint8_t* bound, size_t blen) {
  okv_biter* b = (okv_biter*)calloc(1, sizeof(okv_biter));
  b->base.db = db;
  b->base.snap = s ? s->seq : db->last_seq;
  if (bound) {
    b->has_bound = 1;
    buf_set(&b->bound, bound, blen);
  }
  return &b->base;
}
void okv_iter_destroy_bounded(okv_iter* it) {
  if (!it) return;
  okv_biter* b = (okv_biter*)it;
  free(b->bound.p);
  free(b->base.key.p);
  free(b->base.val.p);
  free(b);
}

/* iter_forward_from (DBIter::FindNextUserEntry) with the upper-bound check ahead of every entry */
static void biter_forward_from(okv_biter* b, node* x) {
  okv_iter* it = &b->base;
  okv_db* db = it->db;
  it->valid = 0;
  while (x) {
    if (b->has_bound && cmp_user(node_key(x), x->klen, b->bound.p, b->bound.n) >= 0) return;
    if ((x->seqtype >> 8) > it->snap) {
      x = x->next[0];
      continue;
    }
    buf_t out = {0, 0, 0};
    int rc = resolve(db, x, it->snap, &out, NULL, 0);
    if (rc == OKV_OK) {
      buf_set(&it->key, node_key(x), x->klen);
      buf_set(&it->val, out.p, out.n);
      free(out.p);
      it->valid = 1;
      return;
    }
    free(out.p);
    if (rc != OKV_NOT_FOUND) {
      it->status = rc;
      buf_set(&it->key, node_key(x), x->klen);
      buf_set(&it->val, NULL, 0);
      it->valid = 1;
      return;
    }
    const uint8_t* k = node_key(x);
    size_t kl = x->klen;
    node* y = x->next[0];
    while (y && cmp_user(node_key(y), y->klen, k, kl) == 0) y = y->next[0];
    x = y;
  }
}

void okv_biter_seek_to_first(okv_iter* it) { biter_forward_from((okv_biter*)it, it->db->head->next[0]); }
void okv_biter_seek(okv_iter* it, const uint8_t* key, size_t klen) {
  biter_forward_from((okv_biter*)it, find_ge(it->db, key, klen, ~0ull, NULL));
}
void okv_biter_next(okv_iter* it) {
  if (!it->valid) return;
  node* x = find_ge(it->db, it->key.p, it->key.n, 0, NULL);
  while (x && cmp_user(node_key(x), x->klen, it->key.p, it->key.n) == 0) x = x->next[0];
  biter_forward_from((okv_biter*)it, x);
}
/* the last entry whose user key is <= key: every version of key sorts before (key, seq 0) */
void okv_iter_seek_for_prev(okv_iter* it, const uint8_t* key, size_t klen) {
  iter_backward_from(it, find_lt(it->db, key, klen, 0));
}
void okv_biter_seek_to_last(okv_iter* it) {
  okv_biter* b = (okv_biter*)it;
  if (!b->has_bound || !it->db->head->next[0]) {
    okv_iter_seek_to_last(it);
    return;
  }
  okv_iter_seek_for_prev(it, b->bound.p, b->bound.n);
  if (it->valid && cmp_user(it->key.p, it->key.n, b->bound.p, b->bound.n) == 0) okv_iter_prev(it);
}
