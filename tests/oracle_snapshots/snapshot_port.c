/*
 * snapshot_port.c — snapshot reads on the oracle port (TEST INFRASTRUCTURE, not product code).
 *
 * The port (oracle/kv_oracle.c, compiled into this translation unit as it is) keeps every version in its skiplist, so
 * a snapshot is a sequence number: DB::GetSnapshot records the latest one, and Get / MultiGet / NewIterator with
 * ReadOptions::snapshot run the port's own version walk (first_visible / resolve) at it.  Built by
 * tests/snapshot_oracle.py into a library that exports oracle/okv.h plus the calls below.
 */
#include "../../oracle/kv_oracle.c"

typedef struct okv_snapshot {
  uint64_t seq;
} okv_snapshot;

okv_snapshot* okv_snapshot_create(okv_db* db);
void okv_snapshot_release(okv_db* db, okv_snapshot* s);
uint64_t okv_snapshot_seq(const okv_snapshot* s);
int okv_get_at(okv_db* db, const okv_snapshot* s, const uint8_t* key, size_t klen, uint8_t** val, size_t* vlen,
               char* err, size_t errcap);
int okv_multi_get_at(okv_db* db, const okv_snapshot* s, size_t n, const uint8_t* keys, const uint64_t* koff,
                     int32_t* st, uint8_t** vals, uint64_t* voff);
okv_iter* okv_iter_create_at(okv_db* db, const okv_snapshot* s);

okv_snapshot* okv_snapshot_create(okv_db* db) {
  okv_snapshot* s = (okv_snapshot*)calloc(1, sizeof(okv_snapshot));
  s->seq = db->last_seq;
  return s;
}
void okv_snapshot_release(okv_db* db, okv_snapshot* s) {
  (void)db;
  free(s);
}
uint64_t okv_snapshot_seq(const okv_snapshot* s) { return s->seq; }

/* okv_get's walk at the snapshot's sequence number */
int okv_get_at(okv_db* db, const okv_snapshot* s, const uint8_t* key, size_t klen, uint8_t** val, size_t* vlen,
               char* err, size_t errcap) {
  node* x = first_visible(db, key, klen, s->seq);
  *val = NULL;
  *vlen = 0;
  if (!x) return OKV_NOT_FOUND;
  buf_t out = {0, 0, 0};
  int rc = resolve(db, x, s->seq, &out, err, errcap);
  if (rc == OKV_OK) {
    *val = out.p ? out.p : (uint8_t*)malloc(1);
    *vlen = out.n;
  } else {
    free(out.p);
  }
  return rc;
}

/* okv_multi_get's loop at the snapshot's sequence number */
int okv_multi_get_at(okv_db* db, const okv_snapshot* s, size_t n, const uint8_t* keys, const uint64_t* koff,
                     int32_t* st, uint8_t** vals, uint64_t* voff) {
  buf_t all = {0, 0, 0};
  for (size_t i = 0; i < n; i++) {
    voff[i] = all.n;
    const uint8_t* k = keys + koff[i];
    size_t kl = (size_t)(koff[i + 1] - koff[i]);
    node* x = first_visible(db, k, kl, s->seq);
    if (!x) {
      st[i] = OKV_NOT_FOUND;
      continue;
    }
    buf_t out = {0, 0, 0};
    st[i] = resolve(db, x, s->seq, &out, NULL, 0);
    if (st[i] == OKV_OK) buf_append(&all, out.p, out.n);
    free(out.p);
  }
  voff[n] = all.n;
  *vals = all.p ? all.p : (uint8_t*)malloc(1);
  return OKV_OK;
}

okv_iter* okv_iter_create_at(okv_db* db, const okv_snapshot* s) {
  okv_iter* it = okv_iter_create(db);
  it->snap = s->seq;
  return it;
}
