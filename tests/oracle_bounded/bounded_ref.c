/*
 * bounded_ref.c — bounded iterators on the reference's own RocksDB binary (TEST INFRASTRUCTURE, not product code).
 *
 * tests/oracle_snapshots/snapshot_ref.c (oracle/ref_driver.c with snapshot reads), compiled into this translation unit
 * as it is, plus ReadOptions::iterate_upper_bound and Iterator::SeekForPrev through the binary's C API
 * (rocksdb_readoptions_set_iterate_upper_bound, rocksdb_iter_seek_for_prev).  The C API keeps a Slice of the caller's
 * bytes in the read options, and DBIter a pointer to that Slice: a bounded iterator owns its read options and its copy
 * of the bound until it is destroyed.  Exports the same calls as bounded_port.c; tests/bounded_oracle.py builds it
 * next to the binary in oracle/_ref/ when the reference is available.
 */
#include "../oracle_snapshots/snapshot_ref.c"

typedef struct okv_biter {
  okv_iter base; /* first member: okv_iter_* take a bounded iterator as it is */
  rocksdb_readoptions_t* ro;
  char* bound;
} okv_biter;

okv_iter* okv_iter_create_bounded(okv_db* d, const okv_snapshot* s, const uint8_t* bound, size_t blen);
void okv_iter_destroy_bounded(okv_iter* it);
void okv_biter_seek_to_first(okv_iter* it);
void okv_biter_seek_to_last(okv_iter* it);
void okv_biter_seek(okv_iter* it, const uint8_t* key, size_t klen);
void okv_biter_next(okv_iter* it);
void okv_iter_seek_for_prev(okv_iter* it, const uint8_t* key, size_t klen);

static void (*p_set_iterate_upper_bound)(rocksdb_readoptions_t*, const char*, size_t);
static void (*p_iter_seek_for_prev)(rocksdb_iterator_t*, const char*, size_t);
static void load_bounded_calls(void) {
  *(void**)(&p_set_iterate_upper_bound) = dlsym(RTLD_DEFAULT, "rocksdb_readoptions_set_iterate_upper_bound");
  *(void**)(&p_iter_seek_for_prev) = dlsym(RTLD_DEFAULT, "rocksdb_iter_seek_for_prev");
  if (!p_set_iterate_upper_bound || !p_iter_seek_for_prev) {
    fprintf(stderr, "bounded_ref: a bounded-iterator symbol is missing from librocksdb.so.5.4\n");
    abort();
  }
}
static pthread_once_t g_bounded_once = PTHREAD_ONCE_INIT;

okv_iter* okv_iter_create_bounded(okv_db* d, const okv_snapshot* s, const uint8_t* bound, size_t blen) {
  pthread_once(&g_snap_once, load_snapshot_calls);
  pthread_once(&g_bounded_once, load_bounded_calls);
  okv_biter* b = (okv_biter*)calloc(1, sizeof(okv_biter));
  b->ro = p_rocksdb_readoptions_create();
  if (s) p_readoptions_set_snapshot(b->ro, s->snap);
  if (bound) {
    b->bound = (char*)malloc(blen ? blen : 1);
    if (blen) memcpy(b->bound, bound, blen);
    p_set_iterate_upper_bound(b->ro, b->bound, blen);
  }
  b->base.it = p_rocksdb_create_iterator(d->db, b->ro);
  return &b->base;
}
void okv_iter_destroy_bounded(okv_iter* it) {
  if (!it) return;
  okv_biter* b = (okv_biter*)it;
  p_rocksdb_iter_destroy(b->base.it);
  p_rocksdb_readoptions_destroy(b->ro);
  free(b->bound);
  free(b);
}
/* the binary applies the bound itself */
void okv_biter_seek_to_first(okv_iter* it) { okv_iter_seek_to_first(it); }
void okv_biter_seek_to_last(okv_iter* it) { okv_iter_seek_to_last(it); }
void okv_biter_seek(okv_iter* it, const uint8_t* key, size_t klen) { okv_iter_seek(it, key, klen); }
void okv_biter_next(okv_iter* it) { okv_iter_next(it); }
void okv_iter_seek_for_prev(okv_iter* it, const uint8_t* key, size_t klen) {
  pthread_once(&g_bounded_once, load_bounded_calls);
  p_iter_seek_for_prev(it->it, (const char*)key, klen);
}
