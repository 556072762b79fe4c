/*
 * snapshot_ref.c — snapshot reads on the reference's own RocksDB binary (TEST INFRASTRUCTURE, not product code).
 *
 * oracle/ref_driver.c, compiled into this translation unit as it is, plus DB::GetSnapshot / ReleaseSnapshot,
 * Snapshot::GetSequenceNumber and reads with ReadOptions::snapshot through the binary's C API
 * (rocksdb_create_snapshot, rocksdb_readoptions_set_snapshot), and IngestExternalFile with
 * IngestExternalFileOptions::snapshot_consistency set explicitly.  The library has to sit next to the binary in
 * oracle/_ref/ (the driver loads it from its own directory); tests/snapshot_oracle.py builds it there when the
 * reference is available, to regenerate tests/golden/snapshots.json.
 */
#include "../../oracle/ref_driver.c"

typedef struct rocksdb_snapshot_t rocksdb_snapshot_t;
typedef struct okv_snapshot {
  const rocksdb_snapshot_t* snap;
  rocksdb_readoptions_t* ro;
} okv_snapshot;

okv_snapshot* okv_snapshot_create(okv_db* d);
void okv_snapshot_release(okv_db* d, okv_snapshot* s);
uint64_t okv_snapshot_seq(const okv_snapshot* s);
int okv_get_at(okv_db* d, const okv_snapshot* s, const uint8_t* key, size_t klen, uint8_t** val, size_t* vlen,
               char* err, size_t errcap);
int okv_multi_get_at(okv_db* d, const okv_snapshot* s, size_t n, const uint8_t* keys, const uint64_t* koff,
                     int32_t* st, uint8_t** vals, uint64_t* voff);
okv_iter* okv_iter_create_at(okv_db* d, const okv_snapshot* s);
int okv_ingest_sst_consistency(okv_db* d, const char* path, int allow_global_seqno, int snapshot_consistency, char* err,
                               size_t errcap);

/* the binary was loaded RTLD_GLOBAL by the driver (okv_open): these resolve against it */
static const rocksdb_snapshot_t* (*p_create_snapshot)(rocksdb_t*);
static void (*p_release_snapshot)(rocksdb_t*, const rocksdb_snapshot_t*);
static void (*p_readoptions_set_snapshot)(rocksdb_readoptions_t*, const rocksdb_snapshot_t*);
static void (*p_set_snapshot_consistency)(rocksdb_ingestexternalfileoptions_t*, unsigned char);
/* not in the C API: SnapshotImpl::GetSequenceNumber() const, called on *(Snapshot**)rocksdb_snapshot_t */
static uint64_t (*p_snapshot_seq)(const void*);
static void load_snapshot_calls(void) {
  *(void**)(&p_create_snapshot) = dlsym(RTLD_DEFAULT, "rocksdb_create_snapshot");
  *(void**)(&p_release_snapshot) = dlsym(RTLD_DEFAULT, "rocksdb_release_snapshot");
  *(void**)(&p_readoptions_set_snapshot) = dlsym(RTLD_DEFAULT, "rocksdb_readoptions_set_snapshot");
  *(void**)(&p_set_snapshot_consistency) = dlsym(RTLD_DEFAULT, "rocksdb_ingestexternalfileoptions_set_snapshot_consistency");
  *(void**)(&p_snapshot_seq) = dlsym(RTLD_DEFAULT, "_ZNK7rocksdb12SnapshotImpl17GetSequenceNumberEv");
  if (!p_create_snapshot || !p_release_snapshot || !p_readoptions_set_snapshot || !p_set_snapshot_consistency ||
      !p_snapshot_seq) {
    fprintf(stderr, "snapshot_ref: a snapshot symbol is missing from librocksdb.so.5.4\n");
    abort();
  }
}
static pthread_once_t g_snap_once = PTHREAD_ONCE_INIT;

okv_snapshot* okv_snapshot_create(okv_db* d) {
  pthread_once(&g_snap_once, load_snapshot_calls);
  okv_snapshot* s = (okv_snapshot*)calloc(1, sizeof(okv_snapshot));
  s->snap = p_create_snapshot(d->db);
  s->ro = p_rocksdb_readoptions_create();
  p_readoptions_set_snapshot(s->ro, s->snap);
  return s;
}
void okv_snapshot_release(okv_db* d, okv_snapshot* s) {
  if (!s) return;
  p_release_snapshot(d->db, s->snap);
  p_rocksdb_readoptions_destroy(s->ro);
  free(s);
}
uint64_t okv_snapshot_seq(const okv_snapshot* s) { return p_snapshot_seq(*(void* const*)s->snap); }

/* okv_get / okv_multi_get / okv_iter_create with the snapshot's ReadOptions */
int okv_get_at(okv_db* d, const okv_snapshot* s, const uint8_t* key, size_t klen, uint8_t** val, size_t* vlen,
               char* err, size_t errcap) {
  rocksdb_readoptions_t* keep = d->ro;
  d->ro = s->ro;
  int rc = okv_get(d, key, klen, val, vlen, err, errcap);
  d->ro = keep;
  return rc;
}
int okv_multi_get_at(okv_db* d, const okv_snapshot* s, size_t n, const uint8_t* keys, const uint64_t* koff,
                     int32_t* st, uint8_t** vals, uint64_t* voff) {
  rocksdb_readoptions_t* keep = d->ro;
  d->ro = s->ro;
  int rc = okv_multi_get(d, n, keys, koff, st, vals, voff);
  d->ro = keep;
  return rc;
}
okv_iter* okv_iter_create_at(okv_db* d, const okv_snapshot* s) {
  okv_iter* it = (okv_iter*)calloc(1, sizeof(okv_iter));
  it->it = p_rocksdb_create_iterator(d->db, s->ro);
  return it;
}

/* okv_ingest_sst with snapshot_consistency set explicitly (RocksDB's default: true) */
int okv_ingest_sst_consistency(okv_db* d, const char* path, int allow_global_seqno, int snapshot_consistency, char* err,
                               size_t errcap) {
  pthread_once(&g_snap_once, load_snapshot_calls);
  rocksdb_ingestexternalfileoptions_t* io = p_rocksdb_ingestexternalfileoptions_create();
  p_rocksdb_ingestexternalfileoptions_set_move_files(io, 0);
  p_set_snapshot_consistency(io, snapshot_consistency ? 1 : 0);
  p_rocksdb_ingestexternalfileoptions_set_allow_global_seqno(io, allow_global_seqno ? 1 : 0);
  p_rocksdb_ingestexternalfileoptions_set_allow_blocking_flush(io, allow_global_seqno ? 1 : 0);
  const char* files[1] = {path};
  char* e = NULL;
  p_rocksdb_ingest_external_file(d->db, files, 1, io, &e);
  p_rocksdb_ingestexternalfileoptions_destroy(io);
  return take_err(e, err, errcap);
}
