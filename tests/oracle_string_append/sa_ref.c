/*
 * sa_ref.c — RocksDB's StringAppendOperator semantics on the reference's own RocksDB binary (TEST INFRASTRUCTURE, not
 * product code).
 *
 * tests/oracle_bounded/bounded_ref.c (the reference driver with snapshot reads, bounded iterators and SeekForPrev),
 * compiled into this translation unit as it is, plus okv_open_string_append: a DB opened with the options of
 * okv_open and a C-API merge operator named "StringAppendOperator" whose state holds the delimiter (0 = none,
 * 0x100 | c = the byte c).  FullMerge folds the operands oldest first onto the existing value (none: the first operand
 * alone); PartialMerge joins two or more operands with the delimiter, as AssociativeMergeOperator::PartialMerge does for
 * utilities/merge_operators/string_append.  Every other call is the driver's own.  tests/string_append_oracle.py builds
 * it next to the binary in oracle/_ref/ when the reference is available.
 */
#include "../oracle_bounded/bounded_ref.c"

okv_db* okv_open_string_append(const char* path, uint32_t delim, int wal, char* err, size_t errcap);

typedef struct sa_state {
  uint32_t delim;
} sa_state;

static char* sa_join(const sa_state* s, const char* first, size_t firstl, int has_first, const char* const* ops,
                     const size_t* opl, int from, int n, size_t* outl) {
  const size_t dl = s->delim ? 1 : 0;
  size_t tot = has_first ? firstl : 0;
  for (int i = from; i < n; i++) tot += opl[i] + ((has_first || i > from) ? dl : 0);
  char* out = (char*)malloc(tot ? tot : 1);
  size_t at = 0;
  if (has_first) {
    memcpy(out, first, firstl);
    at = firstl;
  }
  for (int i = from; i < n; i++) {
    if ((has_first || i > from) && dl) out[at++] = (char)(s->delim & 0xff);
    memcpy(out + at, ops[i], opl[i]);
    at += opl[i];
  }
  *outl = tot;
  return out;
}
static char* sa_full(void* st, const char* k, size_t kl, const char* ex, size_t exl, const char* const* ops,
                     const size_t* opl, int n, unsigned char* success, size_t* outl) {
  (void)k; (void)kl;
  *success = 1;
  return sa_join((const sa_state*)st, ex, exl, ex != NULL, ops, opl, 0, n, outl);
}
static char* sa_partial(void* st, const char* k, size_t kl, const char* const* ops, const size_t* opl, int n,
                        unsigned char* success, size_t* outl) {
  (void)k; (void)kl;
  if (n < 2) {
    *success = 0;
    return NULL;
  }
  *success = 1;
  return sa_join((const sa_state*)st, NULL, 0, 0, ops, opl, 0, n, outl);
}
static void sa_destroy(void* st) { free(st); }
static const char* sa_name(void* st) { (void)st; return "StringAppendOperator"; }

okv_db* okv_open_string_append(const char* path, uint32_t delim, int wal, char* err, size_t errcap) {
  pthread_once(&g_once, load_all);
  if (!g_loaded) {
    if (err && errcap) snprintf(err, errcap, "%s", g_load_err);
    return NULL;
  }
  okv_db* d = (okv_db*)calloc(1, sizeof(okv_db));
  d->opts = p_rocksdb_options_create();
  p_rocksdb_options_set_create_if_missing(d->opts, 1);
  p_rocksdb_options_set_compression(d->opts, 0);
  d->bbto = p_rocksdb_block_based_options_create();
  p_rocksdb_block_based_options_set_block_size(d->bbto, 4096);
  p_rocksdb_block_based_options_set_filter_policy(d->bbto, p_rocksdb_filterpolicy_create_bloom(10));
  p_rocksdb_block_based_options_set_block_cache(d->bbto, g_cache);
  p_rocksdb_options_set_block_based_table_factory(d->opts, d->bbto);
  const size_t wbs = (size_t)8 << 20;
  p_rocksdb_options_set_write_buffer_size(d->opts, wbs);
  p_rocksdb_options_set_min_write_buffer_number_to_merge(d->opts, 1);
  p_rocksdb_options_set_level0_file_num_compaction_trigger(d->opts, 4);
  p_rocksdb_options_set_max_bytes_for_level_base(d->opts, (uint64_t)wbs * 4);
  p_rocksdb_options_set_max_open_files(d->opts, -1);
  p_rocksdb_options_set_keep_log_file_num(d->opts, 1);
  p_rocksdb_options_set_info_log_level(d->opts, 3 /* ERROR */);
  sa_state* st = (sa_state*)malloc(sizeof(sa_state));
  st->delim = delim;
  p_rocksdb_options_set_merge_operator(
      d->opts, p_rocksdb_mergeoperator_create(st, sa_destroy, sa_full, sa_partial, mo_delete_value, sa_name));
  mkdir(path, 0755);
  char* e = NULL;
  d->db = p_rocksdb_open(d->opts, path, &e);
  if (e || !d->db) {
    take_err(e, err, errcap);
    p_rocksdb_options_destroy(d->opts);
    free(d);
    return NULL;
  }
  d->wo = p_rocksdb_writeoptions_create();
  if (!wal) p_rocksdb_writeoptions_disable_WAL(d->wo, 1);
  d->ro = p_rocksdb_readoptions_create();
  return d;
}
