// rocksdb/options.h — option structs named by the reference's call sites.  Only the fields the hot path
// reads are honoured by the GPU engine (write_buffer_size, merge_operator, level0 trigger).
#pragma once
#include <cstdint>
#include <memory>
#include <string>

namespace rocksdb {
class MergeOperator;
class Snapshot;
class Slice;
struct WriteOptions { bool sync = false; bool disableWAL = false; };
// snapshot: read as of DB::GetSnapshot's handle (nullptr = the latest state)
struct ReadOptions {
  bool verify_checksums = true;
  bool fill_cache = true;
  const Snapshot* snapshot = nullptr;
  // exclusive upper bound of an iterator's forward moves (bytewise); the Slice must outlive the iterator
  const Slice* iterate_upper_bound = nullptr;
};
struct CompactRangeOptions { bool change_level = false; int target_level = -1; };
struct FlushOptions { bool wait = true; };
// rocksdb_admin/admin_handler.cpp:1820-1828 sets move_files and allow_global_seqno, the rest stay default
struct IngestExternalFileOptions {
  bool move_files = false;
  bool snapshot_consistency = true;
  bool allow_global_seqno = true;
  bool allow_blocking_flush = true;
  // RocksDB 5.7: the file goes below everything the DB holds (needs DBOptions::allow_ingest_behind)
  bool ingest_behind = false;
};
// admin_handler.cpp:1669-1688 reads allow_ingest_behind through DB::GetDBOptions()
struct DBOptions {
  // keep the bottom level for files ingested behind: no compaction is bottom-most, tombstones are never dropped
  bool allow_ingest_behind = false;
};
struct Options : DBOptions {
  bool create_if_missing = false;
  bool error_if_exists = false;
  size_t write_buffer_size = 64 << 20;
  int max_write_buffer_number = 2;
  int min_write_buffer_number_to_merge = 1;
  int level0_file_num_compaction_trigger = 4;
  int num_levels = 7;
  uint64_t WAL_ttl_seconds = 0;
  uint64_t WAL_size_limit_MB = 0;
  std::shared_ptr<MergeOperator> merge_operator;
};
}  // namespace rocksdb
