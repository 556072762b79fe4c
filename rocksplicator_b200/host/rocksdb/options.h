// rocksdb/options.h — option structs named by the reference's call sites.  Only the fields the hot path
// reads are honoured by the GPU engine (write_buffer_size, merge_operator, level0 trigger).
#pragma once
#include <cstdint>
#include <memory>
#include <string>

namespace rocksdb {
class MergeOperator;
struct WriteOptions { bool sync = false; bool disableWAL = false; };
struct ReadOptions { bool verify_checksums = true; bool fill_cache = true; };
struct CompactRangeOptions { bool change_level = false; int target_level = -1; };
struct FlushOptions { bool wait = true; };
// rocksdb_admin/admin_handler.cpp:1820-1828 sets move_files and allow_global_seqno, the rest stay default
struct IngestExternalFileOptions {
  bool move_files = false;
  bool snapshot_consistency = true;
  bool allow_global_seqno = true;
  bool allow_blocking_flush = true;
};
struct Options {
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
