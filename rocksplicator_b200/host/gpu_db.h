// gpu_db.h — rocksdb::DB over the GPU engine's C ABI (include/rsp_b200.h).  This is the object handed to
// RocksDBReplicator::addDB / ApplicationDB in place of the rocksdb::DB* that rocksdb::DB::Open returns at
// rocksdb_admin/admin_handler.cpp:640.  Host code only: no CUDA types; every data call ends in librsp_b200.so.
#pragma once
#include <atomic>
#include <condition_variable>
#include <deque>
#include <map>
#include <thread>
#include <functional>
#include <memory>
#include <mutex>
#include <string>

#include "../../include/rsp_b200.h"
#include "rocksdb/db.h"
#include "rocksdb_replicator/replicator_types.h"

namespace b200 {

// one engine per GPU, shared by every DB placed on it (shard_id -> GPU partitioning, SURVEY §8e)
class GpuEngine {
 public:
  static std::shared_ptr<GpuEngine> ForDevice(int device);
  ~GpuEngine();
  rsp_engine* raw() const { return e_; }

 private:
  explicit GpuEngine(rsp_engine* e) : e_(e) {}
  rsp_engine* e_;
};

class GpuDB : public rocksdb::DB {
 public:
  // rocksdb::DB::Open(options, path, &db): `name` plays the path's role (segmentNNNNN)
  static rocksdb::Status Open(const rocksdb::Options& options, const std::string& name, rocksdb::DB** dbptr,
                              int device = 0);
  ~GpuDB() override;

  rocksdb::Status Write(const rocksdb::WriteOptions& options, rocksdb::WriteBatch* updates) override;
  // Several independent writes of this shard in ONE engine call (rsp_apply_updates with write semantics): each batch
  // is its own DB::Write — own sequence numbers, own status — but they share a device tick.  The message-ingestion
  // writer (rocksdb_admin/message_ingestion.h) turns a poll of Kafka messages into one call here.
  std::vector<rocksdb::Status> WriteMany(const rocksdb::WriteOptions& options, const std::vector<rocksdb::WriteBatch*>& updates);
  rocksdb::Status Get(const rocksdb::ReadOptions& options, const rocksdb::Slice& key, std::string* value) override;
  rocksdb::Status Get(const rocksdb::ReadOptions& options, rocksdb::ColumnFamilyHandle* cf, const rocksdb::Slice& key,
                      rocksdb::PinnableSlice* value) override;
  std::vector<rocksdb::Status> MultiGet(const rocksdb::ReadOptions& options, const std::vector<rocksdb::Slice>& keys,
                                        std::vector<std::string>* values) override;
  rocksdb::Iterator* NewIterator(const rocksdb::ReadOptions& options) override;
  rocksdb::Status CompactRange(const rocksdb::CompactRangeOptions& options, const rocksdb::Slice* begin,
                               const rocksdb::Slice* end) override;
  rocksdb::Status Flush(const rocksdb::FlushOptions& options) override;
  // bulk load of SstFileWriter output (rocksdb_admin/admin_handler.cpp:1820-1845): the files are parsed on the host
  // (sst/sst_format.h) and become ONE new sorted run on the device; sequence rules of
  // rocksdb_replicator/tests/rocksdb_assumption_test.cpp:248-283
  rocksdb::Status IngestExternalFile(const std::vector<std::string>& external_files,
                                     const rocksdb::IngestExternalFileOptions& options) override;
  // the shard's visible contents (merges folded, tombstones dropped) as one ingestible block-based SST file: what a
  // backup of a volatile HBM shard is.  Returns the number of entries through *entries when it is not null.
  rocksdb::Status ExportSstFile(const std::string& path, uint64_t* entries = nullptr);
  // HBM is volatile: a backup is the shard's visible contents as one SST file plus a small "dbmeta" file (name,
  // sequence number, entry count) in `dir` — the role of BackupEngine::CreateNewBackupWithMetadata in
  // rocksdb_admin/admin_handler.cpp:696-766.  Written to a temporary name and renamed: a crash leaves the old backup.
  rocksdb::Status Backup(const std::string& dir, uint64_t* seq_out = nullptr);
  // restoreDBHelper (admin_handler.cpp:768-860): a fresh shard `name` with the backup's contents, continuing at the
  // backup's sequence number (its pull loop resumes from LatestSequenceNumber() exactly as after a RocksDB restore)
  static rocksdb::Status Restore(const rocksdb::Options& options, const std::string& name, const std::string& dir,
                                 rocksdb::DB** dbptr, int device = 0);
  rocksdb::SequenceNumber GetLatestSequenceNumber() const override;
  rocksdb::Status GetUpdatesSince(rocksdb::SequenceNumber seq,
                                  std::unique_ptr<rocksdb::TransactionLogIterator>* iter) override;
  rocksdb::ColumnFamilyHandle* DefaultColumnFamily() const override { return &default_cf_; }
  rocksdb::Options GetOptions() const override { return options_; }
  bool GetProperty(const rocksdb::Slice& property, std::string* value) override;
  int NumberLevels() override { return options_.num_levels; }
  void GetColumnFamilyMetaData(rocksdb::ColumnFamilyMetaData* meta) override;
  const std::string& GetName() const override { return name_; }

  // The follower fast path: RocksDbWrapper::HandleReplicateResponse's body
  // (rocksdb_replicator/rocksdb_wrapper.cpp:13-28) as one engine call — the raw bytes go to the device,
  // which appends the LogData(timestamp) record, decodes, sequences and inserts.
  rocksdb::Status ApplyReplicated(const rocksdb::Slice& raw_data, uint64_t timestamp_ms);
  // The same for all updates of one ReplicateResponse (rsp_apply_updates): copied into the engine's open tick, applied
  // in order with every other shard's response; done(n_applied, status of the first failure) runs on an engine
  // completion thread once the tick has run.  `updates` must stay alive until done has been called.
  void ApplyReplicatedBatch(const std::vector<replicator::Update>& updates,
                            std::function<void(size_t, const rocksdb::Status&)> done);

  rsp_shard* shard() const { return shard_; }
  rsp_engine* engine() const { return engine_->raw(); }

 private:
  GpuDB() {}
  rocksdb::Status ToStatus(int code) const;
  void LogAppend(rocksdb::SequenceNumber first_seq, std::string&& bytes, uint32_t count);
  static int MergeTrampoline(void* state, const uint8_t* key, size_t klen, const uint8_t* existing, size_t elen,
                             const uint8_t* operand, size_t olen, void (*out_set)(void*, const uint8_t*, size_t),
                             void* out_ctx);
  // One chunk of the update log = what ONE call appended (a leader's Write: one batch; a follower's response: its <= 50
  // updates), the batches back to back in one string: three allocations per response instead of two per update — with
  // a std::string + shared_ptr per update the completion threads spent their time in malloc / free and bounded the
  // whole pull loop.
  struct LogChunk {
    struct Rec { uint32_t off, len, count; rocksdb::SequenceNumber first_seq; };
    rocksdb::SequenceNumber first_seq = 0, last_seq = 0;
    std::vector<Rec> recs;
    std::string bytes;
  };
  class LogIter;

  std::string name_;
  rocksdb::Options options_;
  std::shared_ptr<GpuEngine> engine_;
  rsp_shard* shard_ = nullptr;
  mutable rocksdb::ColumnFamilyHandle default_cf_;
  // update log (the WAL's role for GetUpdatesSince): applied batches by sequence number, bounded
  std::mutex write_mu_;  // keeps log order == sequence order
  std::mutex log_mu_;
  std::deque<std::shared_ptr<const LogChunk>> log_;
  uint64_t log_base_id_ = 0;  // id of log_[0] (chunk ids)
  void LogPush(std::shared_ptr<const LogChunk> c);  // log_mu_ held
  size_t log_bytes_ = 0;
  size_t log_cap_bytes_ = 256u << 20;
  std::atomic<size_t> value_hint_{0};  // largest value MultiGet has seen (the staging stride of its first pass)
};

// Spills shards on a schedule: every `period_ms` each registered DB whose sequence number moved since its last backup
// is backed up to <root>/<db name>/ (the reference's operators schedule backupDB calls from outside; HBM being
// volatile, the schedule lives next to the engine here).
class BackupScheduler {
 public:
  BackupScheduler(const std::string& root, uint64_t period_ms);
  ~BackupScheduler();
  void Add(const std::string& name, std::shared_ptr<rocksdb::DB> db);
  void Remove(const std::string& name);
  uint64_t backups_done() const { return done_.load(); }
  // one pass now (also what the timer thread runs); returns the number of shards written
  size_t RunOnce();

 private:
  struct Item { std::shared_ptr<rocksdb::DB> db; uint64_t last_seq = ~0ull; };
  const std::string root_;
  const uint64_t period_ms_;
  std::mutex mu_;
  std::condition_variable cv_;
  std::map<std::string, Item> items_;
  bool stop_ = false;
  std::atomic<uint64_t> done_{0};
  std::thread th_;
};

}  // namespace b200
