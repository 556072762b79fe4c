// rocksdb/db.h — the rocksdb::DB surface ApplicationDB and RocksDbWrapper call
// (rocksdb_admin/application_db.cpp:78-225, rocksdb_replicator/rocksdb_wrapper.cpp:4-28).  The GPU
// implementation is gpu_db.h's GpuDB; members the hot path never reaches answer NotSupported.
#pragma once
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "rocksdb/iterator.h"
#include "rocksdb/merge_operator.h"
#include "rocksdb/options.h"
#include "rocksdb/slice.h"
#include "rocksdb/status.h"
#include "rocksdb/transaction_log.h"
#include "rocksdb/write_batch.h"

namespace rocksdb {

// DB::GetSnapshot's handle: the DB as of GetSequenceNumber(); released with DB::ReleaseSnapshot
class Snapshot {
 public:
  virtual SequenceNumber GetSequenceNumber() const = 0;

 protected:
  virtual ~Snapshot() {}
};

class ColumnFamilyHandle {
 public:
  virtual ~ColumnFamilyHandle() {}
  virtual uint32_t GetID() const { return 0; }
};
struct LevelMetaData { int level; uint64_t size; };
struct ColumnFamilyMetaData { uint64_t size = 0; size_t file_count = 0; std::string name = "default"; std::vector<LevelMetaData> levels; };

class DB {
 public:
  virtual ~DB() {}
  virtual Status Put(const WriteOptions& o, const Slice& k, const Slice& v) { WriteBatch b; b.Put(k, v); return Write(o, &b); }
  virtual Status Delete(const WriteOptions& o, const Slice& k) { WriteBatch b; b.Delete(k); return Write(o, &b); }
  virtual Status Merge(const WriteOptions& o, const Slice& k, const Slice& v) { WriteBatch b; b.Merge(k, v); return Write(o, &b); }
  virtual Status Write(const WriteOptions& options, WriteBatch* updates) = 0;
  virtual Status Get(const ReadOptions& options, const Slice& key, std::string* value) = 0;
  virtual Status Get(const ReadOptions& options, ColumnFamilyHandle* cf, const Slice& key, PinnableSlice* value) = 0;
  virtual std::vector<Status> MultiGet(const ReadOptions& options, const std::vector<Slice>& keys,
                                       std::vector<std::string>* values) = 0;
  virtual Iterator* NewIterator(const ReadOptions& options) = 0;
  virtual Status CompactRange(const CompactRangeOptions& options, const Slice* begin, const Slice* end) = 0;
  virtual Status Flush(const FlushOptions& options) = 0;
  virtual Status IngestExternalFile(const std::vector<std::string>& /*external_files*/, const IngestExternalFileOptions&) {
    return Status::NotSupported("IngestExternalFile");
  }
  virtual SequenceNumber GetLatestSequenceNumber() const = 0;
  virtual const Snapshot* GetSnapshot() { return nullptr; }
  virtual void ReleaseSnapshot(const Snapshot* /*snapshot*/) {}
  virtual Status GetUpdatesSince(SequenceNumber seq, std::unique_ptr<TransactionLogIterator>* iter) = 0;
  virtual ColumnFamilyHandle* DefaultColumnFamily() const = 0;
  virtual Options GetOptions() const = 0;
  virtual DBOptions GetDBOptions() const { return GetOptions(); }
  virtual bool GetProperty(const Slice& property, std::string* value) = 0;
  virtual int NumberLevels() = 0;
  virtual void GetColumnFamilyMetaData(ColumnFamilyMetaData* meta) = 0;
  virtual const std::string& GetName() const = 0;
};

}  // namespace rocksdb
