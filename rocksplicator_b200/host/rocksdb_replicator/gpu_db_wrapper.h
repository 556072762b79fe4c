// gpu_db_wrapper.h — replicator::DbWrapper over the GPU engine: the drop-in for RocksDbWrapper
// (rocksdb_replicator/rocksdb_wrapper.{h,cpp}).  Same four methods, same meaning.
#pragma once
#include <memory>
#include <string>

#include "rocksdb_replicator/db_wrapper.h"

namespace replicator {
class GpuDbWrapper : public DbWrapper {
 public:
  GpuDbWrapper(const std::string& db_name, std::shared_ptr<rocksdb::DB> db);
  uint64_t LatestSequenceNumber() override;                                              // rocksdb_wrapper.cpp:4
  rocksdb::Status WriteToLeader(const rocksdb::WriteOptions& options, rocksdb::WriteBatch* updates) override;  // :5-8
  rocksdb::Status GetUpdatesFromLeader(rocksdb::SequenceNumber seq_number,
                                       std::unique_ptr<rocksdb::TransactionLogIterator>* iter) override;       // :9-12
  bool HandleReplicateResponse(Update* update) override;                                 // :13-28
  // the whole response in one engine call, completion on an engine thread (rsp_apply_updates)
  void HandleReplicateResponses(std::vector<Update>* updates, AppliedCallback done) override;

 private:
  const std::string db_name_;
  std::shared_ptr<rocksdb::DB> db_;
  rocksdb::WriteOptions write_options_;
};
}  // namespace replicator
