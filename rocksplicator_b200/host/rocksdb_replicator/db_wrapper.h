// db_wrapper.h — the plugin seam between the replication state machine and whatever stores the data.
//
// Interface parity target: replicator::DbWrapper in the reference (rocksdb_replicator/db_wrapper.h:6-15) — the same
// four operations with the same argument meaning, so that a wrapper written against one compiles against the other.
// Implementations: GpuDbWrapper (gpu_db_wrapper.h, the GPU engine); in the reference RocksDbWrapper
// (rocksdb_wrapper.cpp), the CDC observer (cdc_admin/cdc_application_db.cpp:19-37) and TestDBProxy.
#pragma once
#include <cstdint>
#include <functional>
#include <memory>
#include <vector>

#include "rocksdb/db.h"
#include "rocksdb_replicator/replicator_types.h"

namespace replicator {

class DbWrapper {
 public:
  using LogIterator = std::unique_ptr<rocksdb::TransactionLogIterator>;

  virtual ~DbWrapper() = default;

  // LEADER side.  Commit a client batch locally (ReplicatedDB::Write has already appended its timestamp record).
  virtual rocksdb::Status WriteToLeader(const rocksdb::WriteOptions& options, rocksdb::WriteBatch* updates) = 0;

  // LEADER side.  Open a cursor over committed batches starting at the one that contains `seq_number`
  // (NotFound when that sequence has not been written yet).
  virtual rocksdb::Status GetUpdatesFromLeader(rocksdb::SequenceNumber seq_number, LogIterator* iter) = 0;

  // Both sides.  Sequence number of the last committed operation; the follower's resume cursor and the
  // quantity ACKed back to the leader.
  virtual uint64_t LatestSequenceNumber() = 0;

  // FOLLOWER side.  Apply one replicated update (raw WriteBatch bytes + the leader's timestamp).  false = not
  // applied; the pull loop backs off and asks for the same sequence again.
  virtual bool HandleReplicateResponse(Update* update) = 0;

  // FOLLOWER side, GPU-engine addition (not in the reference's interface; the default keeps every existing wrapper valid):
  // apply the updates of ONE ReplicateResponse in order and report how many were applied — the body of the
  // reference's hot loop (replicated_db.cpp:369-383: one HandleReplicateResponse per update, stop at the first
  // failure).  done may run later on another thread; `updates` must stay alive until then.  A wrapper whose store
  // batches across shards (GpuDbWrapper) overrides this so that the >= 16 executor threads do not wait for the
  // device one update at a time.
  using AppliedCallback = std::function<void(size_t n_applied)>;
  virtual void HandleReplicateResponses(std::vector<Update>* updates, AppliedCallback done) {
    size_t n = 0;
    for (auto& u : *updates) {
      if (!HandleReplicateResponse(&u)) break;
      n++;
    }
    done(n);
  }
};

}  // namespace replicator
