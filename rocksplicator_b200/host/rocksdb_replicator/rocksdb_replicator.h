// rocksdb_replicator.h — RocksDBReplicator / ReplicatedDB with the reference's public surface
// (rocksdb_replicator/rocksdb_replicator.h:71-216): addDB (two overloads), removeDB, write,
// ReplicatedDB::Write / Introspect, ReturnCode, LogExtractor.  The replication protocol logic (pull loop,
// long-poll serving, ACK modes, upstream reset hook) follows rocksdb_replicator/replicated_db.cpp; the
// storage below the DbWrapper seam is the GPU engine.
#pragma once
#include <atomic>
#include <list>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>

#include "rocksdb/db.h"
#include "rocksdb_replicator/db_wrapper.h"
#include "rocksdb_replicator/executor.h"
#include "rocksdb_replicator/fast_read_map.h"
#include "rocksdb_replicator/max_number_box.h"
#include "rocksdb_replicator/non_blocking_condition_variable.h"
#include "rocksdb_replicator/replicator_types.h"
#include "rocksdb_replicator/transport.h"

namespace replicator {

const uint32_t kMinReplTimeoutMs = 1;

// gflags of replicated_db.cpp:36-90 / rocksdb_replicator.cpp:35-42 as one settable struct
struct ReplicatorFlags {
  int32_t rocksdb_replicator_port = 9091;
  int32_t rocksdb_replicator_executor_threads = 32;
  int32_t replicator_max_server_wait_time_ms = 10 * 1000;
  int32_t replicator_client_server_timeout_difference_ms = 10 * 1000;
  int32_t replicator_max_updates_per_response = 50;
  int32_t replicator_pull_delay_on_error_ms = 5 * 1000;
  int32_t replicator_max_consecutive_no_updates_before_upstream_reset = 5;
  int32_t replicator_replication_mode = 0;
  uint64_t replicator_timeout_ms = 2 * 1000;
  uint64_t replicator_timeout_degraded_ms = 10;
  uint64_t replicator_consecutive_ack_timeout_before_degradation = 100;
  bool reset_upstream_on_empty_updates_from_non_leader = false;
  int32_t replicator_idle_iter_timeout_ms = 60 * 1000;
};
ReplicatorFlags& Flags();

// rocksdb_replicator.h:60-69
struct LogExtractor : public rocksdb::WriteBatch::Handler {
  void LogData(const rocksdb::Slice& blob) override {
    if (blob.size() == sizeof(ms)) memcpy(&ms, blob.data(), sizeof(ms));
  }
  uint64_t ms = 0;
};

enum class ReturnCode { OK = 0, DB_NOT_FOUND = 1, DB_PRE_EXIST = 2, WRITE_TO_SLAVE = 3, WRITE_ERROR = 4, WAIT_SLAVE_TIMEOUT = 5 };

// hook for "ask the cluster manager who the leader is" (common/helix_client over JNI in the reference,
// replicated_db.cpp:278-312); returns "" when unknown
using LeaderResolver = std::function<std::string(const std::string& db_name)>;

class RocksDBReplicator {
 public:
  class ReplicatedDB : public std::enable_shared_from_this<ReplicatedDB> {
   public:
    // rocksdb::DB::Write + (1) *seq_no filled after the write, (2) throws ReturnCode::WRITE_TO_SLAVE on a
    // FOLLOWER / OBSERVER, (3) TimedOut status when modes 1/2 get no ACK in time (rocksdb_replicator.h:96-112)
    rocksdb::Status Write(const rocksdb::WriteOptions& options, rocksdb::WriteBatch* updates,
                          rocksdb::SequenceNumber* seq_no = nullptr);
    std::string Introspect();
    // how often this replica tried to re-resolve its upstream (rocksdb_replicator.h:139: kept for tests)
    uint32_t resetUpstreamAttempts() const { return resetUpstreamAttempts_.load(); }
    ~ReplicatedDB();

   private:
    ReplicatedDB(const std::string& db_name, std::shared_ptr<DbWrapper> db_wrapper, RocksDBReplicator* owner,
                 ReplicaRole role, const SocketAddress& upstream_addr);
    void pullFromUpstream();
    void scheduleNextPull(bool delay_next_pull);
    void resetUpstream();
    rocksdb::Status writeWaitFollowerACK(uint64_t cur_seq_no);
    void handleReplicateRequest(std::unique_ptr<ReplicateRequest> request, ReplicateCallback callback);
    std::unique_ptr<rocksdb::TransactionLogIterator> getCachedIter(rocksdb::SequenceNumber seq_no);
    void putCachedIter(rocksdb::SequenceNumber seq_no, std::unique_ptr<rocksdb::TransactionLogIterator> it);
    void cleanIdleCachedIters();

    const std::string db_name_;
    std::shared_ptr<DbWrapper> db_wrapper_;
    RocksDBReplicator* const owner_;
    const ReplicaRole role_;
    SocketAddress upstream_addr_;
    std::mutex upstream_mu_;
    uint32_t pullFromUpstreamNoUpdates_{0};
    int64_t trace_cont_{0};  // PullTrace: when the continuation of the last response ran (one pull in flight per db)
    std::atomic<uint32_t> resetUpstreamAttempts_{0};
    detail::NonBlockingConditionVariable cond_var_;
    std::unordered_multimap<rocksdb::SequenceNumber,
                            std::pair<std::unique_ptr<rocksdb::TransactionLogIterator>, uint64_t>> cached_iters_;
    std::mutex cached_iters_mutex_;
    detail::MaxNumberBox max_seq_no_acked_;
    std::atomic<uint32_t> current_replicator_timeout_ms_{kMinReplTimeoutMs};
    std::atomic<uint32_t> numConsecutiveReplTimeout_{0};
    std::atomic<bool> removed_{false};

    friend class RocksDBReplicator;
    friend class LocalTransport;
    friend struct ReplicatorTestPeer;
  };

  // process-wide instance on Flags().rocksdb_replicator_port (rocksdb_replicator.h:160-163)
  static RocksDBReplicator* instance();
  // additional instances on other ports in one process (what the reference's tests do with
  // `#define private public`, rocksdb_replicator_test.cpp:24-27,137-144)
  explicit RocksDBReplicator(uint16_t port, std::shared_ptr<Transport> transport = nullptr);
  ~RocksDBReplicator();

  ReturnCode addDB(const std::string& db_name, std::shared_ptr<rocksdb::DB> db, ReplicaRole role,
                   const SocketAddress& upstream_addr = SocketAddress(), ReplicatedDB** replicated_db = nullptr);
  ReturnCode addDB(const std::string& db_name, std::shared_ptr<DbWrapper> db_wrapper, ReplicaRole role,
                   const SocketAddress& upstream_addr = SocketAddress(), ReplicatedDB** replicated_db = nullptr);
  ReturnCode removeDB(const std::string& db_name);
  ReturnCode write(const std::string& db_name, const rocksdb::WriteOptions& options, rocksdb::WriteBatch* updates,
                   rocksdb::SequenceNumber* seq_no = nullptr);

  // server side of Replicator.replicate (replicator_handler.cpp:24-41): look the DB up and forward
  void serveReplicate(std::unique_ptr<ReplicateRequest> request, ReplicateCallback callback);

  void setLeaderResolver(LeaderResolver r) { leader_resolver_ = std::move(r); }
  uint16_t port() const { return port_; }
  Executor* executor() { return executor_.get(); }
  Transport* transport() { return transport_.get(); }

  RocksDBReplicator(const RocksDBReplicator&) = delete;
  RocksDBReplicator& operator=(const RocksDBReplicator&) = delete;

 private:
  const uint16_t port_;
  std::unique_ptr<Executor> executor_;
  std::shared_ptr<Transport> transport_;
  detail::FastReadMap<std::string, std::shared_ptr<ReplicatedDB>> db_map_;
  LeaderResolver leader_resolver_;
  std::thread cleaner_;
  std::mutex cleaner_mu_;
  std::condition_variable cleaner_cv_;
  bool stopping_ = false;
  std::list<std::weak_ptr<ReplicatedDB>> cleaner_dbs_;
  friend class ReplicatedDB;
};

// In-process transport: requests are handed to the RocksDBReplicator registered under the upstream port.
class LocalTransport : public Transport {
 public:
  static std::shared_ptr<LocalTransport> shared();
  void registerServer(uint16_t port, RocksDBReplicator* r);
  void unregisterServer(uint16_t port);
  void replicate(const SocketAddress& upstream, const ReplicateRequest& request, uint32_t timeout_ms,
                 ReplicateCallback cb) override;

 private:
  std::mutex mu_;
  std::unordered_map<uint16_t, RocksDBReplicator*> servers_;
};

}  // namespace replicator
