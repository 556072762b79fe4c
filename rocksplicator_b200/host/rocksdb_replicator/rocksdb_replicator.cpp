// rocksdb_replicator.cpp — the replication state machine above the DbWrapper seam.
// Follows rocksdb_replicator/replicated_db.cpp (leader Write :103-166, ACK wait :236-273, follower pull
// loop :314-433, leader long-poll serving :435-575, iterator cache :577-611) and
// rocksdb_replicator/rocksdb_replicator.cpp (addDB :96-133, removeDB :135-154, write :156-171), on std
// threads and a pluggable transport.
#include "rocksdb_replicator/rocksdb_replicator.h"

#include <chrono>
#include <random>
#include <sstream>

#include "common/dbconfig.h"
#include "rocksdb_replicator/gpu_db_wrapper.h"
#include "rocksdb_replicator/replicator_stats.h"

namespace replicator {

ReplicatorFlags& Flags() {
  static ReplicatorFlags f;
  return f;
}

namespace {
uint64_t NowMs() {
  return std::chrono::duration_cast<std::chrono::milliseconds>(std::chrono::system_clock::now().time_since_epoch()).count();
}
// max(flag, per-dataset setting): replicated_db.cpp:131-136
int EffectiveReplicationMode(const std::string& db_name) {
  const int cfg = (int)common::DBConfigManager::get()->getReplicationMode(db_name);
  return std::max(Flags().replicator_replication_mode, cfg);
}
uint32_t Rand(uint32_t lo, uint32_t hi) {
  static thread_local std::mt19937 g{std::random_device{}()};
  return std::uniform_int_distribution<uint32_t>(lo, hi)(g);
}
}  // namespace

// ---------------------------------------------------------------------------------------------------
// ReplicatedDB
// ---------------------------------------------------------------------------------------------------
RocksDBReplicator::ReplicatedDB::ReplicatedDB(const std::string& db_name, std::shared_ptr<DbWrapper> db_wrapper,
                                              RocksDBReplicator* owner, ReplicaRole role,
                                              const SocketAddress& upstream_addr)
    : db_name_(db_name), db_wrapper_(std::move(db_wrapper)), owner_(owner), role_(role), upstream_addr_(upstream_addr),
      cond_var_(owner->executor()) {
  if (Flags().replicator_timeout_ms > kMinReplTimeoutMs)
    current_replicator_timeout_ms_.store((uint32_t)Flags().replicator_timeout_ms);
}

RocksDBReplicator::ReplicatedDB::~ReplicatedDB() {}

rocksdb::Status RocksDBReplicator::ReplicatedDB::Write(const rocksdb::WriteOptions& options,
                                                       rocksdb::WriteBatch* updates, rocksdb::SequenceNumber* seq_no) {
  if (role_ == ReplicaRole::FOLLOWER || role_ == ReplicaRole::OBSERVER) throw ReturnCode::WRITE_TO_SLAVE;
  incCounter(kReplicatorWriteBytes, updates->GetDataSize(), db_name_);
  // the timestamp travels inside the batch (replicated_db.cpp:115-117)
  const uint64_t ms = NowMs();
  updates->PutLogData(rocksdb::Slice(reinterpret_cast<const char*>(&ms), sizeof(ms)));
  auto status = db_wrapper_->WriteToLeader(options, updates);
  logMetric(kReplicatorWriteToLeaderMs, (int64_t)(NowMs() - ms), db_name_);
  if (!status.ok()) {
    incCounter(kReplicatorWriteLeaderFailure, 1, db_name_);
    return status;
  }
  cond_var_.notifyAll();  // release the followers' long-polls
  const auto cur_seq_no = db_wrapper_->LatestSequenceNumber();
  if (seq_no) *seq_no = cur_seq_no;
  switch (EffectiveReplicationMode(db_name_)) {
    case 1:
    case 2: {
      auto s = writeWaitFollowerACK(cur_seq_no);
      if (!s.ok()) return s;
      break;
    }
    default:
      break;
  }
  incCounter(kReplicatorWriteSuccess, 1, db_name_);
  return status;
}

rocksdb::Status RocksDBReplicator::ReplicatedDB::writeWaitFollowerACK(uint64_t cur_seq_no) {
  const auto& F = Flags();
  if (!max_seq_no_acked_.wait(cur_seq_no, current_replicator_timeout_ms_.load())) {
    incCounter(kReplicatorWriteWaitTimedOut, 1, db_name_);
    numConsecutiveReplTimeout_++;
    // degrade to a short timeout after a run of timeouts, to fail fast (replicated_db.cpp:245-259)
    if (numConsecutiveReplTimeout_.load() >= F.replicator_consecutive_ack_timeout_before_degradation &&
        current_replicator_timeout_ms_.load() == F.replicator_timeout_ms &&
        F.replicator_timeout_degraded_ms < F.replicator_timeout_ms && F.replicator_timeout_degraded_ms >= kMinReplTimeoutMs) {
      current_replicator_timeout_ms_.store((uint32_t)F.replicator_timeout_degraded_ms);
      incCounter(kReplicatorWriteTwoAckDegraded, 1, db_name_);
    }
    return rocksdb::Status::TimedOut("Failed to receive ack from follower");
  }
  numConsecutiveReplTimeout_.store(0);
  if (current_replicator_timeout_ms_.load() != F.replicator_timeout_ms) {
    current_replicator_timeout_ms_.store((uint32_t)F.replicator_timeout_ms);
    incCounter(kReplicatorWriteTwoAckRecovered, 1, db_name_);
  }
  return rocksdb::Status::OK();
}

std::string RocksDBReplicator::ReplicatedDB::Introspect() {
  std::stringstream ss;
  SocketAddress up;
  {
    std::lock_guard<std::mutex> g(upstream_mu_);
    up = upstream_addr_;
  }
  ss << "ReplicatedDB:" << std::endl;
  ss << "  name: " << db_name_ << std::endl;
  ss << "  ReplicaRole: " << ReplicaRoleString(role_) << std::endl;
  ss << "  upstream_addr: " << up.describe() << std::endl;
  ss << "  cur_seq_no: " << db_wrapper_->LatestSequenceNumber() << std::endl;
  ss << "  current_replicator_timeout_ms_: " << current_replicator_timeout_ms_.load() << std::endl;
  return ss.str();
}

void RocksDBReplicator::ReplicatedDB::resetUpstream() {
  resetUpstreamAttempts_++;
  if (!owner_->leader_resolver_) return;
  const std::string leader = owner_->leader_resolver_(db_name_);  // "ip_port"
  const auto us = leader.find('_');
  if (us == std::string::npos) return;
  const std::string ip = leader.substr(0, us);
  std::lock_guard<std::mutex> g(upstream_mu_);
  if (ip != upstream_addr_.getAddressStr()) upstream_addr_.setFromIpPort(ip, (uint16_t)Flags().rocksdb_replicator_port);
}

void RocksDBReplicator::ReplicatedDB::pullFromUpstream() {
  if (removed_.load()) return;
  ReplicateRequest req;
  req.seq_no = (int64_t)db_wrapper_->LatestSequenceNumber();
  req.db_name = db_name_;
  req.max_wait_ms = Flags().replicator_max_server_wait_time_ms;
  req.max_updates = Flags().replicator_max_updates_per_response;
  req.set_role(role_);
  if (trace_cont_) { PullTrace::Get().Add(5, trace_cont_, PullTrace::Now()); trace_cont_ = 0; }
  incCounter(kReplicatorPullRequests, 1, db_name_);
  SocketAddress up;
  {
    std::lock_guard<std::mutex> g(upstream_mu_);
    up = upstream_addr_;
  }
  std::weak_ptr<ReplicatedDB> weak_db = shared_from_this();
  const uint32_t timeout = (uint32_t)(Flags().replicator_max_server_wait_time_ms +
                                      Flags().replicator_client_server_timeout_difference_ms);
  Executor* my_executor = owner_->executor();
  const int64_t t_call = PullTrace::Get().enabled.load(std::memory_order_relaxed) ? PullTrace::Now() : 0;
  owner_->transport()->replicate(up, req, timeout, [weak_db, my_executor, t_call](ReplicateResult&& tr) {
   // continue on OUR executor (the reference's `.via(executor_)`, replicated_db.cpp:328)
   auto shared_t = std::make_shared<ReplicateResult>(std::move(tr));
   if (t_call) { const int64_t now = PullTrace::Now(); PullTrace::Get().Add(0, t_call, now); shared_t->t_mark = now; }
   my_executor->add([weak_db, shared_t] {
    ReplicateResult& t = *shared_t;
    if (t.t_mark) { const int64_t now = PullTrace::Now(); PullTrace::Get().Add(1, t.t_mark, now); t.t_mark = now; }
    auto db = weak_db.lock();
    if (!db || db->removed_.load()) return;
    bool delay_next_pull = false;
    if (!t.ok) {
      delay_next_pull = true;
      incCounter(kReplicatorPullRequestsFailure, 1, db->db_name_);
      if (t.is_replicate_exception) {
        incCounter(kReplicatorRemoteApplicationExceptions, 1, db->db_name_);
        if (t.ex.code == ErrorCode::SOURCE_NOT_FOUND) db->resetUpstream();
      } else {
        incCounter(kReplicatorConnectionErrors, 1, db->db_name_);
      }
    } else {
      incCounter(kReplicatorPullRequestsSuccess, 1, db->db_name_);
      auto& response = t.response;
      uint64_t in_bytes = 0;
      const uint64_t now = NowMs();
      for (auto& update : response.updates) {
        if (update.timestamp != 0)
          logMetric(kReplicatorLatency, (uint64_t)update.timestamp < now ? (int64_t)(now - (uint64_t)update.timestamp) : 0, db->db_name_);
        in_bytes += update.raw_data.size();
      }
      incCounter(kReplicatorInBytes, in_bytes, db->db_name_);
      if (response.has_role && response.role != ReplicaRole::LEADER) incCounter(kReplicatorPullFromNonLeader, 1, db->db_name_);
      if (!response.updates.empty()) {
        // THE HOT LOOP (replicated_db.cpp:369-383: one DbWrapper call per update, in order, stop at the first
        // failure) as ONE call for the whole response; the rest of this function continues in its completion
        // (shared_t keeps the updates alive)
        const size_t n_updates = response.updates.size();
        // The completion runs on one of the engine's completion threads; what is left of this function — counters, the
        // wake-up of chained followers, the next pull (an asynchronous call) — is short and never blocks, so it runs
        // right there instead of hopping to our executor once more (the reference has no such hop either: its loop
        // continues in the same task, replicated_db.cpp:384-431).
        auto staged_at = std::make_shared<std::atomic<int64_t>>(0);
        db->db_wrapper_->HandleReplicateResponses(&response.updates, [weak_db, shared_t, n_updates, staged_at](size_t n_applied) {
          int64_t t_done = 0;
          if (shared_t->t_mark) {
            t_done = PullTrace::Now();
            const int64_t st = staged_at->load(std::memory_order_acquire);
            if (st) PullTrace::Get().Add(3, st, t_done);
          }
          auto db = weak_db.lock();
          if (!db || db->removed_.load()) return;
          db->trace_cont_ = t_done;
          const bool failed = n_applied < n_updates;
          if (failed) incCounter(kReplicatorHandleResponseFailure, 1, db->db_name_);
          db->pullFromUpstreamNoUpdates_ = 0;
          db->cond_var_.notifyAll();  // chained followers long-polling on us
          db->scheduleNextPull(failed);
        });
        if (t.t_mark) { const int64_t now = PullTrace::Now(); PullTrace::Get().Add(2, t.t_mark, now); staged_at->store(now, std::memory_order_release); }
        return;
      }
      incCounter(kReplicatorPullRequestsNoUpdates, 1, db->db_name_);
      db->pullFromUpstreamNoUpdates_++;
      if (response.has_role && response.role != ReplicaRole::LEADER &&
          Flags().reset_upstream_on_empty_updates_from_non_leader &&
          db->pullFromUpstreamNoUpdates_ >= (uint32_t)Flags().replicator_max_consecutive_no_updates_before_upstream_reset) {
        incCounter(kReplicatorResetUpstreamOnNoUpdates, 1, db->db_name_);
        db->resetUpstream();
        db->pullFromUpstreamNoUpdates_ = 0;
      }
    }
    db->scheduleNextPull(delay_next_pull);
   });
  });
}

// the tail of the pull loop (replicated_db.cpp:412-431): back off after an error, otherwise pull again at once
void RocksDBReplicator::ReplicatedDB::scheduleNextPull(bool delay_next_pull) {
  std::weak_ptr<ReplicatedDB> weak_db = shared_from_this();
  {
    auto* db = this;
    if (delay_next_pull) {
      const uint32_t d = (uint32_t)Flags().replicator_pull_delay_on_error_ms;
      db->owner_->executor()->addDelayed([weak_db] {
        if (auto d2 = weak_db.lock()) d2->pullFromUpstream();
      }, Rand(d, d * 2));
    } else {
      db->pullFromUpstream();
    }
  }
}

void RocksDBReplicator::ReplicatedDB::handleReplicateRequest(std::unique_ptr<ReplicateRequest> request,
                                                             ReplicateCallback callback) {
  auto db = shared_from_this();
  std::weak_ptr<ReplicatedDB> weak_db = db;
  const auto seq_no = static_cast<rocksdb::SequenceNumber>(request->seq_no);
  // the follower's request carries the largest sequence number it has committed: that is the ACK
  const uint64_t leader_seq = db_wrapper_->LatestSequenceNumber();
  if (leader_seq < seq_no) logMetric(kReplicatorLeaderSequenceNumbersBehind, (int64_t)(seq_no - leader_seq), db_name_);
  if (request->has_role && request->role == ReplicaRole::OBSERVER) incCounter(kReplicatorHandleObserverRequests, 1, db_name_);
  else max_seq_no_acked_.post(seq_no);
  const int replication_mode = EffectiveReplicationMode(db_name_);
  const uint64_t timeout = (uint64_t)request->max_wait_ms;
  std::shared_ptr<ReplicateRequest> req(std::move(request));
  auto cb = std::make_shared<ReplicateCallback>(std::move(callback));
  cond_var_.runIfConditionOrWaitForNotify(
      [weak_db, replication_mode, req, cb]() {
        auto db = weak_db.lock();
        ReplicateResult out;
        if (!db || db->removed_.load()) {
          out.is_replicate_exception = true;
          out.ex.code = ErrorCode::SOURCE_NOT_FOUND;
          out.ex.msg = req->db_name + " has been removed";
          (*cb)(std::move(out));
          return;
        }
        const rocksdb::SequenceNumber expected_seq_no = (rocksdb::SequenceNumber)req->seq_no + 1;
        rocksdb::SequenceNumber next_seq_no = expected_seq_no;
        auto iter = db->getCachedIter(expected_seq_no);
        if (iter && !iter->Valid()) {
          iter->Next();
          if (!iter->Valid()) iter.reset(nullptr);
        }
        rocksdb::Status status;
        const bool use_cached_iter = iter != nullptr;
        if (!use_cached_iter) status = db->db_wrapper_->GetUpdatesFromLeader(expected_seq_no, &iter);
        if (use_cached_iter || status.ok() || status.IsNotFound()) {
          out.ok = true;
          out.response.set_role(db->role_);
          for (int32_t i = 0; i < req->max_updates && iter && iter->Valid(); ++i, iter->Next()) {
            auto result = iter->GetBatch();
            Update update;
            update.set_seq_no(result.sequence);
            next_seq_no += (rocksdb::SequenceNumber)result.writeBatchPtr->Count();
            update.raw_data = result.writeBatchPtr->Data();
            LogExtractor extractor;
            auto ret = result.writeBatchPtr->Iterate(&extractor);
            update.timestamp = ret.ok() ? (int64_t)extractor.ms : 0;
            out.response.updates.emplace_back(std::move(update));
          }
          uint64_t out_bytes = 0;
          for (const auto& u : out.response.updates) out_bytes += u.raw_data.size();
          logMetric(kReplicatorOutNumUpdates, (int64_t)out.response.updates.size(), db->db_name_);
          incCounter(kReplicatorOutBytes, out_bytes, db->db_name_);
          (*cb)(std::move(out));
          if (replication_mode == 1) db->max_seq_no_acked_.post(next_seq_no - 1);
        } else {
          out.is_replicate_exception = true;
          incCounter(kReplicatorGetUpdatesSinceErrors, 1, db->db_name_);
          out.ex.code = ErrorCode::SOURCE_READ_ERROR;
          out.ex.msg = status.ToString();
          (*cb)(std::move(out));
        }
        if (iter) db->putCachedIter(next_seq_no, std::move(iter));
      },
      [db, seq_no] { return db->db_wrapper_->LatestSequenceNumber() > seq_no; }, timeout);
}

std::unique_ptr<rocksdb::TransactionLogIterator> RocksDBReplicator::ReplicatedDB::getCachedIter(rocksdb::SequenceNumber seq_no) {
  std::lock_guard<std::mutex> g(cached_iters_mutex_);
  auto it = cached_iters_.find(seq_no);
  if (it == cached_iters_.end()) return nullptr;
  auto ret = std::move(it->second.first);
  cached_iters_.erase(it);
  return ret;
}
void RocksDBReplicator::ReplicatedDB::putCachedIter(rocksdb::SequenceNumber seq_no,
                                                    std::unique_ptr<rocksdb::TransactionLogIterator> it) {
  std::lock_guard<std::mutex> g(cached_iters_mutex_);
  cached_iters_.emplace(seq_no, std::make_pair(std::move(it), NowMs()));
}
void RocksDBReplicator::ReplicatedDB::cleanIdleCachedIters() {
  const auto now = NowMs();
  std::lock_guard<std::mutex> g(cached_iters_mutex_);
  for (auto it = cached_iters_.begin(); it != cached_iters_.end();) {
    if (it->second.second + (uint64_t)Flags().replicator_idle_iter_timeout_ms < now) it = cached_iters_.erase(it);
    else ++it;
  }
}

// ---------------------------------------------------------------------------------------------------
// RocksDBReplicator
// ---------------------------------------------------------------------------------------------------
RocksDBReplicator* RocksDBReplicator::instance() {
  static RocksDBReplicator inst((uint16_t)Flags().rocksdb_replicator_port);
  return &inst;
}

RocksDBReplicator::RocksDBReplicator(uint16_t port, std::shared_ptr<Transport> transport)
    : port_(port), executor_(new Executor((size_t)std::max(Flags().rocksdb_replicator_executor_threads, 16))),
      transport_(transport ? std::move(transport) : std::static_pointer_cast<Transport>(LocalTransport::shared())) {
  LocalTransport::shared()->registerServer(port_, this);
  cleaner_ = std::thread([this] {  // idle WAL-iterator GC (cached_iter_cleaner.cpp:48-67)
    std::unique_lock<std::mutex> l(cleaner_mu_);
    while (!stopping_) {
      cleaner_cv_.wait_for(l, std::chrono::milliseconds(std::max(1000, Flags().replicator_idle_iter_timeout_ms / 2)));
      if (stopping_) break;
      for (auto it = cleaner_dbs_.begin(); it != cleaner_dbs_.end();) {
        if (auto db = it->lock()) { db->cleanIdleCachedIters(); ++it; }
        else it = cleaner_dbs_.erase(it);
      }
    }
  });
}

RocksDBReplicator::~RocksDBReplicator() {
  LocalTransport::shared()->unregisterServer(port_);
  {
    std::lock_guard<std::mutex> g(cleaner_mu_);
    stopping_ = true;
  }
  cleaner_cv_.notify_all();
  cleaner_.join();
  executor_->Stop();
  db_map_.clear();
}

ReturnCode RocksDBReplicator::addDB(const std::string& db_name, std::shared_ptr<rocksdb::DB> db, ReplicaRole role,
                                    const SocketAddress& upstream_addr, ReplicatedDB** replicated_db) {
  // rocksdb_replicator.cpp:96-105 wraps the DB in RocksDbWrapper; here the wrapper is the GPU one
  return addDB(db_name, std::static_pointer_cast<DbWrapper>(std::make_shared<GpuDbWrapper>(db_name, std::move(db))), role,
               upstream_addr, replicated_db);
}

ReturnCode RocksDBReplicator::addDB(const std::string& db_name, std::shared_ptr<DbWrapper> db_wrapper, ReplicaRole role,
                                    const SocketAddress& upstream_addr, ReplicatedDB** replicated_db) {
  std::shared_ptr<ReplicatedDB> new_db(new ReplicatedDB(db_name, std::move(db_wrapper), this, role, upstream_addr));
  if (!db_map_.add(db_name, new_db)) return ReturnCode::DB_PRE_EXIST;
  if (replicated_db) *replicated_db = new_db.get();
  {
    std::lock_guard<std::mutex> g(cleaner_mu_);
    cleaner_dbs_.push_back(new_db);
  }
  if (role == ReplicaRole::FOLLOWER || role == ReplicaRole::OBSERVER) new_db->pullFromUpstream();
  return ReturnCode::OK;
}

ReturnCode RocksDBReplicator::removeDB(const std::string& db_name) {
  std::shared_ptr<ReplicatedDB> db;
  if (!db_map_.get(db_name, &db)) return ReturnCode::DB_NOT_FOUND;
  db->removed_.store(true);
  if (!db_map_.remove(db_name)) return ReturnCode::DB_NOT_FOUND;
  db->cond_var_.notifyAll();  // parked long-polls answer SOURCE_NOT_FOUND
  std::weak_ptr<ReplicatedDB> weak = db;
  db.reset();
  // wait until nobody else holds the ReplicatedDB (rocksdb_replicator.cpp:143-151)
  while (!weak.expired()) std::this_thread::sleep_for(std::chrono::milliseconds(20));
  return ReturnCode::OK;
}

ReturnCode RocksDBReplicator::write(const std::string& db_name, const rocksdb::WriteOptions& options,
                                    rocksdb::WriteBatch* updates, rocksdb::SequenceNumber* seq_no) {
  std::shared_ptr<ReplicatedDB> db;
  if (!db_map_.get(db_name, &db)) return ReturnCode::DB_NOT_FOUND;
  try {
    auto status = db->Write(options, updates, seq_no);
    if (status.IsTimedOut()) return ReturnCode::WAIT_SLAVE_TIMEOUT;
    return status.ok() ? ReturnCode::OK : ReturnCode::WRITE_ERROR;
  } catch (const ReturnCode code) {
    return code;
  }
}

void RocksDBReplicator::serveReplicate(std::unique_ptr<ReplicateRequest> request, ReplicateCallback callback) {
  std::shared_ptr<ReplicatedDB> db;
  if (!db_map_.get(request->db_name, &db)) {
    ReplicateResult out;
    out.is_replicate_exception = true;
    out.ex.code = ErrorCode::SOURCE_NOT_FOUND;
    out.ex.msg = request->db_name + " not found";
    callback(std::move(out));
    return;
  }
  db->handleReplicateRequest(std::move(request), std::move(callback));
}

// ---------------------------------------------------------------------------------------------------
// LocalTransport
// ---------------------------------------------------------------------------------------------------
std::shared_ptr<LocalTransport> LocalTransport::shared() {
  static std::shared_ptr<LocalTransport> t = std::make_shared<LocalTransport>();
  return t;
}
void LocalTransport::registerServer(uint16_t port, RocksDBReplicator* r) {
  std::lock_guard<std::mutex> g(mu_);
  servers_[port] = r;
}
void LocalTransport::unregisterServer(uint16_t port) {
  std::lock_guard<std::mutex> g(mu_);
  servers_.erase(port);
}
void LocalTransport::replicate(const SocketAddress& upstream, const ReplicateRequest& request, uint32_t /*timeout_ms*/,
                               ReplicateCallback cb) {
  RocksDBReplicator* server = nullptr;
  {
    std::lock_guard<std::mutex> g(mu_);
    auto it = servers_.find(upstream.port);
    if (it != servers_.end()) server = it->second;
  }
  if (!server) {
    // connection refused: surfaces as a std::exception in the reference (replicated_db.cpp:352-362);
    // deliver it asynchronously like a socket error would be
    ReplicateResult out;
    out.transport_error = "connect to " + upstream.describe() + " failed";
    std::thread([cb, out]() mutable { cb(std::move(out)); }).detach();
    return;
  }
  auto req = std::make_unique<ReplicateRequest>(request);
  Executor* ex = server->executor();
  auto shared_cb = std::make_shared<ReplicateCallback>(std::move(cb));
  // request and response each hop through the server's executor, never the caller's stack
  ex->add([server, shared_cb, r = std::shared_ptr<ReplicateRequest>(std::move(req))]() mutable {
    server->serveReplicate(std::make_unique<ReplicateRequest>(*r), [shared_cb](ReplicateResult&& res) {
      (*shared_cb)(std::move(res));
    });
  });
}

}  // namespace replicator
