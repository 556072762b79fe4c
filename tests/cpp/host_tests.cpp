// host_tests.cpp — tests of the C++ mirror of the reference interfaces (rocksplicator_b200/host/).
// Modelled on the reference's own tests:
//   rocksdb_replicator/tests/{fast_read_map,max_number_box,non_blocking_condition_variable}_test.cpp
//   rocksdb_replicator/tests/rocksdb_replicator_test.cpp:146-368, 494-738 (topologies, ACK modes, observer)
//   rocksdb_replicator/tests/rocksdb_assumption_test.cpp:136-187, 329-432
//   rocksdb_admin/tests/application_db_manager_test.cpp:40-85, admin_handler_test.cpp:218-265,681-697
//   examples/counter_service (config #1: 4 shards x 1000 keys, Put + int64 Merge, leader + follower)
// `host_tests cpu` runs what needs no GPU (helpers + the replication protocol over a counting DbWrapper, the
// role rocksdb_replicator/test_db_proxy.cpp plays in the reference); `host_tests gpu` adds the GpuDB-backed ones.
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <string>
#include <thread>
#include <vector>

#include <unistd.h>

#include "../../rocksplicator_b200/csrc/stager.h"
#include "common/dbconfig.h"
#include "common/segment_utils.h"
#include "common/stats.h"
#include "rocksdb_replicator/replicator_stats.h"
#include "gpu_db.h"
#include "rocksdb_admin/application_db_manager.h"
#include "rocksdb_admin/message_ingestion.h"
#include "rocksdb_replicator/rocksdb_replicator.h"

using namespace replicator;
using rocksdb::Slice;
using rocksdb::Status;
using rocksdb::WriteBatch;

static int g_fail = 0, g_checks = 0;
#define EXPECT_TRUE(c) do { g_checks++; if (!(c)) { g_fail++; printf("  FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); } } while (0)
#define EXPECT_EQ(a, b) do { g_checks++; if (!((a) == (b))) { g_fail++; printf("  FAIL %s:%d: %s == %s\n", __FILE__, __LINE__, #a, #b); } } while (0)
static void sleep_ms(int ms) { std::this_thread::sleep_for(std::chrono::milliseconds(ms)); }
template <class F> static bool wait_until(F f, int timeout_ms = 10000) {
  for (int i = 0; i < timeout_ms / 5; i++) { if (f()) return true; sleep_ms(5); }
  return f();
}

// ---- helpers ----------------------------------------------------------------------------------------
static void test_fast_read_map() {
  detail::FastReadMap<std::string, int> m;
  int v = 0;
  EXPECT_TRUE(!m.get("a", &v));
  EXPECT_TRUE(m.add("a", 1));
  EXPECT_TRUE(!m.add("a", 2));
  EXPECT_TRUE(m.get("a", &v) && v == 1);
  EXPECT_TRUE(m.remove("a"));
  EXPECT_TRUE(!m.remove("a"));
  // concurrent readers while a writer adds/removes (fast_read_map_test.cpp:76-99)
  std::atomic<bool> stop{false};
  std::vector<std::thread> readers;
  for (int t = 0; t < 4; t++) readers.emplace_back([&] { int x; while (!stop) m.get("k7", &x); });
  for (int i = 0; i < 2000; i++) { m.add("k" + std::to_string(i % 16), i); m.remove("k" + std::to_string((i + 8) % 16)); }
  stop = true;
  for (auto& t : readers) t.join();
  m.clear();
  EXPECT_EQ(m.size(), 0u);
}

static void test_max_number_box() {
  detail::MaxNumberBox box;
  EXPECT_TRUE(box.wait(0, 1));
  EXPECT_TRUE(!box.wait(5, 20));
  box.post(5);
  EXPECT_TRUE(box.wait(5, 1));
  box.post(3);  // monotone max
  EXPECT_TRUE(box.wait(5, 1));
  std::thread t([&] { sleep_ms(30); box.post(9); });
  EXPECT_TRUE(box.wait(9, 2000));
  t.join();
  EXPECT_TRUE(!box.wait(10, 10));
}

static void test_nbcv() {
  Executor ex(4);
  {
    detail::NonBlockingConditionVariable cv(&ex);
    std::atomic<int> ran{0};
    cv.runIfConditionOrWaitForNotify([&] { ran++; }, [] { return true; }, 0);  // predicate already true
    EXPECT_TRUE(wait_until([&] { return ran == 1; }));
    bool flag = false;
    cv.runIfConditionOrWaitForNotify([&] { ran++; }, [&] { return flag; }, 0);  // waits for notify
    sleep_ms(30);
    EXPECT_EQ(ran.load(), 1);
    cv.notifyAll();
    EXPECT_TRUE(wait_until([&] { return ran == 2; }));
    cv.notifyAll();  // fires once only
    sleep_ms(20);
    EXPECT_EQ(ran.load(), 2);
    cv.runIfConditionOrWaitForNotify([&] { ran++; }, [] { return false; }, 40);  // timeout
    EXPECT_TRUE(wait_until([&] { return ran == 3; }, 2000));
    cv.runIfConditionOrWaitForNotify([&] { ran++; }, [] { return false; }, 0);  // destructor releases it
    sleep_ms(10);
    EXPECT_EQ(ran.load(), 3);
  }
  sleep_ms(50);
  ex.Stop();
}

static void test_write_batch_and_status() {
  WriteBatch b;
  b.Put("k1", "v1"); b.Delete("k2");
  uint64_t five = 5, ts = 1234;
  b.Merge("c", Slice((const char*)&five, 8));
  b.PutLogData(Slice((const char*)&ts, 8));
  static const unsigned char want[] = {0,0,0,0,0,0,0,0, 3,0,0,0, 1,2,'k','1',2,'v','1', 0,2,'k','2', 2,1,'c',8,5,0,0,0,0,0,0,0, 3,8,0xd2,4,0,0,0,0,0,0};
  EXPECT_EQ(b.Data(), std::string((const char*)want, sizeof(want)));  // SURVEY §9 wire-format sample
  EXPECT_EQ(b.Count(), 3);
  LogExtractor ex;
  EXPECT_TRUE(b.Iterate(&ex).ok());
  EXPECT_EQ(ex.ms, 1234u);
  WriteBatch bad(b.Data().substr(0, b.Data().size() - 3));
  rocksdb::WriteBatch::Handler h;
  EXPECT_TRUE(bad.Iterate(&h).IsCorruption());
  EXPECT_EQ(Status::TimedOut("Failed to receive ack from follower").ToString(),
            std::string("Operation timed out: Failed to receive ack from follower"));
  EXPECT_TRUE(Status::TimedOut("x") == Status::TimedOut("y"));
  EXPECT_EQ(common::SegmentToDbName("seg", 7), std::string("seg00007"));
  EXPECT_EQ(common::DbNameToSegment("seg00007"), std::string("seg"));
  EXPECT_EQ(common::ExtractShardId("seg00042"), 42);
}

// the batching front-end's core: concurrent callers copy into the open batch's staging slices in parallel and share
// device batches; a dispatcher runs one batch after the other (csrc/stager.h)
static void test_stager() {
  constexpr size_t CAP = 256;
  static int in_buf[rsp::Stager::kBuffers][CAP], out_buf[rsp::Stager::kBuffers][CAP];
  std::atomic<int> executed{0}, async_done{0}, posts{0};
  std::atomic<bool> classes_ok{true};
  rsp::Stager st(CAP, CAP * 4, [&](const rsp::Stager::BatchInfo& b) {
    sleep_ms(1);  // a "tick"
    for (size_t i = 0; i < b.n_items; i++) {
      if ((uint32_t)(in_buf[b.buf][i] & 1) != b.klass) classes_ok = false;  // requests of different classes never mix
      out_buf[b.buf][i] = in_buf[b.buf][i] * 2 + 1;
      executed++;
    }
  }, [&] { posts++; });
  std::vector<std::thread> th;
  std::atomic<int> wrong{0};
  for (int t = 0; t < 16; t++)
    th.emplace_back([&, t] {
      for (int i = 0; i < 50; i++) {
        rsp::Stager::Ticket k;
        const int n = 1 + (i % 3);
        const uint32_t klass = (uint32_t)(t & 1);
        if (!st.begin(n, n * 4, klass, CAP, &k)) { wrong++; continue; }
        for (int j = 0; j < n; j++) in_buf[k.buf][k.item0 + j] = ((t * 100000 + i * 10 + j) << 1) | (int)klass;
        if (i % 5 == 4) {  // asynchronous completion: checked on the dispatcher thread
          const int buf = k.buf; const size_t i0 = k.item0;
          st.commit_async(k, [&, buf, i0, n, t, i, klass] {
            for (int j = 0; j < n; j++) if (out_buf[buf][i0 + j] != ((((t * 100000 + i * 10 + j) << 1) | (int)klass) * 2 + 1)) wrong++;
            async_done++;
          });
        } else {
          st.commit(k);
          st.wait(k);
          for (int j = 0; j < n; j++) if (out_buf[k.buf][k.item0 + j] != in_buf[k.buf][k.item0 + j] * 2 + 1) wrong++;
          st.release(k);
        }
      }
    });
  for (auto& t : th) t.join();
  EXPECT_TRUE(wait_until([&] { return async_done.load() == 16 * 10; }));
  rsp::Stager::Ticket big;
  EXPECT_TRUE(!st.begin(CAP + 1, 4, 0, CAP, &big));  // can never fit: the caller takes its direct path
  EXPECT_EQ(wrong.load(), 0);
  EXPECT_TRUE(classes_ok.load());
  EXPECT_TRUE(st.batches() < 800);  // combining happened: fewer batches than requests
  EXPECT_TRUE(posts.load() == (int)st.batches() || posts.load() == (int)st.batches() + 1);
  printf("  stager: 800 requests (%d items) in %llu batches\n", executed.load(), (unsigned long long)st.batches());
}

// ---- a DbWrapper that only counts and logs: rocksdb_replicator/test_db_proxy.cpp's role -------------
class CountingDb : public DbWrapper {
 public:
  uint64_t LatestSequenceNumber() override { return seq_.load(); }
  Status WriteToLeader(const rocksdb::WriteOptions&, WriteBatch* updates) override {
    std::lock_guard<std::mutex> g(mu_);
    const uint64_t first = seq_ + 1;
    std::string rep = updates->Data();
    memcpy(&rep[0], &first, 8);
    log_.push_back({first, rep});
    seq_ += (uint64_t)updates->Count();
    return Status::OK();
  }
  bool HandleReplicateResponse(Update* u) override {
    WriteBatch wb(u->raw_data);
    wb.PutLogData(Slice((const char*)&u->timestamp, 8));
    return WriteToLeader(rocksdb::WriteOptions(), &wb).ok();
  }
  struct It : public rocksdb::TransactionLogIterator {
    CountingDb* d; size_t i;
    bool Valid() override { std::lock_guard<std::mutex> g(d->mu_); return i < d->log_.size(); }
    void Next() override { i++; }
    Status status() override { return Status::OK(); }
    rocksdb::BatchResult GetBatch() override {
      std::lock_guard<std::mutex> g(d->mu_);
      rocksdb::BatchResult r; r.sequence = d->log_[i].first; r.writeBatchPtr.reset(new WriteBatch(d->log_[i].second)); return r;
    }
  };
  Status GetUpdatesFromLeader(rocksdb::SequenceNumber seq, std::unique_ptr<rocksdb::TransactionLogIterator>* it) override {
    std::lock_guard<std::mutex> g(mu_);
    if (seq > seq_) return Status::NotFound();
    size_t i = 0;
    while (i < log_.size() && log_[i].first + (uint64_t)WriteBatch(log_[i].second).Count() - 1 < seq) i++;
    auto* p = new It(); p->d = this; p->i = i;
    it->reset(p);
    return Status::OK();
  }
  std::atomic<uint64_t> seq_{0};
  std::mutex mu_;
  std::vector<std::pair<uint64_t, std::string>> log_;
};

static void fast_flags() {
  auto& F = Flags();
  F.replicator_pull_delay_on_error_ms = 50;
  F.replicator_max_server_wait_time_ms = 200;
  F.replicator_client_server_timeout_difference_ms = 100;
  F.replicator_replication_mode = 0;
  F.replicator_timeout_ms = 2000;
}

// rocksdb_replicator_test.cpp:146-208 (1 leader + 1 follower), :105-120 (Introspect text) — protocol only
static void test_replication_protocol_counting() {
  fast_flags();
  RocksDBReplicator leader_host(19091), follower_host(19092);
  auto ldb = std::make_shared<CountingDb>(), fdb = std::make_shared<CountingDb>();
  RocksDBReplicator::ReplicatedDB *rl = nullptr, *rf = nullptr;
  EXPECT_EQ(leader_host.addDB("master", std::static_pointer_cast<DbWrapper>(ldb), ReplicaRole::LEADER, SocketAddress(), &rl), ReturnCode::OK);
  EXPECT_EQ(leader_host.addDB("master", std::static_pointer_cast<DbWrapper>(ldb), ReplicaRole::LEADER), ReturnCode::DB_PRE_EXIST);
  EXPECT_EQ(follower_host.addDB("master", std::static_pointer_cast<DbWrapper>(fdb), ReplicaRole::FOLLOWER, SocketAddress("127.0.0.1", 19091), &rf), ReturnCode::OK);
  rocksdb::WriteOptions wo;
  for (int i = 0; i < 100; i++) {
    WriteBatch b;
    b.Put(std::to_string(i) + "key", std::to_string(i) + "value");
    b.Put(std::to_string(i) + "key2", std::to_string(i) + "value2");
    rocksdb::SequenceNumber seq = 0;
    EXPECT_TRUE(rl->Write(wo, &b, &seq).ok());
    EXPECT_EQ(seq, (uint64_t)(2 * (i + 1)));
  }
  EXPECT_TRUE(wait_until([&] { return fdb->LatestSequenceNumber() == 200; }));
  EXPECT_EQ(ldb->LatestSequenceNumber(), 200u);
  // WRITE_TO_SLAVE is thrown by ReplicatedDB::Write and returned by RocksDBReplicator::write
  WriteBatch b; b.Put("x", "y");
  bool thrown = false;
  try { rf->Write(wo, &b); } catch (ReturnCode rc) { thrown = rc == ReturnCode::WRITE_TO_SLAVE; }
  EXPECT_TRUE(thrown);
  EXPECT_EQ(follower_host.write("master", wo, &b), ReturnCode::WRITE_TO_SLAVE);
  EXPECT_EQ(follower_host.write("nope", wo, &b), ReturnCode::DB_NOT_FOUND);
  EXPECT_EQ(rl->Introspect(), std::string("ReplicatedDB:\n  name: master\n  ReplicaRole: LEADER\n  upstream_addr: uninitialized_addr\n  cur_seq_no: 200\n  current_replicator_timeout_ms_: 2000\n"));
  EXPECT_EQ(rf->Introspect(), std::string("ReplicatedDB:\n  name: master\n  ReplicaRole: FOLLOWER\n  upstream_addr: 127.0.0.1\n  cur_seq_no: 200\n  current_replicator_timeout_ms_: 2000\n"));
  EXPECT_EQ(follower_host.removeDB("master"), ReturnCode::OK);
  EXPECT_EQ(follower_host.removeDB("master"), ReturnCode::DB_NOT_FOUND);
  EXPECT_EQ(leader_host.removeDB("master"), ReturnCode::OK);
}

// what a follower's log must hold: the leader's batches, in order, each followed by the follower's own LogData(ts)
static bool follower_matches(CountingDb& leader, CountingDb& follower) {
  std::lock_guard<std::mutex> g1(leader.mu_);
  std::lock_guard<std::mutex> g2(follower.mu_);
  if (leader.log_.size() != follower.log_.size()) return false;
  for (size_t i = 0; i < leader.log_.size(); i++) {
    const std::string& a = leader.log_[i].second;
    const std::string& b = follower.log_[i].second;
    if (leader.log_[i].first != follower.log_[i].first) return false;
    if (b.size() != a.size() + 10 || b.compare(0, a.size(), a) != 0 || (uint8_t)b[a.size()] != 0x03 || (uint8_t)b[a.size() + 1] != 8) return false;
  }
  return true;
}

// rocksdb_replicator_test.cpp:210-268: two followers pulling from the same leader
static void test_tree_counting() {
  fast_flags();
  RocksDBReplicator leader_host(19101), f1_host(19102), f2_host(19103);
  auto ldb = std::make_shared<CountingDb>(), f1 = std::make_shared<CountingDb>(), f2 = std::make_shared<CountingDb>();
  EXPECT_EQ(leader_host.addDB("shard1", std::static_pointer_cast<DbWrapper>(ldb), ReplicaRole::LEADER), ReturnCode::OK);
  EXPECT_EQ(f1_host.addDB("shard1", std::static_pointer_cast<DbWrapper>(f1), ReplicaRole::FOLLOWER, SocketAddress("127.0.0.1", 19101)), ReturnCode::OK);
  EXPECT_EQ(f2_host.addDB("shard1", std::static_pointer_cast<DbWrapper>(f2), ReplicaRole::FOLLOWER, SocketAddress("127.0.0.1", 19101)), ReturnCode::OK);
  rocksdb::WriteOptions wo;
  for (uint32_t i = 0; i < 100; i++) {
    WriteBatch b;
    b.Put(std::to_string(i) + "key", std::to_string(i) + "value");
    EXPECT_EQ(leader_host.write("shard1", wo, &b), ReturnCode::OK);
    EXPECT_EQ(ldb->LatestSequenceNumber(), (uint64_t)i + 1);
  }
  EXPECT_TRUE(wait_until([&] { return f1->LatestSequenceNumber() == 100 && f2->LatestSequenceNumber() == 100; }));
  EXPECT_TRUE(follower_matches(*ldb, *f1));
  EXPECT_TRUE(follower_matches(*ldb, *f2));
  f1_host.removeDB("shard1"); f2_host.removeDB("shard1"); leader_host.removeDB("shard1");
}

// rocksdb_replicator_test.cpp:372-428 and :430-492: a follower whose upstream is itself, and two followers whose
// upstreams are each other, never see the leader's writes; empty responses from a non-leader make them try to reset
// their upstream (which cannot succeed without a cluster manager), the leader never does
static void test_upstream_reset_counting() {
  fast_flags();
  auto& F = Flags();
  F.replicator_max_server_wait_time_ms = 100;
  F.replicator_client_server_timeout_difference_ms = 100;
  F.reset_upstream_on_empty_updates_from_non_leader = true;
  F.replicator_max_consecutive_no_updates_before_upstream_reset = 1;
  {
    RocksDBReplicator leader_host(19104), self_host(19105), a_host(19106), b_host(19107);
    auto ldb = std::make_shared<CountingDb>(), sdb = std::make_shared<CountingDb>(), adb = std::make_shared<CountingDb>(), bdb = std::make_shared<CountingDb>();
    RocksDBReplicator::ReplicatedDB *rl = nullptr, *rs = nullptr, *ra = nullptr, *rb = nullptr;
    EXPECT_EQ(leader_host.addDB("shard1", std::static_pointer_cast<DbWrapper>(ldb), ReplicaRole::LEADER, SocketAddress(), &rl), ReturnCode::OK);
    EXPECT_EQ(self_host.addDB("shard1", std::static_pointer_cast<DbWrapper>(sdb), ReplicaRole::FOLLOWER, SocketAddress("127.0.0.1", 19105), &rs), ReturnCode::OK);
    EXPECT_EQ(a_host.addDB("shard1", std::static_pointer_cast<DbWrapper>(adb), ReplicaRole::FOLLOWER, SocketAddress("127.0.0.1", 19107), &ra), ReturnCode::OK);
    EXPECT_EQ(b_host.addDB("shard1", std::static_pointer_cast<DbWrapper>(bdb), ReplicaRole::FOLLOWER, SocketAddress("127.0.0.1", 19106), &rb), ReturnCode::OK);
    rocksdb::WriteOptions wo;
    for (uint32_t i = 0; i < 100; i++) {
      WriteBatch b;
      b.Put(std::to_string(i) + "key", std::to_string(i) + "value");
      b.Put(std::to_string(i) + "key2", std::to_string(i) + "value2");
      EXPECT_EQ(leader_host.write("shard1", wo, &b), ReturnCode::OK);
    }
    EXPECT_EQ(ldb->LatestSequenceNumber(), 200u);
    EXPECT_TRUE(wait_until([&] { return rs->resetUpstreamAttempts() != 0 && ra->resetUpstreamAttempts() != 0 && rb->resetUpstreamAttempts() != 0; }, 3000));
    EXPECT_EQ(rl->resetUpstreamAttempts(), 0u);
    EXPECT_EQ(sdb->LatestSequenceNumber(), 0u);
    EXPECT_EQ(adb->LatestSequenceNumber(), 0u);
    EXPECT_EQ(bdb->LatestSequenceNumber(), 0u);
    self_host.removeDB("shard1"); a_host.removeDB("shard1"); b_host.removeDB("shard1"); leader_host.removeDB("shard1");
  }
  Flags() = ReplicatorFlags();
  fast_flags();
}

// rocksdb_replicator_test.cpp:740-823: 20 shards over three hosts, leader on host i % 3, followers on the other two;
// every write is offered to all three hosts and lands only on the shard's leader
static void test_stress_counting() {
  fast_flags();
  const int n_shards = 20;
  const uint32_t n_keys = 100;
  const uint16_t ports[3] = {19108, 19109, 19110};
  RocksDBReplicator h0(ports[0]), h1(ports[1]), h2(ports[2]);
  RocksDBReplicator* hosts[3] = {&h0, &h1, &h2};
  std::vector<std::shared_ptr<CountingDb>> leaders, f1s, f2s;
  for (int i = 0; i < n_shards; i++) {
    leaders.push_back(std::make_shared<CountingDb>());
    f1s.push_back(std::make_shared<CountingDb>());
    f2s.push_back(std::make_shared<CountingDb>());
    const std::string shard = "shard" + std::to_string(i);
    const int start = i % 3;
    EXPECT_EQ(hosts[start]->addDB(shard, std::static_pointer_cast<DbWrapper>(leaders[i]), ReplicaRole::LEADER), ReturnCode::OK);
    EXPECT_EQ(hosts[(start + 1) % 3]->addDB(shard, std::static_pointer_cast<DbWrapper>(f1s[i]), ReplicaRole::FOLLOWER, SocketAddress("127.0.0.1", ports[start])), ReturnCode::OK);
    EXPECT_EQ(hosts[(start + 2) % 3]->addDB(shard, std::static_pointer_cast<DbWrapper>(f2s[i]), ReplicaRole::FOLLOWER, SocketAddress("127.0.0.1", ports[start])), ReturnCode::OK);
  }
  rocksdb::WriteOptions wo;
  int bad_codes = 0;
  for (uint32_t i = 0; i < n_keys; i++)
    for (int j = 0; j < n_shards; j++) {
      const std::string shard = "shard" + std::to_string(j);
      WriteBatch b;
      b.Put(std::to_string(i) + "key", std::to_string(i) + "value");
      int oks = 0;
      for (auto* h : hosts) {
        const ReturnCode rc = h->write(shard, wo, &b);
        if (rc == ReturnCode::OK) oks++;
        else if (rc != ReturnCode::WRITE_TO_SLAVE) bad_codes++;
      }
      if (oks != 1) bad_codes++;
    }
  EXPECT_EQ(bad_codes, 0);
  for (int i = 0; i < n_shards; i++) {
    EXPECT_EQ(leaders[i]->LatestSequenceNumber(), (uint64_t)n_keys);
    EXPECT_TRUE(wait_until([&] { return f1s[i]->LatestSequenceNumber() == n_keys && f2s[i]->LatestSequenceNumber() == n_keys; }));
    EXPECT_TRUE(follower_matches(*leaders[i], *f1s[i]));
    EXPECT_TRUE(follower_matches(*leaders[i], *f2s[i]));
  }
  for (int i = 0; i < n_shards; i++)
    for (auto* h : hosts) EXPECT_EQ(h->removeDB("shard" + std::to_string(i)), ReturnCode::OK);
}

// rocksdb_replicator_test.cpp:494-624 (2-ACK mode: success, timeout, degradation) and :626-738 (observer is no ACK)
static void test_ack_modes_counting() {
  fast_flags();
  auto& F = Flags();
  F.replicator_replication_mode = 2;
  F.replicator_timeout_ms = 300;
  F.replicator_timeout_degraded_ms = 5;
  F.replicator_consecutive_ack_timeout_before_degradation = 3;
  {
    RocksDBReplicator leader_host(19093), follower_host(19094), observer_host(19095);
    auto ldb = std::make_shared<CountingDb>(), fdb = std::make_shared<CountingDb>(), odb = std::make_shared<CountingDb>();
    RocksDBReplicator::ReplicatedDB* rl = nullptr;
    leader_host.addDB("db", std::static_pointer_cast<DbWrapper>(ldb), ReplicaRole::LEADER, SocketAddress(), &rl);
    rocksdb::WriteOptions wo;
    // no follower yet: the write commits on the leader but times out waiting for the ACK
    WriteBatch b1; b1.Put("a", "1");
    Status s = rl->Write(wo, &b1);
    EXPECT_TRUE(s == Status::TimedOut("Failed to receive ack from follower"));
    EXPECT_EQ(ldb->LatestSequenceNumber(), 1u);
    // an OBSERVER pulling does not count as an ACK
    observer_host.addDB("db", std::static_pointer_cast<DbWrapper>(odb), ReplicaRole::OBSERVER, SocketAddress("127.0.0.1", 19093));
    EXPECT_TRUE(wait_until([&] { return odb->LatestSequenceNumber() == 1; }));
    WriteBatch b2; b2.Put("a", "2");
    EXPECT_TRUE(rl->Write(wo, &b2).IsTimedOut());
    WriteBatch b3; b3.Put("a", "3");
    EXPECT_TRUE(rl->Write(wo, &b3).IsTimedOut());  // third consecutive timeout: degraded to 5 ms
    EXPECT_TRUE(rl->Introspect().find("current_replicator_timeout_ms_: 5\n") != std::string::npos);
    // a real follower ACKs: writes succeed again and the timeout recovers
    follower_host.addDB("db", std::static_pointer_cast<DbWrapper>(fdb), ReplicaRole::FOLLOWER, SocketAddress("127.0.0.1", 19093));
    EXPECT_TRUE(wait_until([&] { return fdb->LatestSequenceNumber() == 3; }));
    bool ok = false;
    for (int i = 0; i < 50 && !ok; i++) { WriteBatch b; b.Put("k", "v"); ok = rl->Write(wo, &b).ok(); }
    EXPECT_TRUE(ok);
    EXPECT_TRUE(rl->Introspect().find("current_replicator_timeout_ms_: 300\n") != std::string::npos);
    observer_host.removeDB("db"); follower_host.removeDB("db"); leader_host.removeDB("db");
  }
  fast_flags();
}

// common/dbconfig: per-dataset ack mode from the reference's JSON document; max(flag, dataset) is what Write uses
static void test_dbconfig_and_stats() {
  fast_flags();
  auto* cfg = common::DBConfigManager::get();
  cfg->clear();
  EXPECT_EQ(cfg->getReplicationMode("seg00001"), 0u);
  EXPECT_TRUE(cfg->loadJsonText("{\"dataset\": {\"seg\": {\"ack_mode\": 2, \"other\": [1, {\"x\": null}]}, \"b\": {\"ack_mode\": 1}}, \"v\": \"1\"}"));
  EXPECT_EQ(cfg->getReplicationMode("seg00001"), 2u);
  EXPECT_EQ(cfg->getReplicationMode("b00042"), 1u);
  EXPECT_EQ(cfg->getReplicationMode("zzz00001", 7), 7u);
  EXPECT_TRUE(!cfg->loadJsonText("{\"dataset\": {\"seg\": {\"ack_mode\": }}}"));  // malformed: config unchanged
  EXPECT_EQ(cfg->getReplicationMode("seg00001"), 2u);
  // dataset "seg" is in 2-ACK mode through the config alone (flag stays 0): a leader without followers times out
  Flags().replicator_timeout_ms = 100;
  const uint64_t timed_out_before = common::Stats::get()->GetCounter(kReplicatorWriteWaitTimedOut);
  const uint64_t success_before = common::Stats::get()->GetCounter(kReplicatorWriteSuccess);
  {
    RocksDBReplicator host(19141);
    auto db = std::make_shared<CountingDb>(), db2 = std::make_shared<CountingDb>();
    RocksDBReplicator::ReplicatedDB *r = nullptr, *r2 = nullptr;
    host.addDB("seg00001", std::static_pointer_cast<DbWrapper>(db), ReplicaRole::LEADER, SocketAddress(), &r);
    host.addDB("plain00001", std::static_pointer_cast<DbWrapper>(db2), ReplicaRole::LEADER, SocketAddress(), &r2);
    WriteBatch b; b.Put("k", "v");
    EXPECT_TRUE(r->Write(rocksdb::WriteOptions(), &b).IsTimedOut());
    WriteBatch b2; b2.Put("k", "v");
    EXPECT_TRUE(r2->Write(rocksdb::WriteOptions(), &b2).ok());  // other datasets stay in mode 0
    host.removeDB("seg00001"); host.removeDB("plain00001");
  }
  EXPECT_EQ(common::Stats::get()->GetCounter(kReplicatorWriteWaitTimedOut), timed_out_before + 1);
  EXPECT_EQ(common::Stats::get()->GetCounter(kReplicatorWriteSuccess), success_before + 1);
  EXPECT_TRUE(common::Stats::get()->GetCounter(kReplicatorWriteBytes) > 0);
  StatFlags().replicator_enable_per_dataset_stats = true;
  EXPECT_EQ(TaggedName(kReplicatorPullRequests, "seg00007"), std::string("replicator_pull_requests dataset=seg"));
  StatFlags().replicator_enable_per_dataset_stats = false;
  cfg->clear();
  fast_flags();
}

// ---- GPU-backed: the DB below the seam is the GPU engine -----------------------------------------------
class CounterMergeOperator : public rocksdb::AssociativeMergeOperator {  // examples/counter_service/merge_operator.cpp
 public:
  bool Merge(const Slice&, const Slice* existing, const Slice& value, std::string* nv, rocksdb::Logger*) const override {
    if (!existing) { *nv = value.ToString(); return true; }
    if (existing->size() != 8 || value.size() != 8) return false;
    int64_t a, b; memcpy(&a, existing->data(), 8); memcpy(&b, value.data(), 8); b += a;
    nv->assign((const char*)&b, 8); return true;
  }
  const char* Name() const override { return "CounterMergeOperator"; }
};
class SimpleMergeOperator : public rocksdb::AssociativeMergeOperator {  // rocksdb_assumption_test.cpp:58-77
 public:
  bool Merge(const Slice&, const Slice* existing, const Slice& value, std::string* nv, rocksdb::Logger*) const override {
    if (existing) *nv = existing->ToString();
    *nv += value.ToString();
    return true;
  }
  const char* Name() const override { return "SimpleMergeOperator"; }
};

static std::shared_ptr<rocksdb::DB> open_gpu(const std::string& name, std::shared_ptr<rocksdb::MergeOperator> mo = nullptr) {
  rocksdb::Options o;
  o.create_if_missing = true;
  o.merge_operator = mo;
  o.write_buffer_size = 1 << 20;
  rocksdb::DB* db = nullptr;
  Status s = b200::GpuDB::Open(o, name, &db);
  if (!s.ok()) { printf("  GpuDB::Open(%s): %s\n", name.c_str(), s.ToString().c_str()); g_fail++; return nullptr; }
  return std::shared_ptr<rocksdb::DB>(db);
}

// rocksdb_assumption_test.cpp:136-187: sequence arithmetic
static void test_gpu_sequence_numbers() {
  auto db = open_gpu("assumption_seq", std::make_shared<SimpleMergeOperator>());
  if (!db) return;
  rocksdb::WriteOptions wo; rocksdb::ReadOptions ro;
  EXPECT_EQ(db->GetLatestSequenceNumber(), 0u);
  EXPECT_TRUE(db->Put(wo, "key", "value").ok());
  EXPECT_EQ(db->GetLatestSequenceNumber(), 1u);
  std::string v;
  EXPECT_TRUE(db->Get(ro, "key", &v).ok() && v == "value");
  EXPECT_EQ(db->GetLatestSequenceNumber(), 1u);  // Get consumes none
  EXPECT_TRUE(db->Delete(wo, "key").ok());
  EXPECT_EQ(db->GetLatestSequenceNumber(), 2u);
  EXPECT_TRUE(db->Get(ro, "key", &v).IsNotFound());
  EXPECT_TRUE(db->Merge(wo, "key", "m").ok());
  EXPECT_EQ(db->GetLatestSequenceNumber(), 3u);
  WriteBatch b; b.Delete("a"); b.Put("b", "1"); b.Put("c", "2"); b.Merge("b", "3");
  EXPECT_TRUE(db->Write(wo, &b).ok());
  EXPECT_EQ(db->GetLatestSequenceNumber(), 7u);
  EXPECT_TRUE(db->Get(ro, "b", &v).ok() && v == "13");
  std::vector<std::string> vals;
  auto sts = db->MultiGet(ro, {Slice("b"), Slice("zz"), Slice("c")}, &vals);
  EXPECT_TRUE(sts[0].ok() && vals[0] == "13" && sts[1].IsNotFound() && sts[2].ok() && vals[2] == "2");
  // GetUpdatesSince(seq + 1) returns the batch whose sequence == seq + 1 (rocksdb_assumption_test.cpp:329-359)
  std::unique_ptr<rocksdb::TransactionLogIterator> it;
  EXPECT_TRUE(db->GetUpdatesSince(4, &it).ok() && it->Valid());
  auto br = it->GetBatch();
  EXPECT_EQ(br.sequence, 4u);
  EXPECT_EQ(br.writeBatchPtr->Count(), 4);
  EXPECT_TRUE(db->GetUpdatesSince(8, &it).IsNotFound());
  // iterator: sst_binary.cpp:43-58 style
  for (int i = 0; i < 10; i++) db->Put(wo, "key" + std::to_string(i), "value" + std::to_string(i));
  std::unique_ptr<rocksdb::Iterator> iter(db->NewIterator(ro));
  int n = 0;
  for (iter->Seek("key0"); iter->Valid() && n < 10; iter->Next(), n++) {
    EXPECT_EQ(iter->key().ToString(), "key" + std::to_string(n));
    EXPECT_EQ(iter->value().ToString(), "value" + std::to_string(n));
  }
  EXPECT_EQ(n, 10);
  EXPECT_TRUE(db->CompactRange(rocksdb::CompactRangeOptions(), nullptr, nullptr).ok());
  n = 0;
  iter.reset(db->NewIterator(ro));
  for (iter->Seek("key0"); iter->Valid() && n < 10; iter->Next(), n++) EXPECT_EQ(iter->value().ToString(), "value" + std::to_string(n));
  EXPECT_EQ(n, 10);
}

// backup / bulk load through SST files: ExportSstFile -> IngestExternalFile (admin_handler.cpp:1820-1845), with the
// sequence rules of rocksdb_assumption_test.cpp:248-283 (empty target: none consumed; overlap: +1; refused without
// allow_global_seqno)
static void test_gpu_export_and_ingest() {
  auto src = open_gpu("sst_src", std::make_shared<SimpleMergeOperator>());
  if (!src) return;
  rocksdb::WriteOptions wo; rocksdb::ReadOptions ro;
  std::map<std::string, std::string> want;
  for (int i = 0; i < 2000; i++) {
    char k[32]; snprintf(k, sizeof(k), "key%06d", i * 3);
    const std::string v = "value" + std::to_string(i) + std::string(i % 97, 'x');
    EXPECT_TRUE(src->Put(wo, k, v).ok());
    want[k] = v;
  }
  EXPECT_TRUE(src->Merge(wo, "key000003", "+m").ok()); want["key000003"] += "+m";
  EXPECT_TRUE(src->Delete(wo, "key000006").ok()); want.erase("key000006");
  const char* tdir = getenv("TMPDIR") ? getenv("TMPDIR") : "/tmp";
  const std::string path = std::string(tdir) + "/rsp_host_test_" + std::to_string((long)getpid()) + ".sst";
  uint64_t n = 0;
  auto* gsrc = static_cast<b200::GpuDB*>(src.get());
  EXPECT_TRUE(gsrc->ExportSstFile(path, &n).ok());
  EXPECT_EQ(n, (uint64_t)want.size());
  auto dst = open_gpu("sst_dst", std::make_shared<SimpleMergeOperator>());
  rocksdb::IngestExternalFileOptions io;
  EXPECT_TRUE(dst->IngestExternalFile({path}, io).ok());
  EXPECT_EQ(dst->GetLatestSequenceNumber(), 0u);
  {
    std::unique_ptr<rocksdb::Iterator> it(dst->NewIterator(ro));
    auto w = want.begin();
    size_t seen = 0;
    for (it->SeekToFirst(); it->Valid() && w != want.end(); it->Next(), ++w, seen++) {
      if (it->key().ToString() != w->first || it->value().ToString() != w->second) break;
    }
    EXPECT_EQ(seen, want.size());
    EXPECT_TRUE(!it->Valid());
  }
  std::string v;
  EXPECT_TRUE(dst->Get(ro, "key000003", &v).ok() && v == want["key000003"]);
  EXPECT_TRUE(dst->Get(ro, "key000006", &v).IsNotFound());
  // the same file again overlaps what is there: refused without global sequence numbers, else last + 1
  io.allow_global_seqno = false;
  Status st = dst->IngestExternalFile({path}, io);
  EXPECT_TRUE(st.IsInvalidArgument());
  EXPECT_EQ(dst->GetLatestSequenceNumber(), 0u);
  io.allow_global_seqno = true;
  EXPECT_TRUE(dst->Put(wo, "key000003", "newer").ok());
  EXPECT_TRUE(dst->IngestExternalFile({path}, io).ok());
  EXPECT_EQ(dst->GetLatestSequenceNumber(), 2u);
  EXPECT_TRUE(dst->Get(ro, "key000003", &v).ok() && v == want["key000003"]);  // the ingested file is the newest
  EXPECT_TRUE(dst->IngestExternalFile({path + ".missing"}, io).IsIOError());
  EXPECT_TRUE(dst->IngestExternalFile({}, io).IsInvalidArgument());
  io.move_files = true;
  auto dst2 = open_gpu("sst_dst2", nullptr);
  EXPECT_TRUE(dst2->IngestExternalFile({path}, io).ok());
  FILE* gone = fopen(path.c_str(), "rb");
  EXPECT_TRUE(gone == nullptr);
  if (gone) fclose(gone);
  remove(path.c_str());
}

// rocksdb_replicator_test.cpp:146-208 + :270-368 with real engines: leader -> follower -> chained follower
static void test_gpu_replication_chain() {
  fast_flags();
  RocksDBReplicator h1(19101), h2(19102), h3(19103);
  auto d1 = open_gpu("chain_leader"), d2 = open_gpu("chain_mid"), d3 = open_gpu("chain_tail");
  if (!d1 || !d2 || !d3) return;
  RocksDBReplicator::ReplicatedDB* rl = nullptr;
  EXPECT_EQ(h1.addDB("shard", d1, ReplicaRole::LEADER, SocketAddress(), &rl), ReturnCode::OK);
  EXPECT_EQ(h2.addDB("shard", d2, ReplicaRole::FOLLOWER, SocketAddress("127.0.0.1", 19101)), ReturnCode::OK);
  EXPECT_EQ(h3.addDB("shard", d3, ReplicaRole::FOLLOWER, SocketAddress("127.0.0.1", 19102)), ReturnCode::OK);
  rocksdb::WriteOptions wo; rocksdb::ReadOptions ro;
  const int n = 100;
  for (int i = 0; i < n; i++) {
    WriteBatch b;
    b.Put(std::to_string(i) + "key", std::to_string(i) + "value");
    b.Put(std::to_string(i) + "key2", std::to_string(i) + "value2");
    EXPECT_TRUE(rl->Write(wo, &b).ok());
  }
  EXPECT_TRUE(wait_until([&] { return d3->GetLatestSequenceNumber() == (uint64_t)2 * n; }));
  EXPECT_EQ(d1->GetLatestSequenceNumber(), (uint64_t)2 * n);
  EXPECT_EQ(d2->GetLatestSequenceNumber(), (uint64_t)2 * n);
  for (int i = 0; i < n; i++) {
    std::string v;
    EXPECT_TRUE(d3->Get(ro, std::to_string(i) + "key", &v).ok() && v == std::to_string(i) + "value");
    EXPECT_TRUE(d2->Get(ro, std::to_string(i) + "key2", &v).ok() && v == std::to_string(i) + "value2");
  }
  // remove the middle node and re-add it: the tail catches up again (rocksdb_replicator_test.cpp:318-368)
  EXPECT_EQ(h2.removeDB("shard"), ReturnCode::OK);
  for (int i = n; i < 2 * n; i++) { WriteBatch b; b.Put(std::to_string(i) + "key", "v"); EXPECT_TRUE(rl->Write(wo, &b).ok()); }
  EXPECT_EQ(h2.addDB("shard", d2, ReplicaRole::FOLLOWER, SocketAddress("127.0.0.1", 19101)), ReturnCode::OK);
  EXPECT_TRUE(wait_until([&] { return d3->GetLatestSequenceNumber() == (uint64_t)3 * n; }, 20000));
  // the leader's timestamp LogData is extractable downstream (admin_handler_test.cpp:681-697, checkDB)
  std::unique_ptr<rocksdb::TransactionLogIterator> it;
  EXPECT_TRUE(d3->GetUpdatesSince(1, &it).ok() && it->Valid());
  LogExtractor ex;
  EXPECT_TRUE(it->GetBatch().writeBatchPtr->Iterate(&ex).ok());
  EXPECT_TRUE(ex.ms > 1500000000000ull);
  h3.removeDB("shard"); h2.removeDB("shard"); h1.removeDB("shard");
}

// rocksdb_assumption_test.cpp:361-432: {Put, Merge, Merge, Delete} batches, follower equal to leader
static void test_gpu_follower_equals_leader() {
  fast_flags();
  RocksDBReplicator h1(19111), h2(19112);
  auto mo = std::make_shared<SimpleMergeOperator>();
  auto d1 = open_gpu("eq_leader", mo), d2 = open_gpu("eq_follower", mo);
  if (!d1 || !d2) return;
  RocksDBReplicator::ReplicatedDB* rl = nullptr;
  h1.addDB("db", d1, ReplicaRole::LEADER, SocketAddress(), &rl);
  h2.addDB("db", d2, ReplicaRole::FOLLOWER, SocketAddress("127.0.0.1", 19111));
  const int nKeys = 100, nOps = 1000;
  std::vector<std::string> keys, values;
  for (int i = 0; i < nKeys; i++) { keys.push_back(std::to_string(i)); values.push_back("value" + std::to_string(i)); }
  rocksdb::WriteOptions wo; rocksdb::ReadOptions ro;
  for (int j = 0; j < nOps; j++) {
    const int i = (j * 7919) % nOps;  // a fixed shuffle
    WriteBatch b;
    b.Put(keys[i % nKeys], values[i % nKeys]);
    b.Merge(keys[i % nKeys], values[i % nKeys]);
    b.Merge(keys[(i + 1) % nKeys], values[(i + 1) % nKeys]);
    b.Delete(keys[(i + 2) % nKeys]);
    EXPECT_TRUE(rl->Write(wo, &b).ok());
    if (j % 250 == 100) d2->Flush(rocksdb::FlushOptions());
  }
  EXPECT_TRUE(wait_until([&] { return d2->GetLatestSequenceNumber() == (uint64_t)4 * nOps; }, 30000));
  for (int i = 0; i < nKeys; i++) {
    std::string a, b;
    Status sa = d1->Get(ro, keys[i], &a), sb = d2->Get(ro, keys[i], &b);
    EXPECT_TRUE(sa == sb);
    if (sa.ok()) EXPECT_EQ(a, b);
  }
  h2.removeDB("db"); h1.removeDB("db");
}

// BASELINE config #1 — examples/counter_service: 4 shards x 1000 keys, setCounter (Put) + bumpCounter
// (int64 Merge) through ApplicationDB::Write on the leader, getCounter through ApplicationDB::Get on the follower
static void test_counter_service_config1() {
  fast_flags();
  RocksDBReplicator leader_host(19121), follower_host(19122);
  admin::ApplicationDBManager lm(&leader_host), fm(&follower_host);
  auto mo = std::make_shared<CounterMergeOperator>();
  const int shards = 4, keys = 1000;
  std::string err;
  for (int s = 0; s < shards; s++) {
    const std::string name = common::SegmentToDbName("counter", s);
    rocksdb::Options o; o.merge_operator = mo; o.write_buffer_size = 1 << 20;
    rocksdb::DB *l = nullptr, *f = nullptr;
    EXPECT_TRUE(b200::GpuDB::Open(o, "L" + name, &l).ok());
    EXPECT_TRUE(b200::GpuDB::Open(o, "F" + name, &f).ok());
    EXPECT_TRUE(lm.addDB(name, std::unique_ptr<rocksdb::DB>(l), ReplicaRole::LEADER, &err));
    EXPECT_TRUE(fm.addDB(name, std::unique_ptr<rocksdb::DB>(f), ReplicaRole::FOLLOWER,
                         std::make_unique<SocketAddress>("127.0.0.1", 19121), &err));
  }
  // counter_router.cpp:23-30: Java String.hashCode-style shard hash
  auto shard_of = [&](const std::string& k) { int32_t h = 0; for (char c : k) h = 31 * h + c; return (int)((h < 0 ? -(int64_t)h : h) % shards); };
  rocksdb::WriteOptions wo; rocksdb::ReadOptions ro;
  std::vector<int64_t> want(keys, 0);
  for (int i = 0; i < keys; i++) {
    const std::string k = "counter_" + std::to_string(i);
    auto db = lm.getDB(common::SegmentToDbName("counter", shard_of(k)), &err);
    int64_t v = i;
    WriteBatch set; set.Put(k, Slice((const char*)&v, 8));              // counter_handler.cpp:152-158
    EXPECT_TRUE(db->Write(wo, &set).ok());
    for (int r = 0; r < 3; r++) {
      int64_t d = r + 1;
      WriteBatch bump; bump.Merge(k, Slice((const char*)&d, 8));        // counter_handler.cpp:212-218
      EXPECT_TRUE(db->Write(wo, &bump).ok());
    }
    want[i] = i + 6;
  }
  for (int s = 0; s < shards; s++) {
    const std::string name = common::SegmentToDbName("counter", s);
    auto l = lm.getDB(name, &err), f = fm.getDB(name, &err);
    EXPECT_TRUE(wait_until([&] { return f->rocksdb()->GetLatestSequenceNumber() == l->rocksdb()->GetLatestSequenceNumber(); }, 30000));
    EXPECT_TRUE(f->IsSlave() && !l->IsSlave());
  }
  for (int i = 0; i < keys; i++) {
    const std::string k = "counter_" + std::to_string(i);
    auto f = fm.getDB(common::SegmentToDbName("counter", shard_of(k)), &err);
    std::string v;
    EXPECT_TRUE(f->Get(ro, k, &v).ok() && v.size() == 8);               // counter_handler.cpp:88
    int64_t got = 0; memcpy(&got, v.data(), v.size() == 8 ? 8 : 0);
    EXPECT_EQ(got, want[i]);
  }
  // writes to a follower are refused (ReturnCode::WRITE_TO_SLAVE thrown through ApplicationDB::Write)
  bool thrown = false;
  try { WriteBatch b; b.Put("x", "y"); fm.getDB("counter00000", &err)->Write(wo, &b); } catch (ReturnCode rc) { thrown = rc == ReturnCode::WRITE_TO_SLAVE; }
  EXPECT_TRUE(thrown);
}

// application_db_manager_test.cpp:40-85: exact Introspect strings, add/remove semantics
static void test_application_db_manager() {
  fast_flags();
  RocksDBReplicator host(19131);
  admin::ApplicationDBManager m(&host);
  std::string err;
  rocksdb::DB* raw = nullptr;
  EXPECT_TRUE(b200::GpuDB::Open(rocksdb::Options(), "adm_test_db", &raw).ok());
  EXPECT_TRUE(m.addDB("test_db", std::unique_ptr<rocksdb::DB>(raw), ReplicaRole::LEADER, &err));
  EXPECT_TRUE(!m.addDB("test_db", nullptr, ReplicaRole::LEADER, &err));
  EXPECT_TRUE(m.getDB("test_db", &err) != nullptr);
  EXPECT_EQ(m.Introspect(), std::string("ApplicationDBManager:\ntest_db:\n ReplicatedDB:\n  name: test_db\n  ReplicaRole: LEADER\n  upstream_addr: uninitialized_addr\n  cur_seq_no: 0\n  current_replicator_timeout_ms_: 2000\n\n"));
  // admin_handler_test.cpp:218-265: write / delete then Get / NotFound through ApplicationDB; :681-697 seq after one Delete
  auto adb = m.getDB("test_db", &err);
  rocksdb::WriteOptions wo; rocksdb::ReadOptions ro;
  WriteBatch del; del.Delete("a");
  EXPECT_TRUE(adb->Write(wo, &del).ok());
  EXPECT_EQ(adb->rocksdb()->GetLatestSequenceNumber(), 1u);
  WriteBatch put; put.Put("a", "1");
  EXPECT_TRUE(adb->Write(wo, &put).ok());
  std::string v;
  EXPECT_TRUE(adb->Get(ro, "a", &v).ok() && v == "1");
  rocksdb::PinnableSlice ps;
  EXPECT_TRUE(adb->Get(ro, "a", &ps).ok() && ps.ToString() == "1");
  EXPECT_TRUE(adb->Get(ro, "nope", &v).IsNotFound());
  std::string prop;
  EXPECT_TRUE(adb->GetProperty(admin::ApplicationDB::Properties::kNumLevels, &prop) && prop == "7");
  EXPECT_TRUE(adb->CompactRange(rocksdb::CompactRangeOptions(), nullptr, nullptr).ok());
  EXPECT_TRUE(adb->Get(ro, "a", &v).ok() && v == "1");
  adb.reset();
  auto back = m.removeDB("test_db", &err);
  EXPECT_TRUE(back != nullptr);
  EXPECT_TRUE(m.removeDB("test_db", &err) == nullptr);
  back.reset();
  EXPECT_TRUE(b200::GpuDB::Open(rocksdb::Options(), "adm_test_db1", &raw).ok());
  EXPECT_TRUE(m.addDB("test_db1", std::unique_ptr<rocksdb::DB>(raw), ReplicaRole::FOLLOWER, &err));
  EXPECT_EQ(m.Introspect(), std::string("ApplicationDBManager:\ntest_db1:\n __no_replicated_db__\n"));
}

// the hot path through the reference's seams (host/bench/seam_bench.cpp): followers pull from a synthetic leader through
// RocksDBReplicator / DbWrapper, readers call ApplicationDB::MultiGet / Get from several threads, updates race reads;
// every value read back is checked against the generator
#include "bench/seam_bench.h"
static void test_gpu_seams() {
  rsp_seam_cfg c;
  memset(&c, 0, sizeof(c));
  c.shards = 6; c.kv_total = 6 * 700; c.value_len = 64; c.executor_threads = 16; c.updates_per_response = 50; c.update_rounds = 4;
  c.multiget_threads = 4; c.multiget_batch = 256; c.multiget_secs = 0.3; c.get_threads = 4; c.get_secs = 0.2; c.first_shard_id = 40;
  c.steady_rounds = 3;
  rsp_seam_result r;
  EXPECT_EQ(rsp_seam_bench(&c, &r), 0);
  EXPECT_EQ(r.parity_errors, (uint64_t)0);
  EXPECT_EQ(r.status_errors, (uint64_t)0);
  EXPECT_EQ(r.applied_total, (uint64_t)(6 * (700 + 4 * 50 + 3 * 50)));
  EXPECT_TRUE(r.mget_calls > 0 && r.get_per_s > 0 && r.load_applies_per_s > 0 && r.mixed_applies_per_s > 0 && r.steady_applies_per_s > 0);
  EXPECT_TRUE(r.trace_us[0] > 0 && r.apply_comb[1] >= 6 * 3 * 50);
  printf("  seams: load %.0f applies/s, MultiGet %.0f lookups/s (%llu calls), Get %.0f /s, mixed %.0f applies/s + %.0f lookups/s\n",
         r.load_applies_per_s, r.mget_lookups_per_s, (unsigned long long)r.mget_calls, r.get_per_s, r.mixed_applies_per_s, r.mixed_lookups_per_s);
  c.value_len = 256; c.first_shard_id = 60; c.update_rounds = 0; c.steady_rounds = 0;  // config-5 shape: 256-byte values
  EXPECT_EQ(rsp_seam_bench(&c, &r), 0);
  EXPECT_EQ(r.parity_errors + r.status_errors, (uint64_t)0);
}

// HBM is volatile: backup = visible contents as one SST + dbmeta (sequence number); restore = a fresh shard that
// continues at that sequence number; the scheduler spills shards whose sequence number moved
// (rocksdb_admin/admin_handler.cpp:696-860 backupDBHelper / restoreDBHelper)
static void test_gpu_backup_restore() {
  rocksdb::Options opt;
  opt.merge_operator = std::make_shared<CounterMergeOperator>();
  rocksdb::DB* raw = nullptr;
  EXPECT_TRUE(b200::GpuDB::Open(opt, "bk_src00001", &raw).ok());
  std::shared_ptr<rocksdb::DB> src(raw);
  for (int i = 0; i < 500; i++) {
    WriteBatch wb;
    wb.Put("key" + std::to_string(i), "value" + std::to_string(i));
    if (i % 7 == 0) wb.Delete("key" + std::to_string(i / 2));
    int64_t one = i;
    if (i % 5 == 0) wb.Merge("ctr" + std::to_string(i % 20), Slice((const char*)&one, 8));
    EXPECT_TRUE(src->Write(rocksdb::WriteOptions(), &wb).ok());
    if (i == 250) EXPECT_TRUE(src->Flush(rocksdb::FlushOptions()).ok());
  }
  const std::string root = "/tmp/rsp_bk_" + std::to_string(getpid());
  auto* gsrc = static_cast<b200::GpuDB*>(src.get());
  uint64_t seq = 0;
  EXPECT_TRUE(gsrc->Backup(root + "/manual", &seq).ok());
  EXPECT_EQ(seq, (uint64_t)src->GetLatestSequenceNumber());
  rocksdb::DB* raw2 = nullptr;
  EXPECT_TRUE(b200::GpuDB::Restore(opt, "bk_dst00001", root + "/manual", &raw2).ok());
  std::unique_ptr<rocksdb::DB> dst(raw2);
  EXPECT_TRUE(dst != nullptr);
  if (dst) {
    EXPECT_EQ(dst->GetLatestSequenceNumber(), src->GetLatestSequenceNumber());
    std::unique_ptr<rocksdb::Iterator> a(src->NewIterator(rocksdb::ReadOptions())), b(dst->NewIterator(rocksdb::ReadOptions()));
    size_t n = 0;
    for (a->SeekToFirst(), b->SeekToFirst(); a->Valid() && b->Valid(); a->Next(), b->Next(), n++) {
      EXPECT_TRUE(a->key() == b->key() && a->value() == b->value());
    }
    EXPECT_TRUE(!a->Valid() && !b->Valid() && n > 400);
    // the restored replica goes on from the backup's sequence number
    WriteBatch wb;
    wb.Put("after", "restore");
    EXPECT_TRUE(dst->Write(rocksdb::WriteOptions(), &wb).ok());
    EXPECT_EQ(dst->GetLatestSequenceNumber(), seq + 1);
  }
  // scheduled spilling: only shards whose sequence number moved are written again
  {
    b200::BackupScheduler sched(root + "/sched", 20);
    sched.Add("bk_src00001", src);
    EXPECT_TRUE(wait_until([&] { return sched.backups_done() >= 1; }));
    sleep_ms(100);
    const uint64_t done = sched.backups_done();
    EXPECT_EQ(done, (uint64_t)1);  // nothing moved: no second backup
    WriteBatch wb;
    wb.Put("more", "data");
    EXPECT_TRUE(src->Write(rocksdb::WriteOptions(), &wb).ok());
    EXPECT_TRUE(wait_until([&] { return sched.backups_done() >= 2; }));
    sched.Remove("bk_src00001");
  }
  rocksdb::DB* raw3 = nullptr;
  EXPECT_TRUE(b200::GpuDB::Restore(opt, "bk_dst00002", root + "/sched/bk_src00001", &raw3).ok());
  std::unique_ptr<rocksdb::DB> dst3(raw3);
  std::string v;
  EXPECT_TRUE(dst3 && dst3->Get(rocksdb::ReadOptions(), "more", &v).ok() && v == "data");
  EXPECT_TRUE(dst3 && dst3->GetLatestSequenceNumber() == src->GetLatestSequenceNumber());
  const std::string rm = "rm -rf '" + root + "'";
  EXPECT_EQ(system(rm.c_str()), 0);
}

// the Kafka-style writer front-end (rocksdb_admin/admin_handler.cpp:1855-2084): messages -> Put / Delete / Merge, one
// sequence number per message, a whole poll in one engine call; contents equal to the same operations issued one by one
static void test_gpu_message_ingestion() {
  struct VecSource : public admin::MessageSource {
    std::vector<admin::IngestMessage> all;
    size_t at = 0;
    size_t Poll(std::vector<admin::IngestMessage>* out, size_t max, int) override {
      size_t n = 0;
      while (at < all.size() && n < max) { out->push_back(all[at++]); n++; }
      if (!n) sleep_ms(1);
      return n;
    }
  };
  rocksdb::Options opt;
  opt.merge_operator = std::make_shared<CounterMergeOperator>();
  rocksdb::DB *ra = nullptr, *rb = nullptr;
  EXPECT_TRUE(b200::GpuDB::Open(opt, "kafka_a00001", &ra).ok());
  EXPECT_TRUE(b200::GpuDB::Open(opt, "kafka_b00001", &rb).ok());
  std::shared_ptr<rocksdb::DB> a(ra), b(rb);
  auto adb = std::make_shared<admin::ApplicationDB>("kafka_a00001", a, ReplicaRole::FOLLOWER, nullptr);
  auto src = std::make_shared<VecSource>();
  for (int i = 0; i < 5000; i++) {
    admin::IngestMessage m;
    m.key = "k" + std::to_string(i % 700);
    m.timestamp_ms = 1000 + i;
    m.offset = i;
    if (i % 11 == 0) { m.op_code = admin::KafkaOperationCode::DELETE; }
    else if (i % 5 == 0) { m.op_code = admin::KafkaOperationCode::MERGE; int64_t v = i; m.key = "c" + std::to_string(i % 30); m.value.assign((const char*)&v, 8); }
    else { m.op_code = admin::KafkaOperationCode::PUT; m.value = "v" + std::to_string(i); }
    if (i == 4321) m.op_code = (admin::KafkaOperationCode)9;  // invalid op code: counted and skipped
    src->all.push_back(m);
  }
  // the same operations one DB call at a time on the second shard
  for (auto& m : src->all) {
    if (m.op_code == admin::KafkaOperationCode::PUT) EXPECT_TRUE(b->Put(rocksdb::WriteOptions(), m.key, m.value).ok());
    else if (m.op_code == admin::KafkaOperationCode::DELETE) EXPECT_TRUE(b->Delete(rocksdb::WriteOptions(), m.key).ok());
    else if (m.op_code == admin::KafkaOperationCode::MERGE) EXPECT_TRUE(b->Merge(rocksdb::WriteOptions(), m.key, m.value).ok());
  }
  int64_t seen_ts = 0;
  admin::MessageIngestionOptions io;
  io.max_poll_messages = 512;
  io.on_timestamp = [&](int64_t t) { seen_ts = t; };
  admin::MessageIngestor ing(adb, src, io);
  ing.Start();
  EXPECT_TRUE(wait_until([&] { return ing.messages() == 5000; }));
  ing.Stop();
  EXPECT_EQ(ing.errors(), (uint64_t)0);
  EXPECT_TRUE(seen_ts >= 1000 + 4000);
  EXPECT_EQ(a->GetLatestSequenceNumber(), b->GetLatestSequenceNumber());  // one sequence number per valid message
  EXPECT_EQ(a->GetLatestSequenceNumber(), (uint64_t)4999);
  std::unique_ptr<rocksdb::Iterator> ia(a->NewIterator(rocksdb::ReadOptions())), ib(b->NewIterator(rocksdb::ReadOptions()));
  size_t n = 0;
  for (ia->SeekToFirst(), ib->SeekToFirst(); ia->Valid() && ib->Valid(); ia->Next(), ib->Next(), n++)
    EXPECT_TRUE(ia->key() == ib->key() && ia->value() == ib->value());
  EXPECT_TRUE(!ia->Valid() && !ib->Valid() && n > 300);
  // the ingested writes are in the update log: a downstream follower can pull them
  std::unique_ptr<rocksdb::TransactionLogIterator> li;
  EXPECT_TRUE(a->GetUpdatesSince(1, &li).ok() && li && li->Valid());
}

int main(int argc, char** argv) {
  const std::string mode = argc > 1 ? argv[1] : "cpu";
  // `only=<name>` (second argument) runs one test by name, whatever its mode
  const std::string only = argc > 2 ? argv[2] : "";
  struct T { const char* name; std::function<void()> fn; bool gpu; };
  std::vector<T> tests = {
      {"fast_read_map", test_fast_read_map, false},
      {"max_number_box", test_max_number_box, false},
      {"non_blocking_condition_variable", test_nbcv, false},
      {"write_batch_and_status", test_write_batch_and_status, false},
      {"stager", test_stager, false},
      {"replication_protocol_counting", test_replication_protocol_counting, false},
      {"tree_counting", test_tree_counting, false},
      {"upstream_reset_counting", test_upstream_reset_counting, false},
      {"stress_counting", test_stress_counting, false},
      {"ack_modes_counting", test_ack_modes_counting, false},
      {"dbconfig_and_stats", test_dbconfig_and_stats, false},
      {"gpu_sequence_numbers", test_gpu_sequence_numbers, true},
      {"gpu_export_and_ingest", test_gpu_export_and_ingest, true},
      {"gpu_replication_chain", test_gpu_replication_chain, true},
      {"gpu_follower_equals_leader", test_gpu_follower_equals_leader, true},
      {"counter_service_config1", test_counter_service_config1, true},
      {"application_db_manager", test_application_db_manager, true},
      {"gpu_seams", test_gpu_seams, true},
      {"gpu_backup_restore", test_gpu_backup_restore, true},
      {"gpu_message_ingestion", test_gpu_message_ingestion, true},
  };
  for (auto& t : tests) {
    if (!only.empty()) {
      if (only != t.name) continue;
    } else {
      if (t.gpu && mode != "gpu" && mode != "gpu-only") continue;
      if (!t.gpu && mode == "gpu-only") continue;
      if (std::string(t.name) == "gpu_export_and_ingest") continue;  // run by name from tests/test_zz_ingest_gpu.py
    }
    const int before = g_fail;
    printf("[ RUN  ] %s\n", t.name);
    fflush(stdout);
    t.fn();
    printf("[ %s ] %s\n", g_fail == before ? " OK " : "FAIL", t.name);
    fflush(stdout);
  }
  printf("%d checks, %d failures\n", g_checks, g_fail);
  return g_fail ? 1 : 0;
}
