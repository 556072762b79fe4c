// bounded_iter_tests.cpp — GpuDB / ApplicationDB iterators with ReadOptions::iterate_upper_bound (with and without
// ReadOptions::snapshot) and Iterator::SeekForPrev on a follower while replicated updates keep arriving through
// RocksDBReplicator.  Run by tests/test_bounded_iter_host_gpu.py.
#include <atomic>
#include <chrono>
#include <cstdio>
#include <memory>
#include <string>
#include <thread>
#include <vector>

#include "gpu_db.h"
#include "rocksdb_admin/application_db_manager.h"
#include "rocksdb_replicator/rocksdb_replicator.h"

using namespace replicator;
using rocksdb::Slice;
using rocksdb::WriteBatch;

static int g_checks = 0, g_fail = 0;
#define EXPECT_TRUE(c) do { g_checks++; if (!(c)) { g_fail++; printf("  FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); } } while (0)

template <class F> static bool wait_until(F f, int timeout_ms = 30000) {
  for (int t = 0; t < timeout_ms; t += 5) {
    if (f()) return true;
    std::this_thread::sleep_for(std::chrono::milliseconds(5));
  }
  return f();
}

static std::string key(int i) { char b[16]; snprintf(b, sizeof(b), "key%04d", i); return b; }
static std::string val(int i, int round) { return "v" + std::to_string(round) + "-" + std::to_string(i) + std::string(i % 7 * 40, 'x'); }
static bool live(int i, int round) { return round == 0 || i % 5 != 0; }

// the live keys an iterator walks forward from SeekToFirst, and whether every value is the one of `round`
static int walk_forward(rocksdb::Iterator* it, int round, bool* same) {
  int seen = 0;
  *same = true;
  for (it->SeekToFirst(); it->Valid(); it->Next()) {
    const int i = std::stoi(it->key().ToString().substr(3));
    *same = *same && live(i, round) && it->value().ToString() == val(i, round);
    seen++;
  }
  return seen;
}

static void test_bounded_iterators_on_a_follower() {
  auto& F = Flags();
  F.replicator_pull_delay_on_error_ms = 50;
  F.replicator_max_server_wait_time_ms = 200;
  F.replicator_client_server_timeout_difference_ms = 100;
  F.replicator_replication_mode = 0;
  F.replicator_timeout_ms = 2000;
  RocksDBReplicator leader_host(19161), follower_host(19162);
  admin::ApplicationDBManager lm(&leader_host), fm(&follower_host);
  std::string err;
  rocksdb::Options o;
  o.write_buffer_size = 1 << 20;
  rocksdb::DB *l = nullptr, *f = nullptr;
  EXPECT_TRUE(b200::GpuDB::Open(o, "bnd_leader", &l).ok());
  EXPECT_TRUE(b200::GpuDB::Open(o, "bnd_follower", &f).ok());
  EXPECT_TRUE(lm.addDB("seg00000", std::unique_ptr<rocksdb::DB>(l), ReplicaRole::LEADER, &err));
  EXPECT_TRUE(fm.addDB("seg00000", std::unique_ptr<rocksdb::DB>(f), ReplicaRole::FOLLOWER,
                       std::make_unique<SocketAddress>("127.0.0.1", 19161), &err));
  auto ldb = lm.getDB("seg00000", &err), fdb = fm.getDB("seg00000", &err);
  rocksdb::WriteOptions wo;
  const int n = 300, cut = 150;
  auto write_round = [&](int round) {
    for (int i = 0; i < n; i++) {
      WriteBatch b;
      if (!live(i, round)) b.Delete(key(i));
      else b.Put(key(i), val(i, round));
      EXPECT_TRUE(ldb->Write(wo, &b).ok());
    }
  };
  write_round(0);
  EXPECT_TRUE(wait_until([&] { return fdb->rocksdb()->GetLatestSequenceNumber() == (uint64_t)n; }));
  const rocksdb::Snapshot* snap = fdb->rocksdb()->GetSnapshot();
  const std::string bound_bytes = key(cut);
  const Slice bound(bound_bytes);
  rocksdb::ReadOptions latest, at;
  latest.iterate_upper_bound = &bound;
  at.iterate_upper_bound = &bound;
  at.snapshot = snap;
  for (int round = 1; round <= 3; round++) {
    // reads at the snapshot while the round is being replicated
    std::atomic<bool> done{false};
    std::thread writer([&] { write_round(round); done = true; });
    int reads = 0;
    while (!done || reads == 0) {
      std::unique_ptr<rocksdb::Iterator> it(fdb->NewIterator(at));
      bool same = false;
      EXPECT_TRUE(walk_forward(it.get(), 0, &same) == cut && same);
      it->SeekToLast();
      EXPECT_TRUE(it->Valid() && it->key().ToString() == key(cut - 1));
      it->SeekForPrev(key(cut));  // RocksDB 5.4: SeekForPrev does not apply the upper bound
      EXPECT_TRUE(it->Valid() && it->key().ToString() == key(cut) && it->value().ToString() == val(cut, 0));
      it->Next();
      EXPECT_TRUE(!it->Valid() && it->status().ok());
      reads++;
    }
    writer.join();
    EXPECT_TRUE(wait_until([&] { return fdb->rocksdb()->GetLatestSequenceNumber() == (uint64_t)n * (round + 1); }));
    if (round == 2) fdb->rocksdb()->CompactRange(rocksdb::CompactRangeOptions(), nullptr, nullptr);
    std::unique_ptr<rocksdb::Iterator> it(fdb->NewIterator(latest));
    bool same = false;
    EXPECT_TRUE(walk_forward(it.get(), round, &same) == cut - cut / 5 && same);
    it->SeekToLast();
    EXPECT_TRUE(it->Valid() && it->key().ToString() == key(cut - 1));
    it->SeekForPrev(key(cut));  // key(cut) is deleted: the key before it
    EXPECT_TRUE(it->Valid() && it->key().ToString() == key(cut - 1));
    it->SeekForPrev(key(cut + 1));
    EXPECT_TRUE(it->Valid() && it->key().ToString() == key(cut + 1) && it->value().ToString() == val(cut + 1, round));
    it->Seek(key(cut - 2));
    EXPECT_TRUE(it->Valid() && it->key().ToString() == key(cut - 2));
    it->Next();
    EXPECT_TRUE(it->Valid() && it->key().ToString() == key(cut - 1));
    it->Next();
    EXPECT_TRUE(!it->Valid() && it->status().ok());
    it->Seek(key(cut));
    EXPECT_TRUE(!it->Valid());
    // without a bound the same iterator reads on to the last key
    std::unique_ptr<rocksdb::Iterator> all(fdb->NewIterator(rocksdb::ReadOptions()));
    EXPECT_TRUE(walk_forward(all.get(), round, &same) == n - n / 5 && same);
  }
  fdb->rocksdb()->ReleaseSnapshot(snap);
  ldb.reset();  // removeDB waits until the manager holds the only reference
  fdb.reset();
  EXPECT_TRUE(lm.removeDB("seg00000", &err) != nullptr);
  EXPECT_TRUE(fm.removeDB("seg00000", &err) != nullptr);
}

int main() {
  printf("[ RUN  ] bounded_iterators_on_a_follower\n");
  test_bounded_iterators_on_a_follower();
  printf("%d checks, %d failures\n", g_checks, g_fail);
  return g_fail ? 1 : 0;
}
