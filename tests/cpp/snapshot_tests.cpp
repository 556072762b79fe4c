// snapshot_tests.cpp — GpuDB / ApplicationDB reads with ReadOptions::snapshot: a snapshot taken on a follower keeps
// answering what it saw while later updates arrive through RocksDBReplicator.  Run by tests/test_snapshot_host_gpu.py.
#include <chrono>
#include <cstdio>
#include <memory>
#include <string>
#include <thread>
#include <vector>

#include <unistd.h>

#include "gpu_db.h"
#include "rocksdb_admin/application_db_manager.h"
#include "rocksdb_replicator/rocksdb_replicator.h"

using namespace replicator;
using rocksdb::Slice;
using rocksdb::Status;
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

static std::string val(int i, int round) { return "v" + std::to_string(round) + "-" + std::to_string(i) + std::string(i % 7 * 60, 'x'); }

// leader -> follower through RocksDBReplicator, reads on the follower's ApplicationDB at a snapshot
static void test_follower_snapshot_is_stable() {
  auto& F = Flags();
  F.replicator_pull_delay_on_error_ms = 50;
  F.replicator_max_server_wait_time_ms = 200;
  F.replicator_client_server_timeout_difference_ms = 100;
  F.replicator_replication_mode = 0;
  F.replicator_timeout_ms = 2000;
  RocksDBReplicator leader_host(19151), follower_host(19152);
  admin::ApplicationDBManager lm(&leader_host), fm(&follower_host);
  std::string err;
  rocksdb::Options o;
  o.write_buffer_size = 1 << 20;
  rocksdb::DB *l = nullptr, *f = nullptr;
  EXPECT_TRUE(b200::GpuDB::Open(o, "snap_leader", &l).ok());
  EXPECT_TRUE(b200::GpuDB::Open(o, "snap_follower", &f).ok());
  EXPECT_TRUE(lm.addDB("seg00000", std::unique_ptr<rocksdb::DB>(l), ReplicaRole::LEADER, &err));
  EXPECT_TRUE(fm.addDB("seg00000", std::unique_ptr<rocksdb::DB>(f), ReplicaRole::FOLLOWER,
                       std::make_unique<SocketAddress>("127.0.0.1", 19151), &err));
  auto ldb = lm.getDB("seg00000", &err), fdb = fm.getDB("seg00000", &err);
  rocksdb::WriteOptions wo;
  rocksdb::ReadOptions latest;
  const int n = 300;
  auto write_round = [&](int round) {
    for (int i = 0; i < n; i++) {
      WriteBatch b;
      if (round > 0 && i % 5 == 0) b.Delete("key" + std::to_string(i));
      else b.Put("key" + std::to_string(i), val(i, round));
      EXPECT_TRUE(ldb->Write(wo, &b).ok());
    }
  };
  write_round(0);
  EXPECT_TRUE(wait_until([&] { return fdb->rocksdb()->GetLatestSequenceNumber() == (uint64_t)n; }));
  const rocksdb::Snapshot* snap = fdb->rocksdb()->GetSnapshot();
  EXPECT_TRUE(snap != nullptr && snap->GetSequenceNumber() == (uint64_t)n);
  rocksdb::ReadOptions at;
  at.snapshot = snap;
  for (int round = 1; round <= 3; round++) {
    write_round(round);
    EXPECT_TRUE(wait_until([&] { return fdb->rocksdb()->GetLatestSequenceNumber() == (uint64_t)n * (round + 1); }));
    if (round == 2) fdb->rocksdb()->CompactRange(rocksdb::CompactRangeOptions(), nullptr, nullptr);
    std::vector<std::string> keys;
    for (int i = 0; i < n; i++) keys.push_back("key" + std::to_string(i));
    std::vector<Slice> ks(keys.begin(), keys.end());
    std::vector<std::string> vs;
    auto st = fdb->MultiGet(at, ks, &vs);
    bool all = st.size() == (size_t)n;
    for (int i = 0; all && i < n; i++) all = st[i].ok() && vs[i] == val(i, 0);
    EXPECT_TRUE(all);
    for (int i = 0; i < n; i += 17) {
      std::string v;
      EXPECT_TRUE(fdb->Get(at, keys[i], &v).ok() && v == val(i, 0));
      Status s = fdb->Get(latest, keys[i], &v);
      EXPECT_TRUE(i % 5 == 0 ? s.IsNotFound() : (s.ok() && v == val(i, round)));
    }
    std::unique_ptr<rocksdb::Iterator> it(fdb->NewIterator(at));
    int seen = 0;
    bool same = true;
    for (it->SeekToFirst(); it->Valid(); it->Next()) {
      const int i = std::stoi(it->key().ToString().substr(3));
      same = same && it->value().ToString() == val(i, 0);
      seen++;
    }
    EXPECT_TRUE(same && seen == n);
  }
  fdb->rocksdb()->ReleaseSnapshot(snap);
  ldb.reset();  // removeDB waits until the manager holds the only reference
  fdb.reset();
  EXPECT_TRUE(lm.removeDB("seg00000", &err) != nullptr);
  EXPECT_TRUE(fm.removeDB("seg00000", &err) != nullptr);
}

// IngestExternalFile with snapshot_consistency = false while a snapshot is live: the engine cannot hide the file from
// snapshots taken before it, so the call answers NotSupported; with the default the file takes a global sequence number
static void test_ingest_while_snapshot_is_live() {
  rocksdb::Options o;
  rocksdb::DB *a = nullptr, *src = nullptr;
  EXPECT_TRUE(b200::GpuDB::Open(o, "snap_ingest", &a).ok());
  EXPECT_TRUE(b200::GpuDB::Open(o, "snap_ingest_src", &src).ok());
  std::unique_ptr<rocksdb::DB> ga(a), gs(src);
  rocksdb::WriteOptions wo;
  EXPECT_TRUE(a->Put(wo, "a", "1").ok());
  EXPECT_TRUE(src->Put(wo, "z", "2").ok());
  const std::string path = "/tmp/snapshot_tests_" + std::to_string(getpid()) + ".sst";
  EXPECT_TRUE(static_cast<b200::GpuDB*>(src)->ExportSstFile(path).ok());
  const rocksdb::Snapshot* snap = a->GetSnapshot();
  rocksdb::IngestExternalFileOptions io;
  io.snapshot_consistency = false;
  EXPECT_TRUE(a->IngestExternalFile({path}, io).IsNotSupported());
  io.snapshot_consistency = true;
  EXPECT_TRUE(a->IngestExternalFile({path}, io).ok());
  EXPECT_TRUE(a->GetLatestSequenceNumber() == 2);
  std::string v;
  rocksdb::ReadOptions at;
  at.snapshot = snap;
  EXPECT_TRUE(a->Get(at, "z", &v).IsNotFound());
  EXPECT_TRUE(a->Get(rocksdb::ReadOptions(), "z", &v).ok() && v == "2");
  a->ReleaseSnapshot(snap);
  remove(path.c_str());
}

int main() {
  printf("[ RUN  ] follower_snapshot_is_stable\n");
  test_follower_snapshot_is_stable();
  printf("[ RUN  ] ingest_while_snapshot_is_live\n");
  test_ingest_while_snapshot_is_live();
  printf("%d checks, %d failures\n", g_checks, g_fail);
  return g_fail ? 1 : 0;
}
