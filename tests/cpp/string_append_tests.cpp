// string_append_tests.cpp — rocksdb::StringAppendOperator through the host mirror: GpuDB::Open maps it to the device
// operator (RSP_MERGE_STRING_APPEND, with its delimiter), and ApplicationDB's Write(Merge), Get, MultiGet, iterator and
// ReadOptions::snapshot reads, and a Backup / Restore whose SST holds the folded values, answer what the operator's
// own Merge gives.  Run by tests/test_string_append_host_gpu.py.
#include <cstdio>
#include <memory>
#include <string>
#include <vector>

#include <unistd.h>

#include "gpu_db.h"
#include "rocksdb/string_append_operator.h"
#include "rocksdb_admin/application_db_manager.h"
#include "rocksdb_replicator/rocksdb_replicator.h"

using namespace replicator;
using rocksdb::Slice;
using rocksdb::Status;
using rocksdb::WriteBatch;

static int g_checks = 0, g_fail = 0;
#define EXPECT_TRUE(c) do { g_checks++; if (!(c)) { g_fail++; printf("  FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); } } while (0)

// the operator's own rule, one operand at a time (AssociativeMergeOperator::Merge)
static std::string fold(const rocksdb::MergeOperator& op, const std::string* base, const std::vector<std::string>& ops) {
  std::string cur, nv;
  bool has = base != nullptr;
  if (has) cur = *base;
  for (const auto& o : ops) {
    Slice ex(cur);
    EXPECT_TRUE(op.Merge("k", has ? &ex : nullptr, o, &nv, nullptr));
    cur.swap(nv);
    has = true;
  }
  return cur;
}

// the shard runs the device operator: a host-form batched scan over merged keys answers every value with status 0 (a
// host-folded operator answers NotSupported there and hands back the keys alone)
static void expect_device_fold(rocksdb::DB* db, const std::string& key, const std::string& want) {
  auto* g = static_cast<b200::GpuDB*>(db);
  const uint32_t six = rsp_shard_index(g->shard());
  const uint64_t koff[2] = {0, key.size()};
  std::vector<uint8_t> out(4096);
  uint32_t n_out = 0;
  int32_t st = -1;
  EXPECT_TRUE(rsp_multi_scan(g->engine(), 1, &six, (const uint8_t*)key.data(), koff, 1, out.data(), out.size(), &n_out,
                             &st) == RSP_OK);
  EXPECT_TRUE(st == RSP_OK && n_out == 1);
  uint32_t kl = 0, vl = 0;
  memcpy(&kl, &out[0], 4);
  memcpy(&vl, &out[4], 4);
  EXPECT_TRUE(kl == key.size() && vl == want.size() && std::string((const char*)&out[8 + kl], vl) == want);
}

static void test_operator_and_factories() {
  auto comma = rocksdb::MergeOperators::CreateStringAppendOperator();
  auto nul = rocksdb::MergeOperators::CreateStringAppendOperator('\0');
  auto none = rocksdb::MergeOperators::CreateStringAppendOperatorWithoutDelimiter();
  EXPECT_TRUE(std::string(comma->Name()) == "StringAppendOperator");
  const std::string empty, base = "b";
  EXPECT_TRUE(fold(*comma, nullptr, {"x"}) == "x");
  EXPECT_TRUE(fold(*comma, &empty, {"x"}) == ",x");
  EXPECT_TRUE(fold(*comma, &base, {"x", "", "y"}) == "b,x,,y");
  EXPECT_TRUE(fold(*nul, &base, {"x"}) == std::string("b\0x", 3));
  EXPECT_TRUE(fold(*none, &base, {"x", "y"}) == "bxy");
}

static void test_application_db(std::shared_ptr<rocksdb::MergeOperator> op, const std::string& name, int port) {
  RocksDBReplicator host(port);
  admin::ApplicationDBManager m(&host);
  std::string err;
  rocksdb::Options o;
  o.write_buffer_size = 1 << 20;
  o.merge_operator = op;
  rocksdb::DB* raw = nullptr;
  EXPECT_TRUE(b200::GpuDB::Open(o, name, &raw).ok());
  rocksdb::DB* gdb = raw;
  EXPECT_TRUE(m.addDB(name, std::unique_ptr<rocksdb::DB>(raw), ReplicaRole::LEADER, &err));
  auto app = m.getDB(name, &err);
  rocksdb::WriteOptions wo;
  rocksdb::ReadOptions ro;
  const int n = 40, rounds = 6;
  std::vector<std::vector<std::string>> ops(n);
  std::vector<bool> has_base(n);
  const rocksdb::Snapshot* snap = nullptr;
  std::vector<std::string> at_snap(n);
  for (int r = 0; r < rounds; r++) {
    for (int i = 0; i < n; i++) {
      WriteBatch b;
      const std::string k = "key" + std::to_string(100 + i);
      if (r == 0 && i % 3 == 0) { b.Put(k, i % 2 ? "" : "base" + std::to_string(i)); has_base[i] = true; }
      const std::string o1 = "o" + std::to_string(r) + "." + std::to_string(i);
      b.Merge(k, o1);
      ops[i].push_back(o1);
      EXPECT_TRUE(app->Write(wo, &b).ok());
    }
    if (r == 1 || r == 3) EXPECT_TRUE(gdb->Flush(rocksdb::FlushOptions()).ok());
    if (r == 2) {
      snap = gdb->GetSnapshot();
      EXPECT_TRUE(snap != nullptr);
    }
    if (r <= 2)
      for (int i = 0; i < n; i++) {
        const std::string b = i % 2 ? "" : "base" + std::to_string(i);
        at_snap[i] = fold(*op, has_base[i] ? &b : nullptr, ops[i]);
      }
  }
  std::vector<std::string> want(n);
  std::vector<Slice> keys;
  std::vector<std::string> kstore(n);
  for (int i = 0; i < n; i++) {
    const std::string b = i % 2 ? "" : "base" + std::to_string(i);
    want[i] = fold(*op, has_base[i] ? &b : nullptr, ops[i]);
    kstore[i] = "key" + std::to_string(100 + i);
  }
  for (int i = 0; i < n; i++) keys.emplace_back(kstore[i]);
  for (int pass = 0; pass < 2; pass++) {  // pass 1: after a full compaction folded every chain into one Put
    std::string v;
    for (int i = 0; i < n; i++) EXPECT_TRUE(app->Get(ro, kstore[i], &v).ok() && v == want[i]);
    std::vector<std::string> vals;
    auto sts = app->MultiGet(ro, keys, &vals);
    for (int i = 0; i < n; i++) EXPECT_TRUE(sts[i].ok() && vals[i] == want[i]);
    std::unique_ptr<rocksdb::Iterator> it(app->NewIterator(ro));
    int i = 0;
    for (it->SeekToFirst(); it->Valid(); it->Next(), i++) EXPECT_TRUE(i < n && it->key() == kstore[i] && it->value() == want[i]);
    EXPECT_TRUE(i == n && it->status().ok());
    it.reset();
    rocksdb::ReadOptions at;
    at.snapshot = snap;
    for (int j = 0; j < n; j++) EXPECT_TRUE(app->Get(at, kstore[j], &v).ok() && v == at_snap[j]);
    std::unique_ptr<rocksdb::Iterator> sit(app->NewIterator(at));
    int j = n - 1;
    for (sit->SeekToLast(); sit->Valid(); sit->Prev(), j--) EXPECT_TRUE(j >= 0 && sit->value() == at_snap[j]);
    EXPECT_TRUE(j == -1);
    sit.reset();
    expect_device_fold(gdb, kstore[1], want[1]);
    if (pass == 0) EXPECT_TRUE(gdb->CompactRange(rocksdb::CompactRangeOptions(), nullptr, nullptr).ok());
  }
  gdb->ReleaseSnapshot(snap);
  // backup: the SST holds the folded values (one entry per key); the restored shard runs the device operator too
  const std::string root = "/tmp/rsp_sa_bk_" + std::to_string(getpid()) + "_" + name;
  uint64_t seq = 0, entries = 0;
  auto* g = static_cast<b200::GpuDB*>(gdb);
  EXPECT_TRUE(g->ExportSstFile(root + ".sst", &entries).ok() && entries == (uint64_t)n);
  EXPECT_TRUE(g->Backup(root, &seq).ok());
  rocksdb::DB* raw2 = nullptr;
  EXPECT_TRUE(b200::GpuDB::Restore(o, name + "_restored", root, &raw2).ok());
  std::unique_ptr<rocksdb::DB> dst(raw2);
  std::string v;
  for (int i = 0; i < n; i++) EXPECT_TRUE(dst->Get(ro, kstore[i], &v).ok() && v == want[i]);
  WriteBatch b;
  b.Merge(kstore[0], "tail");
  EXPECT_TRUE(dst->Write(wo, &b).ok());
  const std::string w0 = fold(*op, &want[0], {"tail"});
  EXPECT_TRUE(dst->Get(ro, kstore[0], &v).ok() && v == w0);
  expect_device_fold(dst.get(), kstore[0], w0);
  dst.reset();
  app.reset();
  m.removeDB(name, &err);
  remove((root + ".sst").c_str());
  std::string cmd = "rm -rf '" + root + "'";
  if (system(cmd.c_str()) != 0) printf("  (could not remove %s)\n", root.c_str());
}

int main() {
  printf("[ RUN  ] operator_and_factories\n");
  test_operator_and_factories();
  printf("[ RUN  ] application_db comma\n");
  test_application_db(rocksdb::MergeOperators::CreateStringAppendOperator(), "sa_comma00001", 19171);
  printf("[ RUN  ] application_db nul\n");
  test_application_db(rocksdb::MergeOperators::CreateStringAppendOperator('\0'), "sa_nul00001", 19172);
  printf("[ RUN  ] application_db none\n");
  test_application_db(rocksdb::MergeOperators::CreateStringAppendOperatorWithoutDelimiter(), "sa_none00001", 19173);
  printf("%d checks, %d failures\n", g_checks, g_fail);
  return g_fail ? 1 : 0;
}
