// ingest_behind_tests.cpp — RocksDB 5.7's ingest behind through the host mirror, step for step as the reference's
// rocksdb_admin/tests/application_db_test.cpp:300-342 does it: ApplicationDB over GpuDB, the level an ingested-behind
// file occupies (getHighestEmptyLevel / DBLmaxEmpty), CompactRange with and without change_level.  Then what the admin
// handler reads (GetDBOptions().allow_ingest_behind) and the reads of data ingested behind existing writes.  Run by
// tests/test_ingest_behind_host_gpu.py.
#include <cstdio>
#include <memory>
#include <string>
#include <vector>

#include "gpu_db.h"
#include "rocksdb_admin/application_db_manager.h"
#include "rocksdb_replicator/rocksdb_replicator.h"
#include "sst/sst_format.h"

using namespace replicator;
using rocksdb::Status;

static int g_checks = 0, g_fail = 0;
#define EXPECT_TRUE(c) do { g_checks++; if (!(c)) { g_fail++; printf("  FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); } } while (0)
#define EXPECT_FALSE(c) EXPECT_TRUE(!(c))
#define EXPECT_EQ(a, b) EXPECT_TRUE((a) == (b))

static std::string write_sst(const std::string& path, const std::vector<std::pair<std::string, std::string>>& kv) {
  std::string bytes, err;
  EXPECT_TRUE(sst::WriteSst(kv, &bytes, &err));
  FILE* f = fopen(path.c_str(), "wb");
  EXPECT_TRUE(f != nullptr);
  if (f) { fwrite(bytes.data(), 1, bytes.size(), f); fclose(f); }
  return path;
}

// ApplicationDB::getHighestEmptyLevel, through its public property (the reference's test is a friend of the class)
static unsigned highest_empty(admin::ApplicationDB* app) {
  std::string v;
  EXPECT_TRUE(app->GetProperty(admin::ApplicationDB::Properties::kHighestEmptyLevel, &v));
  return v.empty() ? 999u : (unsigned)std::stoul(v);
}

struct Opened {
  std::shared_ptr<admin::ApplicationDB> app;
  rocksdb::DB* db = nullptr;
};
static Opened open_db(admin::ApplicationDBManager* m, const std::string& name, const rocksdb::Options& o) {
  Opened r;
  std::string err;
  rocksdb::DB* raw = nullptr;
  EXPECT_TRUE(b200::GpuDB::Open(o, name, &raw).ok());
  r.db = raw;
  EXPECT_TRUE(m->addDB(name, std::unique_ptr<rocksdb::DB>(raw), ReplicaRole::LEADER, &err));
  r.app = m->getDB(name, &err);
  EXPECT_TRUE(r.app != nullptr);
  return r;
}

static void test_application_db_ingest_behind(const std::string& dir) {
  RocksDBReplicator host(19181);
  admin::ApplicationDBManager m(&host);
  std::string err;
  rocksdb::Options opts;
  opts.write_buffer_size = 1 << 20;
  Opened d = open_db(&m, "ib00001", opts);
  // DB level = 7 at create; levels 0 .. 6, all empty
  EXPECT_EQ(d.db->NumberLevels(), 7);
  EXPECT_EQ(highest_empty(d.app.get()), 6u);

  const std::string sst_file1 = dir + "/ib_file1.sst";
  write_sst(sst_file1, {{"1", "1"}, {"2", "2"}});
  rocksdb::IngestExternalFileOptions ifo;
  ifo.move_files = true;
  ifo.allow_global_seqno = true;
  ifo.ingest_behind = true;
  EXPECT_FALSE(d.db->GetOptions().allow_ingest_behind);
  EXPECT_FALSE(d.db->GetDBOptions().allow_ingest_behind);
  Status s = d.db->IngestExternalFile({sst_file1}, ifo);
  EXPECT_FALSE(s.ok());
  EXPECT_TRUE(s.IsInvalidArgument());
  EXPECT_TRUE(s.ToString().find("can't ingest_behind file in DB with allow_ingest_behind=false") != std::string::npos);
  EXPECT_EQ(highest_empty(d.app.get()), 6u);

  // DestroyAndReopen with allow_ingest_behind
  d.app.reset();
  EXPECT_TRUE(m.removeDB("ib00001", &err) != nullptr);
  rocksdb::Options behind = opts;
  behind.allow_ingest_behind = true;
  d = open_db(&m, "ib00001", behind);
  EXPECT_TRUE(d.db->GetOptions().allow_ingest_behind);
  EXPECT_TRUE(d.db->GetDBOptions().allow_ingest_behind);
  write_sst(sst_file1, {{"1", "1"}, {"2", "2"}});
  s = d.db->IngestExternalFile({sst_file1}, ifo);
  EXPECT_TRUE(s.ok());
  // level 6 is occupied by the ingested data
  EXPECT_EQ(highest_empty(d.app.get()), 5u);
  EXPECT_FALSE(d.app->DBLmaxEmpty());

  rocksdb::CompactRangeOptions co;
  co.change_level = false;  // the default: the bottom level stays where it is
  EXPECT_TRUE(d.db->CompactRange(co, nullptr, nullptr).ok());
  EXPECT_EQ(highest_empty(d.app.get()), 5u);

  co.change_level = true;
  EXPECT_TRUE(d.db->CompactRange(co, nullptr, nullptr).ok());
  EXPECT_EQ(highest_empty(d.app.get()), 6u);
  EXPECT_TRUE(d.app->DBLmaxEmpty());
  std::string v;
  EXPECT_TRUE(d.app->Get(rocksdb::ReadOptions(), "1", &v).ok() && v == "1");
  d.app.reset();
  EXPECT_TRUE(m.removeDB("ib00001", &err) != nullptr);
}

// a backfill below existing writes: every write shadows the file, deletes hide it, the sequence number stays
static void test_backfill_below_writes(const std::string& dir) {
  RocksDBReplicator host(19182);
  admin::ApplicationDBManager m(&host);
  std::string err;
  rocksdb::Options o;
  o.write_buffer_size = 1 << 20;
  o.allow_ingest_behind = true;
  Opened d = open_db(&m, "ib00002", o);
  rocksdb::WriteOptions wo;
  rocksdb::WriteBatch b;
  b.Put("a", "new-a");
  b.Delete("b");
  EXPECT_TRUE(d.app->Write(wo, &b).ok());
  EXPECT_TRUE(d.db->Flush(rocksdb::FlushOptions()).ok());
  EXPECT_TRUE(d.db->CompactRange(rocksdb::CompactRangeOptions(), nullptr, nullptr).ok());  // the tombstone stays
  const uint64_t seq = d.db->GetLatestSequenceNumber();
  rocksdb::IngestExternalFileOptions ifo;
  ifo.ingest_behind = true;
  ifo.allow_global_seqno = false;  // plays no part behind
  EXPECT_TRUE(d.db->IngestExternalFile({write_sst(dir + "/ib_file2.sst", {{"a", "old-a"}, {"b", "old-b"}, {"c", "old-c"}})}, ifo).ok());
  EXPECT_EQ(d.db->GetLatestSequenceNumber(), seq);
  std::string v;
  EXPECT_TRUE(d.app->Get(rocksdb::ReadOptions(), "a", &v).ok() && v == "new-a");
  EXPECT_TRUE(d.app->Get(rocksdb::ReadOptions(), "b", &v).IsNotFound());
  EXPECT_TRUE(d.app->Get(rocksdb::ReadOptions(), "c", &v).ok() && v == "old-c");
  // overlapping the file already behind: refused, nothing changes
  Status s = d.db->IngestExternalFile({write_sst(dir + "/ib_file3.sst", {{"b", "x"}})}, ifo);
  EXPECT_TRUE(s.IsInvalidArgument() && s.ToString().find("doesn't fit at the bottommost level") != std::string::npos);
  EXPECT_TRUE(d.app->Get(rocksdb::ReadOptions(), "c", &v).ok() && v == "old-c");
  EXPECT_FALSE(d.app->DBLmaxEmpty());
  d.app.reset();
  EXPECT_TRUE(m.removeDB("ib00002", &err) != nullptr);
}

int main(int argc, char** argv) {
  const std::string dir = argc > 1 ? argv[1] : "/tmp";
  printf("[ RUN  ] application_db ingest_behind\n");
  test_application_db_ingest_behind(dir);
  printf("[ RUN  ] backfill below writes\n");
  test_backfill_below_writes(dir);
  printf("%d checks, %d failures\n", g_checks, g_fail);
  return g_fail ? 1 : 0;
}
