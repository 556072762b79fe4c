// gpu_db.cpp — see gpu_db.h.  Call sites replaced: rocksdb_replicator/rocksdb_wrapper.cpp:4-28,
// rocksdb_admin/application_db.cpp:78-144.
#include "gpu_db.h"

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <map>

#include "rocksdb/string_append_operator.h"
#include "sst/sst_format.h"

namespace b200 {

using rocksdb::Slice;
using rocksdb::Status;

std::shared_ptr<GpuEngine> GpuEngine::ForDevice(int device) {
  static std::mutex mu;
  static std::map<int, std::weak_ptr<GpuEngine>> engines;
  std::lock_guard<std::mutex> g(mu);
  if (auto e = engines[device].lock()) return e;
  rsp_engine* raw = nullptr;
  rsp_engine_cfg cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.abi_version = RSP_ABI_VERSION;
  if (rsp_engine_create(device, &cfg, &raw) != RSP_OK) return nullptr;
  std::shared_ptr<GpuEngine> e(new GpuEngine(raw));
  engines[device] = e;
  return e;
}
GpuEngine::~GpuEngine() { rsp_engine_destroy(e_); }

int GpuDB::MergeTrampoline(void* state, const uint8_t* key, size_t klen, const uint8_t* existing, size_t elen,
                           const uint8_t* operand, size_t olen, void (*out_set)(void*, const uint8_t*, size_t),
                           void* out_ctx) {
  auto* op = static_cast<rocksdb::MergeOperator*>(state);
  Slice ex((const char*)existing, elen);
  std::string nv;
  if (!op->Merge(Slice((const char*)key, klen), existing ? &ex : nullptr, Slice((const char*)operand, olen), &nv, nullptr))
    return 0;
  out_set(out_ctx, (const uint8_t*)nv.data(), nv.size());
  return 1;
}

Status GpuDB::Open(const rocksdb::Options& options, const std::string& name, rocksdb::DB** dbptr, int device) {
  *dbptr = nullptr;
  auto engine = GpuEngine::ForDevice(device);
  if (!engine) return Status::IOError("no usable CUDA device for the GPU engine (there is no CPU fallback)");
  rsp_shard_opts so;
  memset(&so, 0, sizeof(so));
  so.write_buffer_bytes = options.write_buffer_size;
  if (options.merge_operator) {
    const std::string n = options.merge_operator->Name();
    // operators whose semantics the device implements exactly; anything else folds on the host through the callback
    // (the string-append operator by its type: its delimiter travels with it)
    const auto* sa = dynamic_cast<const rocksdb::StringAppendOperator*>(options.merge_operator.get());
    if (sa) { so.merge_op = RSP_MERGE_STRING_APPEND; so.merge_delim = sa->has_delim() ? 0x100u | (uint8_t)sa->delim() : 0u; }
    else if (n == "CounterMergeOperator") so.merge_op = RSP_MERGE_COUNTER;   // examples/counter_service/merge_operator.cpp
    else if (n == "UInt64AddOperator") so.merge_op = RSP_MERGE_UINT64ADD;    // RocksDB built-in
    else { so.merge_op = RSP_MERGE_CALLBACK; so.merge_fn = &GpuDB::MergeTrampoline; so.merge_state = options.merge_operator.get(); }
  }
  rsp_shard* sh = nullptr;
  const int rc = rsp_shard_open_ex(engine->raw(), name.c_str(), &so,
                                   options.allow_ingest_behind ? RSP_SHARD_ALLOW_INGEST_BEHIND : 0u, &sh);
  if (rc != RSP_OK) return rc == RSP_INVALID_ARGUMENT ? Status::InvalidArgument("db already open: " + name) : Status::IOError("rsp_shard_open");
  GpuDB* db = new GpuDB();
  db->name_ = name;
  db->options_ = options;
  db->engine_ = engine;
  db->shard_ = sh;
  *dbptr = db;
  return Status::OK();
}

GpuDB::~GpuDB() {
  if (shard_) rsp_shard_close(shard_);
}

Status GpuDB::ToStatus(int code) const {
  if (code == RSP_OK) return Status::OK();
  char buf[256];
  buf[0] = 0;
  rsp_last_error(shard_, buf, sizeof(buf));
  return Status::FromCode(code, buf);
}

void GpuDB::LogPush(std::shared_ptr<const LogChunk> c) {
  log_bytes_ += c->bytes.size();
  log_.push_back(std::move(c));
  while (log_bytes_ > log_cap_bytes_ && log_.size() > 1) {  // WAL TTL / size limit stand-in
    log_bytes_ -= log_.front()->bytes.size();
    log_.pop_front();
    log_base_id_++;
  }
}
void GpuDB::LogAppend(rocksdb::SequenceNumber first_seq, std::string&& bytes, uint32_t count) {
  auto c = std::make_shared<LogChunk>();
  c->first_seq = first_seq;
  c->last_seq = first_seq + count - 1;
  c->bytes = std::move(bytes);
  c->recs.push_back(LogChunk::Rec{0u, (uint32_t)c->bytes.size(), count, first_seq});
  std::lock_guard<std::mutex> g(log_mu_);
  LogPush(std::move(c));
}

Status GpuDB::Write(const rocksdb::WriteOptions&, rocksdb::WriteBatch* updates) {
  std::lock_guard<std::mutex> g(write_mu_);
  uint64_t seq = 0;
  const std::string& rep = updates->Data();
  const int rc = rsp_write(shard_, (const uint8_t*)rep.data(), rep.size(), &seq);
  if (rc != RSP_OK) return ToStatus(rc);
  const uint32_t count = (uint32_t)updates->Count();
  if (count) {
    std::string bytes = rep;
    const uint64_t first = seq - count + 1;
    memcpy(&bytes[0], &first, 8);  // DB::Write stamps the batch's sequence in place
    updates->SetSequence(first);
    LogAppend(first, std::move(bytes), count);
  }
  return Status::OK();
}

std::vector<Status> GpuDB::WriteMany(const rocksdb::WriteOptions&, const std::vector<rocksdb::WriteBatch*>& updates) {
  const size_t n = updates.size();
  std::vector<Status> out(n);
  if (!n) return out;
  std::lock_guard<std::mutex> g(write_mu_);  // log order == sequence order
  std::vector<rsp_slice> slices(n);
  for (size_t i = 0; i < n; i++) slices[i] = rsp_slice{(const uint8_t*)updates[i]->Data().data(), updates[i]->Data().size()};
  const uint64_t seq_before = GetLatestSequenceNumber();
  size_t n_applied = 0;
  const int rc = rsp_apply_updates(shard_, n, slices.data(), nullptr, nullptr, nullptr, &n_applied);
  // applied in order until the first failure (which latches the shard, as a failed DB::Write does in RocksDB 5.x)
  uint64_t first = seq_before + 1;
  for (size_t i = 0; i < n; i++) {
    if (i >= n_applied) { out[i] = ToStatus(rc != RSP_OK ? rc : RSP_IO_ERROR); continue; }
    const uint32_t count = (uint32_t)updates[i]->Count();
    if (!count) continue;
    std::string bytes = updates[i]->Data();
    memcpy(&bytes[0], &first, 8);
    updates[i]->SetSequence(first);
    LogAppend(first, std::move(bytes), count);
    first += count;
  }
  return out;
}

namespace {
bool ReadWholeFile(const std::string& path, std::string* out) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return false;
  char buf[1 << 16];
  size_t n;
  out->clear();
  while ((n = fread(buf, 1, sizeof(buf), f)) > 0) out->append(buf, n);
  fclose(f);
  return true;
}
}  // namespace

namespace {
class GpuSnapshot : public rocksdb::Snapshot {
 public:
  explicit GpuSnapshot(rsp_snapshot* s) : s_(s) {}
  ~GpuSnapshot() override {}
  rocksdb::SequenceNumber GetSequenceNumber() const override { return rsp_snapshot_seq(s_); }
  rsp_snapshot* raw() const { return s_; }

 private:
  rsp_snapshot* s_;
};
rsp_snapshot* RawSnapshot(const rocksdb::Snapshot* s) { return static_cast<const GpuSnapshot*>(s)->raw(); }
}  // namespace

const rocksdb::Snapshot* GpuDB::GetSnapshot() {
  rsp_snapshot* s = nullptr;
  if (rsp_snapshot_create(shard_, &s) != RSP_OK) return nullptr;
  n_snapshots_++;
  return new GpuSnapshot(s);
}

void GpuDB::ReleaseSnapshot(const rocksdb::Snapshot* snapshot) {
  if (!snapshot) return;
  rsp_snapshot_release(RawSnapshot(snapshot));
  n_snapshots_--;
  delete static_cast<const GpuSnapshot*>(snapshot);
}

Status GpuDB::IngestExternalFile(const std::vector<std::string>& files, const rocksdb::IngestExternalFileOptions& opt) {
  if (files.empty()) return Status::InvalidArgument("external_files is empty");
  // the engine cannot show a file to snapshots taken before it: with snapshots live, the file is always newer
  if (!opt.snapshot_consistency && n_snapshots_.load() > 0)
    return Status::NotSupported("IngestExternalFile without snapshot_consistency while snapshots are live");
  struct Parsed { std::vector<sst::Entry> entries; };
  std::vector<Parsed> parsed(files.size());
  for (size_t i = 0; i < files.size(); i++) {
    std::string bytes, err;
    if (!ReadWholeFile(files[i], &bytes)) return Status::IOError("While opening a file for sequentially reading: " + files[i]);
    sst::Props props;
    if (!sst::ReadSst(bytes, &parsed[i].entries, &props, &err)) return Status::Corruption(err);
    if (props.external_version == 0) return Status::InvalidArgument("External file version not found");
    if (parsed[i].entries.empty()) return Status::InvalidArgument("Can't ingest empty file: " + files[i]);
    for (const auto& e : parsed[i].entries) {
      if (e.type != 1) return Status::NotSupported("external file holds a record that is not a Put");
      if (e.seq != 0) return Status::Corruption("external file have non zero sequence number");
    }
  }
  // several files: their ranges must be disjoint; together they are one sorted run with one sequence number
  std::sort(parsed.begin(), parsed.end(),
            [](const Parsed& a, const Parsed& b) { return a.entries.front().user_key < b.entries.front().user_key; });
  for (size_t i = 1; i < parsed.size(); i++)
    if (!(parsed[i - 1].entries.back().user_key < parsed[i].entries.front().user_key))
      return Status::NotSupported("Files have overlapping ranges");
  std::string keys, vals;
  std::vector<uint64_t> koff(1, 0), voff(1, 0);
  for (const auto& p : parsed)
    for (const auto& e : p.entries) {
      keys += e.user_key;
      vals += e.value;
      koff.push_back(keys.size());
      voff.push_back(vals.size());
    }
  keys.push_back('\0');
  vals.push_back('\0');
  std::lock_guard<std::mutex> g(write_mu_);
  // ingest_behind: the file goes to the shard's ingested-behind tier; allow_global_seqno plays no part
  const int rc = opt.ingest_behind
      ? rsp_ingest_sorted_behind(shard_, koff.size() - 1, (const uint8_t*)keys.data(), koff.data(), (const uint8_t*)vals.data(),
                                 voff.data())
      : rsp_ingest_sorted(shard_, koff.size() - 1, (const uint8_t*)keys.data(), koff.data(), (const uint8_t*)vals.data(),
                          voff.data(), opt.allow_global_seqno ? 1 : 0, nullptr);
  if (rc != RSP_OK) return ToStatus(rc);
  if (opt.move_files)
    for (const auto& f : files) remove(f.c_str());  // the data now lives in HBM; a moved file is gone from its old place
  return Status::OK();
}

Status GpuDB::ExportSstFile(const std::string& path, uint64_t* entries) {
  std::vector<std::pair<std::string, std::string>> kv;
  {
    std::unique_ptr<rocksdb::Iterator> it(NewIterator(rocksdb::ReadOptions()));
    for (it->SeekToFirst(); it->Valid(); it->Next()) kv.emplace_back(it->key().ToString(), it->value().ToString());
    if (!it->status().ok()) return it->status();
  }
  if (kv.empty()) return Status::InvalidArgument("nothing to export: " + name_);
  std::string file, err;
  if (!sst::WriteSst(kv, &file, &err)) return Status::InvalidArgument(err);
  FILE* f = fopen(path.c_str(), "wb");
  if (!f) return Status::IOError("While open a file for appending: " + path);
  const size_t w = fwrite(file.data(), 1, file.size(), f);
  if (fclose(f) != 0 || w != file.size()) return Status::IOError("While appending to file: " + path);
  if (entries) *entries = kv.size();
  return Status::OK();
}

Status GpuDB::Backup(const std::string& dir, uint64_t* seq_out) {
  // contents and sequence number must belong together: writers are held off for the export
  std::lock_guard<std::mutex> g(write_mu_);
  const uint64_t seq = GetLatestSequenceNumber();
  const std::string mk = "mkdir -p '" + dir + "'";
  if (system(mk.c_str()) != 0) return Status::IOError("cannot create " + dir);
  uint64_t entries = 0;
  const std::string tmp_sst = dir + "/data.sst.tmp", tmp_meta = dir + "/dbmeta.tmp";
  Status st = ExportSstFile(tmp_sst, &entries);
  const bool empty = !st.ok() && st.IsInvalidArgument();  // "nothing to export": an empty shard is a valid backup
  if (!st.ok() && !empty) return st;
  if (empty) remove(tmp_sst.c_str());
  FILE* f = fopen(tmp_meta.c_str(), "wb");
  if (!f) return Status::IOError("While open a file for appending: " + tmp_meta);
  fprintf(f, "db_name=%s\nseq_no=%llu\nentries=%llu\nfile=%s\n", name_.c_str(), (unsigned long long)seq,
          (unsigned long long)entries, empty ? "" : "data.sst");
  if (fclose(f) != 0) return Status::IOError("While appending to file: " + tmp_meta);
  if (!empty && rename(tmp_sst.c_str(), (dir + "/data.sst").c_str()) != 0) return Status::IOError("rename " + tmp_sst);
  if (empty) remove((dir + "/data.sst").c_str());
  if (rename(tmp_meta.c_str(), (dir + "/dbmeta").c_str()) != 0) return Status::IOError("rename " + tmp_meta);
  if (seq_out) *seq_out = seq;
  return Status::OK();
}

Status GpuDB::Restore(const rocksdb::Options& options, const std::string& name, const std::string& dir, rocksdb::DB** dbptr,
                      int device) {
  *dbptr = nullptr;
  std::string meta;
  if (!ReadWholeFile(dir + "/dbmeta", &meta)) return Status::IOError("While opening a file for sequentially reading: " + dir + "/dbmeta");
  auto field = [&](const std::string& key) {
    const size_t at = meta.find(key + "=");
    if (at == std::string::npos) return std::string();
    const size_t end = meta.find('\n', at);
    return meta.substr(at + key.size() + 1, end == std::string::npos ? std::string::npos : end - at - key.size() - 1);
  };
  if (field("seq_no").empty()) return Status::Corruption("dbmeta without seq_no in " + dir);
  const uint64_t seq = strtoull(field("seq_no").c_str(), nullptr, 10);
  rocksdb::DB* raw = nullptr;
  Status st = Open(options, name, &raw, device);
  if (!st.ok()) return st;
  std::unique_ptr<rocksdb::DB> db(raw);
  auto* gdb = static_cast<GpuDB*>(raw);
  if (!field("file").empty()) {
    rocksdb::IngestExternalFileOptions io;
    io.move_files = false;
    st = gdb->IngestExternalFile({dir + "/" + field("file")}, io);
    if (!st.ok()) return st;
  }
  const int rc = rsp_set_latest_seq(gdb->shard_, seq);
  if (rc != RSP_OK) return gdb->ToStatus(rc);
  *dbptr = db.release();
  return Status::OK();
}

BackupScheduler::BackupScheduler(const std::string& root, uint64_t period_ms) : root_(root), period_ms_(period_ms) {
  th_ = std::thread([this] {
    std::unique_lock<std::mutex> l(mu_);
    while (!stop_) {
      cv_.wait_for(l, std::chrono::milliseconds(period_ms_));
      if (stop_) break;
      l.unlock();
      RunOnce();
      l.lock();
    }
  });
}
BackupScheduler::~BackupScheduler() {
  {
    std::lock_guard<std::mutex> g(mu_);
    stop_ = true;
  }
  cv_.notify_all();
  th_.join();
}
void BackupScheduler::Add(const std::string& name, std::shared_ptr<rocksdb::DB> db) {
  std::lock_guard<std::mutex> g(mu_);
  items_[name].db = std::move(db);
}
void BackupScheduler::Remove(const std::string& name) {
  std::lock_guard<std::mutex> g(mu_);
  items_.erase(name);
}
size_t BackupScheduler::RunOnce() {
  std::vector<std::pair<std::string, Item>> todo;
  {
    std::lock_guard<std::mutex> g(mu_);
    for (auto& kv : items_)
      if (kv.second.db->GetLatestSequenceNumber() != kv.second.last_seq) todo.push_back(kv);
  }
  size_t n = 0;
  for (auto& kv : todo) {
    auto* gdb = dynamic_cast<GpuDB*>(kv.second.db.get());
    if (!gdb) continue;
    uint64_t seq = 0;
    if (!gdb->Backup(root_ + "/" + kv.first, &seq).ok()) continue;
    n++;
    done_++;
    std::lock_guard<std::mutex> g(mu_);
    auto it = items_.find(kv.first);
    if (it != items_.end()) it->second.last_seq = seq;
  }
  return n;
}

Status GpuDB::ApplyReplicated(const Slice& raw, uint64_t ts) {
  std::lock_guard<std::mutex> g(write_mu_);
  uint64_t seq = 0;
  const int rc = rsp_apply(shard_, (const uint8_t*)raw.data(), raw.size(), ts, &seq);
  if (rc != RSP_OK) return ToStatus(rc);
  if (raw.size() >= rocksdb::WriteBatch::kHeader) {
    uint32_t count;
    memcpy(&count, raw.data() + 8, 4);
    if (count) {  // what the follower's own WAL would hold: the batch + its LogData(timestamp)
      std::string bytes(raw.data(), raw.size());
      bytes.push_back(0x3);
      bytes.push_back(8);
      bytes.append((const char*)&ts, 8);
      const uint64_t first = seq - count + 1;
      memcpy(&bytes[0], &first, 8);
      LogAppend(first, std::move(bytes), count);
    }
  }
  return Status::OK();
}

void GpuDB::ApplyReplicatedBatch(const std::vector<replicator::Update>& updates,
                                 std::function<void(size_t, const rocksdb::Status&)> done) {
  const size_t n = updates.size();
  if (!n) return done(0, Status::OK());
  struct Ctx {
    GpuDB* db;
    const std::vector<replicator::Update>* updates;
    std::function<void(size_t, const rocksdb::Status&)> done;
    uint64_t seq_before;
  };
  std::vector<rsp_slice> slices(n);
  std::vector<uint64_t> ts(n);
  for (size_t i = 0; i < n; i++) {
    slices[i] = rsp_slice{(const uint8_t*)updates[i].raw_data.data(), updates[i].raw_data.size()};
    ts[i] = (uint64_t)updates[i].timestamp;
  }
  // one response at a time per shard (the pull loop is serial per shard): the sequence number before the call is the
  // base of this response's batches in the update log
  Ctx* ctx = new Ctx{this, &updates, std::move(done), GetLatestSequenceNumber()};
  const int rc = rsp_apply_updates(
      shard_, n, slices.data(), ts.data(),
      [](void* c, int status, size_t n_applied, uint64_t) {
        std::unique_ptr<Ctx> x(static_cast<Ctx*>(c));
        uint64_t first = x->seq_before + 1;
        {
          // what the follower's own WAL would hold (its downstream followers pull it): every applied batch + its
          // LogData(timestamp), stamped with its sequence number; built outside the log's lock, appended in one go
          auto chunk = std::make_shared<LogChunk>();
          size_t total = 0;
          for (size_t i = 0; i < n_applied; i++) total += (*x->updates)[i].raw_data.size() + 10;
          chunk->bytes.reserve(total);
          chunk->recs.reserve(n_applied);
          chunk->first_seq = first;
          for (size_t i = 0; i < n_applied; i++) {
            const std::string& raw = (*x->updates)[i].raw_data;
            if (raw.size() < rocksdb::WriteBatch::kHeader) continue;
            uint32_t count;
            memcpy(&count, raw.data() + 8, 4);
            if (!count) continue;
            const uint64_t tsv = (uint64_t)(*x->updates)[i].timestamp;
            const size_t at = chunk->bytes.size();
            chunk->bytes.append(raw.data(), raw.size());
            chunk->bytes.push_back(0x3);
            chunk->bytes.push_back(8);
            chunk->bytes.append((const char*)&tsv, 8);
            memcpy(&chunk->bytes[at], &first, 8);
            chunk->recs.push_back(LogChunk::Rec{(uint32_t)at, (uint32_t)(chunk->bytes.size() - at), count, first});
            first += count;
          }
          chunk->last_seq = first - 1;
          if (!chunk->recs.empty()) {
            std::lock_guard<std::mutex> g(x->db->write_mu_);
            std::lock_guard<std::mutex> g2(x->db->log_mu_);
            x->db->LogPush(std::move(chunk));
          }
        }
        x->done(n_applied, status == RSP_OK ? Status::OK() : x->db->ToStatus(status));
      },
      ctx, nullptr);
  if (rc != RSP_OK) {
    std::unique_ptr<Ctx> x(ctx);
    x->done(0, ToStatus(rc));
  }
}

Status GpuDB::Get(const rocksdb::ReadOptions& o, const Slice& key, std::string* value) {
  size_t cap = 256, n = 0;
  for (;;) {
    value->resize(cap);
    const int rc = o.snapshot ? rsp_get_at(RawSnapshot(o.snapshot), (const uint8_t*)key.data(), key.size(), (uint8_t*)&(*value)[0], cap, &n)
                              : rsp_get(shard_, (const uint8_t*)key.data(), key.size(), (uint8_t*)&(*value)[0], cap, &n);
    if (rc == RSP_INCOMPLETE) { cap = n; continue; }
    if (rc != RSP_OK) { value->clear(); return rc == RSP_NOT_FOUND ? Status::NotFound() : ToStatus(rc); }
    value->resize(n);
    return Status::OK();
  }
}

Status GpuDB::Get(const rocksdb::ReadOptions& o, rocksdb::ColumnFamilyHandle*, const Slice& key, rocksdb::PinnableSlice* value) {
  Status s = Get(o, key, value->GetSelf());
  if (s.ok()) value->PinSelf();
  return s;
}

// MultiGet at a snapshot (rsp_multi_get_at): values larger than the stride come back Incomplete with their size, and
// the call is repeated with a stride that fits them
std::vector<Status> GpuDB::MultiGetAt(const rocksdb::Snapshot* snapshot, const std::vector<Slice>& keys,
                                      std::vector<std::string>* values) {
  const size_t n = keys.size();
  std::vector<Status> out(n);
  values->assign(n, std::string());
  if (!n) return out;
  std::string blob;
  std::vector<uint64_t> koff(n + 1, 0);
  for (size_t i = 0; i < n; i++) { blob.append(keys[i].data(), keys[i].size()); koff[i + 1] = blob.size(); }
  blob.push_back('\0');
  std::vector<rsp_snapshot*> snaps(n, RawSnapshot(snapshot));
  std::vector<uint32_t> vlen(n);
  std::vector<int32_t> st(n);
  size_t stride = std::max<size_t>(256, value_hint_.load(std::memory_order_relaxed));
  for (;;) {
    std::vector<uint8_t> vals(n * stride);
    const int rc = rsp_multi_get_at(engine(), n, snaps.data(), (const uint8_t*)blob.data(), koff.data(), vals.data(), stride,
                                    vlen.data(), st.data());
    if (rc != RSP_OK) {
      for (auto& s : out) s = Status::IOError("rsp_multi_get_at");
      return out;
    }
    size_t more = 0;
    for (size_t i = 0; i < n; i++) if (st[i] == RSP_INCOMPLETE) more = std::max<size_t>(more, vlen[i]);
    if (more) { stride = more; continue; }
    for (size_t i = 0; i < n; i++) {
      if (st[i] == RSP_OK) (*values)[i].assign((const char*)&vals[i * stride], vlen[i]);
      else out[i] = st[i] == RSP_NOT_FOUND ? Status::NotFound() : ToStatus(st[i]);
    }
    return out;
  }
}

std::vector<Status> GpuDB::MultiGet(const rocksdb::ReadOptions& options, const std::vector<Slice>& keys, std::vector<std::string>* values) {
  if (options.snapshot) return MultiGetAt(options.snapshot, keys, values);
  const size_t n = keys.size();
  std::vector<Status> out(n);
  values->assign(n, std::string());
  if (!n) return out;
  // rocksdb::Slice is {pointer, size}: the key array goes to the engine as it is, and every value is assigned from
  // the engine's pinned result buffer straight into its std::string (one copy each way)
  static_assert(sizeof(Slice) == sizeof(rsp_slice), "rocksdb::Slice and rsp_slice share a layout");
  struct Ctx { GpuDB* db; std::vector<Status>* out; std::vector<std::string>* values; size_t max_vlen; } ctx{this, &out, values, 0};
  const int rc = rsp_multi_get_slices(
      shard_, n, reinterpret_cast<const rsp_slice*>(keys.data()), value_hint_.load(std::memory_order_relaxed),
      [](void* c, size_t i, int st, const uint8_t* v, size_t vlen) {
        Ctx* x = static_cast<Ctx*>(c);
        if (st == RSP_OK) {
          (*x->values)[i].assign((const char*)v, vlen);
          if (vlen > x->max_vlen) x->max_vlen = vlen;
        } else {
          (*x->out)[i] = st == RSP_NOT_FOUND ? Status::NotFound() : x->db->ToStatus(st);
        }
      },
      &ctx);
  if (rc != RSP_OK) {
    for (auto& s : out) s = Status::IOError("rsp_multi_get");
    return out;
  }
  if (ctx.max_vlen > value_hint_.load(std::memory_order_relaxed)) value_hint_.store(ctx.max_vlen, std::memory_order_relaxed);
  return out;
}

namespace {
class GpuIterator : public rocksdb::Iterator {
 public:
  explicit GpuIterator(rsp_iter* it) : it_(it) {}
  ~GpuIterator() override { rsp_iter_destroy(it_); }
  bool Valid() const override { return rsp_iter_valid(it_) != 0; }
  void SeekToFirst() override { rsp_iter_seek_to_first(it_); }
  void SeekToLast() override { rsp_iter_seek_to_last(it_); }
  void Seek(const Slice& t) override { rsp_iter_seek(it_, (const uint8_t*)t.data(), t.size()); }
  void SeekForPrev(const Slice& t) override { rsp_iter_seek_for_prev(it_, (const uint8_t*)t.data(), t.size()); }
  void Next() override { rsp_iter_next(it_); }
  void Prev() override { rsp_iter_prev(it_); }
  Slice key() const override { size_t n; auto p = rsp_iter_key(it_, &n); return Slice((const char*)p, n); }
  Slice value() const override { size_t n; auto p = rsp_iter_value(it_, &n); return Slice((const char*)p, n); }
  Status status() const override {
    const int c = rsp_iter_status(it_);
    return c ? Status::FromCode(c, c == 2 ? "Corruption: Error: Could not perform merge." : "error") : Status::OK();
  }

 private:
  rsp_iter* it_;
};
}  // namespace

rocksdb::Iterator* GpuDB::NewIterator(const rocksdb::ReadOptions& o) {
  rsp_iter* it = o.snapshot ? rsp_iter_create_at(RawSnapshot(o.snapshot)) : rsp_iter_create(shard_);
  if (it && o.iterate_upper_bound)  // the engine keeps its own copy of the bound
    rsp_iter_set_upper_bound(it, (const uint8_t*)o.iterate_upper_bound->data(), o.iterate_upper_bound->size());
  return new GpuIterator(it);
}

Status GpuDB::CompactRange(const rocksdb::CompactRangeOptions& o, const Slice* begin, const Slice* end) {
  if (begin || end) return Status::NotSupported("partial CompactRange");  // the reference passes (nullptr, nullptr)
  // change_level: the ingested-behind tier is folded in too (change_level = false leaves it at the bottom level)
  return ToStatus(rsp_compact_ex(shard_, o.change_level ? RSP_COMPACT_CHANGE_LEVEL : 0u));
}
Status GpuDB::Flush(const rocksdb::FlushOptions&) { return ToStatus(rsp_flush(shard_)); }
rocksdb::SequenceNumber GpuDB::GetLatestSequenceNumber() const { return rsp_latest_seq(shard_); }

// TransactionLogIterator over the update log; tails new writes like RocksDB's WAL iterator
class GpuDB::LogIter : public rocksdb::TransactionLogIterator {
 public:
  LogIter(GpuDB* db, uint64_t chunk_id, size_t idx) : db_(db), id_(chunk_id), idx_(idx) { Load(); }
  bool Valid() override { return cur_ != nullptr; }
  void Next() override { if (cur_) idx_++; Load(); }
  Status status() override { return Status::OK(); }
  rocksdb::BatchResult GetBatch() override {
    rocksdb::BatchResult r;
    const LogChunk::Rec& rec = cur_->recs[idx_];
    r.sequence = rec.first_seq;
    r.writeBatchPtr.reset(new rocksdb::WriteBatch(std::string(cur_->bytes.data() + rec.off, rec.len)));
    return r;
  }

 private:
  void Load() {
    std::lock_guard<std::mutex> g(db_->log_mu_);
    if (id_ < db_->log_base_id_) { id_ = db_->log_base_id_; idx_ = 0; }  // trimmed: first available (a gap, as after WAL TTL)
    for (;;) {
      const uint64_t off = id_ - db_->log_base_id_;
      if (off >= db_->log_.size()) { cur_ = nullptr; return; }  // at the tail: a later Next() finds what was appended since
      cur_ = db_->log_[off];
      if (idx_ < cur_->recs.size()) return;
      id_++;
      idx_ = 0;
    }
  }
  GpuDB* db_;
  uint64_t id_;   // chunk id
  size_t idx_;    // batch within the chunk
  std::shared_ptr<const LogChunk> cur_;
};

Status GpuDB::GetUpdatesSince(rocksdb::SequenceNumber seq, std::unique_ptr<rocksdb::TransactionLogIterator>* iter) {
  iter->reset();
  if (seq > GetLatestSequenceNumber()) return Status::NotFound("Requested sequence not yet written in the db");
  uint64_t id;
  size_t idx = 0;
  {
    std::lock_guard<std::mutex> g(log_mu_);
    // first chunk whose last sequence >= seq, then the first batch in it whose last sequence >= seq
    size_t lo = 0, hi = log_.size();
    while (lo < hi) {
      const size_t m = (lo + hi) / 2;
      if (log_[m]->last_seq < seq) lo = m + 1; else hi = m;
    }
    id = log_base_id_ + lo;
    if (lo < log_.size()) {
      const auto& recs = log_[lo]->recs;
      while (idx < recs.size() && recs[idx].first_seq + recs[idx].count - 1 < seq) idx++;
    }
  }
  iter->reset(new LogIter(this, id, idx));
  return Status::OK();
}

bool GpuDB::GetProperty(const Slice& property, std::string* value) {
  rsp_stats st;
  if (rsp_get_stats(shard_, &st) != RSP_OK) return false;
  const std::string p = property.ToString();
  if (p == "rocksdb.estimate-num-keys") { *value = std::to_string(st.memtable_entries + st.run_entries); return true; }
  if (p == "rocksdb.num-entries-active-mem-table") { *value = std::to_string(st.memtable_entries); return true; }
  if (p == "rocksdb.cur-size-active-mem-table") { *value = std::to_string(st.memtable_bytes); return true; }
  if (p == "rocksdb.total-sst-files-size") { *value = std::to_string(st.run_bytes); return true; }
  if (p == "rocksdb.num-files-at-level0") { *value = std::to_string(st.n_runs > 1 ? st.n_runs - 1 : 0); return true; }
  return false;
}

void GpuDB::GetColumnFamilyMetaData(rocksdb::ColumnFamilyMetaData* meta) {
  // the newest runs play level 0, the oldest (fully merged) run the bottom level.  With allow_ingest_behind the bottom
  // level is the ingested-behind tier alone and every other run sits at level 0 (RocksDB keeps Lmax for those files).
  rsp_stats st;
  rsp_get_stats(shard_, &st);
  meta->levels.clear();
  for (int l = 0; l < options_.num_levels; l++) meta->levels.push_back({l, 0});
  if (options_.allow_ingest_behind) {
    const uint64_t behind = rsp_shard_behind_bytes(shard_);
    meta->levels.back().size = behind;
    meta->levels[0].size += st.run_bytes - behind;
  } else if (st.n_runs == 1) meta->levels.back().size = st.run_bytes;
  else if (st.n_runs > 1) { meta->levels[0].size = st.run_bytes / 2; meta->levels.back().size = st.run_bytes - st.run_bytes / 2; }
  meta->size = st.run_bytes;
  meta->file_count = st.n_runs;
}

}  // namespace b200
