// format.cuh — HBM data layout shared by every kernel of the engine.
//
// Replaces (as storage) what rocksdb::DB keeps behind rocksdb_replicator/rocksdb_wrapper.cpp:7,22 and
// rocksdb_admin/application_db.cpp:78-120: a memtable and a stack of sorted, immutable runs per shard.
//
// ENTRY (all offsets in 16-byte "units"; every entry starts unit-aligned):
//   unit 0      : u64 seqtype (sequence << 8 | ValueType, RocksDB's internal-key trailer)
//                 u32 klen, u32 vlen
//   [unit 1]    : memtable entries only: u32 prev_plus1 (next older version of the same user key,
//                 unit offset + 1, 0 = none), u32 pad, u64 key hash
//   key         : klen bytes, zero padded to a multiple of 16
//   value       : vlen bytes, zero padded to a multiple of 16
//   => in a run the benchmark's 16 B key / 64 B value Put is exactly 96 B = three 32-byte sectors.
//
// MEMTABLE (per shard; "per-shard open-addressed HBM memtable"):
//   heap      : append-only entry heap, unit offsets assigned in sequence order by the sequencing kernel
//   slots     : u64 open-addressed table, linear probing; slot = tag32 << 32 | (head unit offset + 1);
//               one slot per USER KEY, pointing at its newest version; older versions chain downward
//               through prev_plus1 in strictly decreasing sequence order, so a reader pinned at a
//               published sequence number walks past newer, not-yet-published versions (WriteBatch
//               atomicity for readers running concurrently with an apply tick)
//   ent_off   : unit offset of entry #i (i = insertion ordinal) — random access for flush
//
// RUN (immutable, sorted by (user key asc, newest first); "SST-like HBM blocks"):
//   heap      : entries back to back in sort order (no link unit)
//   ent_off   : unit offset of sorted entry #i (the restart array: every entry is a restart point)
//   blk_pfx   : first-key 8-byte big-endian prefix of every RSP_BLOCK_ENTRIES-entry block (block index)
//   hslots    : u32 bucketised hash index over the FIRST version of each user key:
//               slot = tag << ord_bits | (ordinal + 1); 8 slots = one 32-byte sector per bucket
//   uniform_units : entry size in units when every entry has the same size (ordinal * U addressing)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rsp {

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;
typedef int32_t i32;
typedef int64_t i64;

// RocksDB ValueType (db/dbformat.h) — the tag bytes of the WriteBatch wire format
enum : u32 {
  kTypeDeletion = 0x0,
  kTypeValue = 0x1,
  kTypeMerge = 0x2,
  kTypeLogData = 0x3,
  kTypeColumnFamilyDeletion = 0x4,
  kTypeColumnFamilyValue = 0x5,
  kTypeColumnFamilyMerge = 0x6,
  kTypeSingleDeletion = 0x7,
  kTypeColumnFamilySingleDeletion = 0x8,
  kTypeBeginPrepareXID = 0x9,
  kTypeEndPrepareXID = 0xA,
  kTypeCommitXID = 0xB,
  kTypeRollbackXID = 0xC,
  kTypeNoop = 0xD,
  kTypeColumnFamilyRangeDeletion = 0xE,
  kTypeRangeDeletion = 0xF,
  kTypeInvalid = 0xFF
};

// decode results: (rocksdb::Status::Code << 8) | message id  (message table in engine.cu)
enum : u32 {
  MSG_NONE = 0,
  MSG_TOO_SMALL,
  MSG_BAD_PUT,
  MSG_BAD_DELETE,
  MSG_BAD_MERGE,
  MSG_BAD_BLOB,
  MSG_UNKNOWN_TAG,
  MSG_WRONG_COUNT,
  MSG_BAD_CF,
  MSG_UNSUPPORTED_TAG,
  MSG_MERGE_NOT_INIT,
  MSG_MERGE_FAILED,
  MSG_TOO_LARGE,
  MSG_BAD_END_PREPARE,
  MSG_BAD_COMMIT,
  MSG_BAD_ROLLBACK,
  MSG_BAD_DELETE_RANGE,
  MSG_COUNT
};
__host__ __device__ inline u32 mk_status(u32 code, u32 msg) { return (code << 8) | msg; }

constexpr u32 RSP_MAX_RUNS = 8;
constexpr u32 RSP_BLOCK_ENTRIES = 32;  // entries per index block of a run
constexpr u32 RUN_BUCKET_SLOTS = 8;    // u32 slots per hash bucket = one 32 B sector

// internal lookup results beyond rocksdb codes
constexpr i32 ST_NEED_HOST_MERGE = 100;

// RSP_MERGE_STRING_APPEND: existing + delimiter + operand, folded on the device.  The device also folds the counter (1)
// and uint64add (2); RSP_MERGE_APPEND (3), RSP_MERGE_CALLBACK (4) and unknown operators are folded on the host.
constexpr u32 MERGE_OP_STRING_APPEND = 5;

struct __align__(16) RunDev {
  const u8* heap;
  const u32* ent_off;
  const u32* hslots;
  const u64* blk_pfx;
  u32 n_ent;
  u32 n_buckets;
  u32 ord_bits;
  u32 uniform_units;
  u32 n_blocks;
  u32 heap_units;
  u32 flags;     // RUN_ALL_PUT_FIXED: every entry is a Put with the same klen and vlen (scan fast path)
  u32 kv_len;    // klen | vlen << 16 when RUN_ALL_PUT_FIXED
};
constexpr u32 RUN_ALL_PUT_FIXED = 1u;

struct __align__(16) ShardDev {
  // ---- memtable
  u8* mt_heap;
  u64* mt_slots;
  u32* mt_ent_off;
  u32 mt_slot_mask;
  u32 mt_heap_cap;   // units
  u32 mt_ent_cap;    // entries
  u32 mt_tail;       // units used        (written by k_sequence)
  u32 mt_count;      // entries inserted  (written by k_sequence)
  u32 merge_op;
  u64 last_seq;      // assigned          (written by k_sequence)
  u64 pub_seq;       // published: readers ignore versions newer than this (batch atomicity)
  u32 latch;         // mk_status(code,msg) of the latched write error, 0 = healthy
  u32 n_runs;
  u32 live;
  u32 merge_delim;   // RSP_MERGE_STRING_APPEND: 0 = no delimiter, 0x100 | c = the byte c
  RunDev runs[RSP_MAX_RUNS];  // [0] = newest
};

// The 32 bytes of a shard the 16-byte-key MultiGet kernel needs before it touches data: small enough
// (32 B x #shards) to stay L1/L2-resident.  Written by the host when runs change, mt_count by k_sequence.
struct __align__(32) ShardFast {
  u64 run0_heap;
  u64 run0_hslots;
  u32 n_buckets;
  u32 meta;      // one byte each: ord_bits | uniform_units << 8 | n_runs << 16 | FAST_META_LIVE
  u32 mt_count;
  u32 merge_op;
};
constexpr u32 FAST_META_UNITS_SHIFT = 8;   // uniform_units, capped at 255 (0 and 255: the generic path)
constexpr u32 FAST_META_RUNS_SHIFT = 16;   // the shard's run count, capped at 255 (per-run descriptors: 0)
constexpr u32 FAST_META_LIVE = 1u << 24;   // the shard is open (per-run descriptors: 0)

// ---- memtable filter -------------------------------------------------------------------------------
// One bit per inserted key hash, MT_FILTER_BITS per shard, in one array behind the ShardFast descriptors (8 MB for 1024
// shards: L2-resident).  The 16-byte-key MultiGet kernels consult it before they touch a memtable: a clear bit means the
// key is not there, and the lookup skips the descriptor + slot-table round trips (a non-empty memtable used to cost
// every lookup of its shard two dependent accesses, one of them to HBM).  Set by the insert kernels before an entry
// is published, cleared when the memtable is flushed.
constexpr u32 MT_FILTER_BITS = 65536;
constexpr u32 MT_FILTER_WORDS = MT_FILTER_BITS / 32;
__host__ __device__ inline u32 mt_filter_bit(u64 h) { return (u32)(h >> 40) & (MT_FILTER_BITS - 1u); }

// ---- entry accessors ----------------------------------------------------------------------------
struct EntryHdr {
  u64 seqtype;
  u32 klen;
  u32 vlen;
};
__host__ __device__ inline u32 units_of(u32 n) { return (n + 15u) >> 4; }
__host__ __device__ inline u32 entry_units(u32 type, u32 klen, u32 vlen, bool in_memtable) {
  (void)type;
  return 1u + (in_memtable ? 1u : 0u) + units_of(klen) + units_of(vlen);
}

// ---- hashing --------------------------------------------------------------------------------------
// One step per 8-byte little-endian word of the zero-padded key, then a finaliser.  Keys are stored
// zero-padded, so stored keys and query keys hash through the same word sequence.
__host__ __device__ inline u64 hash_init(u32 klen) { return 0x5EED0001D1B54A32ull ^ ((u64)klen * 0x9E3779B97F4A7C15ull); }
__host__ __device__ inline u64 hash_step(u64 h, u64 w) {
  h = (h ^ w) * 0xff51afd7ed558ccdull;
  return h ^ (h >> 32);
}
__host__ __device__ inline u64 hash_final(u64 h) {
  h ^= h >> 33;
  h *= 0xc4ceb9fe1a85ec53ull;
  h ^= h >> 29;
  return h;
}
__host__ __device__ inline u32 hash_tag32(u64 h) {
  u32 t = (u32)(h >> 32);
  return t ? t : 1u;
}

#ifdef __CUDACC__
// load the i-th 8-byte LE word of a key of n bytes at arbitrary alignment, zero padded
__device__ __forceinline__ u64 load_key_word(const u8* p, u32 n, u32 i) {
  u32 base = i * 8u;
  u64 w = 0;
  if (base + 8u <= n && ((((uintptr_t)p) + base) & 7u) == 0) {
    return *reinterpret_cast<const u64*>(p + base);
  }
#pragma unroll
  for (u32 b = 0; b < 8; b++) {
    if (base + b < n) w |= (u64)p[base + b] << (8u * b);
  }
  return w;
}
__device__ __forceinline__ u64 hash_key(const u8* p, u32 n) {
  u64 h = hash_init(n);
  u32 nw = (n + 7u) >> 3;
  for (u32 i = 0; i < nw; i++) h = hash_step(h, load_key_word(p, n, i));
  return hash_final(h);
}
// key stored in a heap: 16-byte aligned, zero padded
__device__ __forceinline__ u64 hash_key_padded(const u64* p, u32 n) {
  u64 h = hash_init(n);
  u32 nw = (n + 7u) >> 3;
  for (u32 i = 0; i < nw; i++) h = hash_step(h, p[i]);
  return hash_final(h);
}
__device__ __forceinline__ u64 bswap64(u64 x) {
  u32 lo = (u32)x, hi = (u32)(x >> 32);
  return ((u64)__byte_perm(lo, 0, 0x0123) << 32) | (u64)__byte_perm(hi, 0, 0x0123);
}
// big-endian 8-byte prefix of a key (zero padded): integer order == bytewise order of the prefix
__device__ __forceinline__ u64 key_prefix_be(const u8* p, u32 n) { return bswap64(load_key_word(p, n, 0)); }

// bytewise compare of an arbitrary-alignment key (a) against a padded heap key (b)
__device__ __forceinline__ int cmp_key_vs_padded(const u8* a, u32 an, const u64* b, u32 bn) {
  u32 nw = (min(an, bn) + 7u) >> 3;
  for (u32 i = 0; i < nw; i++) {
    u64 x = bswap64(load_key_word(a, an, i));
    u64 y = bswap64(b[i]);
    if (x != y) return x < y ? -1 : 1;
  }
  return an < bn ? -1 : (an > bn ? 1 : 0);
}
__device__ __forceinline__ int cmp_padded(const u64* a, u32 an, const u64* b, u32 bn) {
  u32 nw = (min(an, bn) + 7u) >> 3;
  for (u32 i = 0; i < nw; i++) {
    u64 x = bswap64(a[i]);
    u64 y = bswap64(b[i]);
    if (x != y) return x < y ? -1 : 1;
  }
  return an < bn ? -1 : (an > bn ? 1 : 0);
}
__device__ __forceinline__ bool eq_key_vs_padded(const u8* a, u32 an, const u64* b, u32 bn) {
  if (an != bn) return false;
  u32 nw = (an + 7u) >> 3;
  for (u32 i = 0; i < nw; i++)
    if (load_key_word(a, an, i) != b[i]) return false;
  return true;
}
// same, the heap key read through L2 (memtable entries may be written by a concurrent kernel)
__device__ __forceinline__ bool eq_key_vs_padded_cg(const u8* a, u32 an, const u64* b, u32 bn) {
  if (an != bn) return false;
  u32 nw = (an + 7u) >> 3;
  for (u32 i = 0; i < nw; i++)
    if (load_key_word(a, an, i) != __ldcg(reinterpret_cast<const unsigned long long*>(b) + i)) return false;
  return true;
}
#endif

}  // namespace rsp
