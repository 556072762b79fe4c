// k_apply.cu — the follower-side WriteBatch replay on the device.
//
// Replaces what RocksDbWrapper::HandleReplicateResponse hands to RocksDB
// (rocksdb_replicator/rocksdb_wrapper.cpp:13-28): WriteBatch::Iterate's record walk, DB::Write's
// sequence assignment, and the memtable insert — for a whole tick of batches across many shards.
//
//   k_decode   : one warp per batch.  Walks the records (tag byte, varint32 lengths), validates
//                them with RocksDB's rules and error classes, counts ops / entry units, and emits
//                one OpRec per op.  HBM read of the batch bytes only.
//   k_sequence : one warp per shard group.  In submission order: accept batches until the first
//                failure (which latches, as RocksDB 5.x does), assign sequence numbers
//                last_seq+1.., heap offsets and ordinals by warp prefix sums.
//   k_insert   : eight lanes per op.  Writes the 16-byte-unit entry (unaligned wire bytes ->
//                aligned heap), then links it into the shard's open-addressed table with a
//                lock-free, sequence-ordered version chain (CAS on the slot / on a link word).
//   k_publish  : publishes last_seq to readers (batch atomicity: readers skip newer versions).
#include <cstdlib>

#include "kernels.h"

namespace rsp {

// ------------------------------------------------------------------------------------------------
// k_decode
// ------------------------------------------------------------------------------------------------
// A batch as RocksDB sees it after PutLogData(&timestamp, 8) (rocksdb_wrapper.cpp:19-20): `raw_len` bytes that are
// physically present (in global or in shared memory: plain loads work on both) followed by the VIRTUAL record
// {0x03, 0x08, timestamp LE} of a packed tick.
struct Cursor {
  const u8* p;  // batch base
  u32 pos, len;
  u32 raw_len;  // bytes present; the rest is the virtual LogData(timestamp) record
  u64 ts;
};
__device__ __forceinline__ u32 batch_byte(const u8* p, u32 raw_len, u64 ts, u32 pos) {
  if (pos < raw_len) return p[pos];
  const u32 t = pos - raw_len;
  return t == 0 ? 0x03u : (t == 1 ? 0x08u : (u32)((ts >> (8u * (t - 2u))) & 0xffu));
}
__device__ __forceinline__ u32 cur_byte(const Cursor& c, u32 pos) { return batch_byte(c.p, c.raw_len, c.ts, pos); }
// util/coding.cc GetVarint32Ptr: at most 5 bytes, shift <= 28
__device__ __forceinline__ bool get_varint32(Cursor& c, u32& v) {
  u32 result = 0;
  for (u32 shift = 0; shift <= 28 && c.pos < c.len; shift += 7) {
    u32 byte = cur_byte(c, c.pos);
    c.pos++;
    if (byte & 128) {
      result |= (byte & 127) << shift;
    } else {
      result |= byte << shift;
      v = result;
      return true;
    }
  }
  return false;
}
// GetLengthPrefixedSlice
__device__ __forceinline__ bool get_slice(Cursor& c, u32& off, u32& n) {
  u32 len;
  if (!get_varint32(c, len)) return false;
  if (c.len - c.pos < len) return false;
  off = c.pos;
  n = len;
  c.pos += len;
  return true;
}

// WriteBatch::Iterate's record walk with RocksDB's validation and error classes.  sink(type, koff, klen, voff, vlen,
// units_before, op_index) is called for every data record (offsets relative to the batch base); returns the batch's
// status word (0 = well formed) and its op count / entry units.
struct WalkResult {
  u32 status, n_ops, units;
};
template <class Sink>
__device__ __forceinline__ WalkResult walk_batch(Cursor c, Sink&& sink) {
  u32 status = 0, found = 0, units = 0;
  bool range_del = false;
  if (c.len < 12) return WalkResult{mk_status(2, MSG_TOO_SMALL), 0u, 0u};
  const u32 count = cur_byte(c, 8) | (cur_byte(c, 9) << 8) | (cur_byte(c, 10) << 16) | (cur_byte(c, 11) << 24);
  // Fast path for the unit of the replication stream: ONE Put with a short key, followed only by 8-byte LogData
  // records (the leader's timestamp, the follower's).  Exactly what the general walk below finds for such bytes —
  // anything else (other tags, long keys, trailing garbage) takes the general walk.
  if (count == 1 && c.len >= 16 && cur_byte(c, 12) == kTypeValue) {
    const u32 kl = cur_byte(c, 13);
    const u32 p = 14u + kl;
    if (kl < 128u && p < c.len) {
      const u32 b0 = cur_byte(c, p);
      u32 vl = b0, nb = 1;
      bool ok = true;
      if (b0 >= 128u) {
        const u32 b1 = p + 1 < c.len ? cur_byte(c, p + 1) : 255u;
        ok = b1 < 128u;
        vl = (b0 & 127u) | (b1 << 7);
        nb = 2;
      }
      const u32 vo = p + nb;
      if (ok && vo <= c.len && c.len - vo >= vl && (c.len - vo - vl) % 10u == 0) {
        for (u32 q = vo + vl; q < c.len; q += 10u) ok = ok && cur_byte(c, q) == kTypeLogData && cur_byte(c, q + 1) == 8u;
        if (ok) {
          sink((u32)kTypeValue, 14u, kl, vo, vl, 0u, 0u);
          return WalkResult{0u, 1u, entry_units(kTypeValue, kl, vl, true)};
        }
      }
    }
  }
  c.pos = 12;
  while (c.pos < c.len && status == 0) {
    const u32 tag = cur_byte(c, c.pos);
    c.pos++;
    u32 cf = 0, koff = 0, klen = 0, voff = 0, vlen = 0, type = kTypeInvalid;
    switch (tag) {
      case kTypeColumnFamilyValue:
        if (!get_varint32(c, cf)) { status = mk_status(2, MSG_BAD_PUT); break; }
        /* fallthrough */
      case kTypeValue:
        if (!get_slice(c, koff, klen) || !get_slice(c, voff, vlen)) { status = mk_status(2, MSG_BAD_PUT); break; }
        type = kTypeValue;
        break;
      case kTypeColumnFamilyDeletion:
      case kTypeColumnFamilySingleDeletion:
        if (!get_varint32(c, cf)) { status = mk_status(2, MSG_BAD_DELETE); break; }
        /* fallthrough */
      case kTypeDeletion:
      case kTypeSingleDeletion:
        if (!get_slice(c, koff, klen)) { status = mk_status(2, MSG_BAD_DELETE); break; }
        type = (tag == kTypeDeletion || tag == kTypeColumnFamilyDeletion) ? kTypeDeletion : kTypeSingleDeletion;
        break;
      case kTypeColumnFamilyMerge:
        if (!get_varint32(c, cf)) { status = mk_status(2, MSG_BAD_MERGE); break; }
        /* fallthrough */
      case kTypeMerge:
        if (!get_slice(c, koff, klen) || !get_slice(c, voff, vlen)) { status = mk_status(2, MSG_BAD_MERGE); break; }
        type = kTypeMerge;
        break;
      case kTypeLogData:
        if (!get_slice(c, koff, klen)) status = mk_status(2, MSG_BAD_BLOB);
        continue;  // not counted, no sequence number
      case kTypeNoop:
        continue;
      // two-phase-commit markers: parsed and (outside WAL recovery) ignored by RocksDB; not counted, no sequence number
      case kTypeBeginPrepareXID:
        continue;
      case kTypeEndPrepareXID:
        if (!get_slice(c, koff, klen)) status = mk_status(2, MSG_BAD_END_PREPARE);
        continue;
      case kTypeCommitXID:
        if (!get_slice(c, koff, klen)) status = mk_status(2, MSG_BAD_COMMIT);
        continue;
      case kTypeRollbackXID:
        if (!get_slice(c, koff, klen)) status = mk_status(2, MSG_BAD_ROLLBACK);
        continue;
      // range deletions: parsed and counted with RocksDB's rules; the batch is refused (NotSupported) only if
      // everything else about it is valid, so any other defect is reported as RocksDB reports it
      case kTypeColumnFamilyRangeDeletion:
        if (!get_varint32(c, cf)) { status = mk_status(2, MSG_BAD_DELETE_RANGE); break; }
        /* fallthrough */
      case kTypeRangeDeletion:
        if (!get_slice(c, koff, klen) || !get_slice(c, voff, vlen)) { status = mk_status(2, MSG_BAD_DELETE_RANGE); break; }
        if (cf != 0) { status = mk_status(4, MSG_BAD_CF); break; }
        range_del = true;
        found++;
        continue;
      default:
        status = mk_status(2, MSG_UNKNOWN_TAG);
        break;
    }
    if (status) break;
    if (cf != 0) { status = mk_status(4, MSG_BAD_CF); break; }
    sink(type, koff, klen, voff, vlen, units, found);
    units += entry_units(type, klen, vlen, true);
    found++;
  }
  if (status == 0 && found != count) status = mk_status(2, MSG_WRONG_COUNT);
  if (status == 0 && range_del) status = mk_status(3, MSG_UNSUPPORTED_TAG);
  return WalkResult{status, status ? 0u : found, status ? 0u : units};
}

// k_decode: one warp per batch, every lane walks the same records (uniform control flow; loads broadcast), lane 0
// writes one OpRec per op
__device__ __forceinline__ void decode_batch(const TickDev& t, const u32 warp, const u32 lane) {
  const BatchDesc bd = t.batches[warp];
  Cursor c{t.blob + bd.boff, 12, bd.len, bd.len, 0ull};  // (staged: the LogData record is in the blob)
  const WalkResult w = walk_batch(c, [&](u32 type, u32 koff, u32 klen, u32 voff, u32 vlen, u32 units, u32 found) {
    if (found < bd.op_cap && lane == 0) {
      OpRec r;
      r.koff = bd.boff + koff; r.klen = klen;
      r.voff = bd.boff + voff; r.vlen = vlen;
      r.rel_units = units; r.type = type;
      r.batch_ix = warp; r.op_ix = found;
      t.ops[bd.op_base + found] = r;
    }
  });
  // unused / rejected reserved op slots must read as invalid for k_insert
  const u32 first_dead = w.status ? 0u : min(w.n_ops, bd.op_cap);
  for (u32 i = first_dead + lane; i < bd.op_cap; i += 32u) t.ops[bd.op_base + i].type = kTypeInvalid;
  if (lane == 0) {
    BatchRes r;
    r.status = w.status; r.n_ops = w.n_ops; r.units = w.units;
    r.unit_base = 0; r.seq_base = 0; r.ord_base = 0; r.accepted = 0;
    t.bres[warp] = r;
  }
}

__global__ void __launch_bounds__(256) k_decode(TickDev t) {
  const u32 warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const u32 lane = threadIdx.x & 31;
  if (warp >= t.n_batches) return;
  decode_batch(t, warp, lane);
}

// ------------------------------------------------------------------------------------------------
// k_sequence
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ u32 warp_incl_scan(u32 v, u32 lane) {
#pragma unroll
  for (u32 d = 1; d < 32; d <<= 1) {
    u32 n = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= d) v += n;
  }
  return v;
}

__device__ __forceinline__ void sequence_body(const TickDev& t, ShardDev* shards, ShardFast* fast, const u32 warp, const u32 lane) {
  const GroupDesc g = t.groups[warp];
  ShardDev* sd = shards + g.shard_ix;
  u32 latch = sd->latch;
  u64 seq = sd->last_seq;
  u32 tail = sd->mt_tail, cnt = sd->mt_count;
  const u32 heap_cap = sd->mt_heap_cap, ent_cap = sd->mt_ent_cap;
  for (u32 base = 0; base < g.n_batches; base += 32) {
    const u32 j = base + lane;
    const bool in = j < g.n_batches;
    BatchRes r;
    r.status = 0; r.n_ops = 0; r.units = 0;
    if (in) r = t.bres[g.first_batch + j];
    const u32 bad_mask = __ballot_sync(0xffffffffu, in && r.status != 0);
    const u32 first_bad = bad_mask ? (u32)(__ffs(bad_mask) - 1) : 32u;
    bool accepted = in && latch == 0 && lane < first_bad;
    const u32 ops_in = accepted ? r.n_ops : 0u, units_in = accepted ? r.units : 0u;
    u32 ops_incl = warp_incl_scan(ops_in, lane);
    u32 units_incl = warp_incl_scan(units_in, lane);
    // defensive capacity guard (the host reserves before the tick; never expected to trigger):
    // the first batch that does not fit and everything after it in this chunk is refused, unlatched
    const bool over = accepted && ((u64)tail + units_incl > heap_cap || (u64)cnt + ops_incl > ent_cap);
    const u32 over_mask = __ballot_sync(0xffffffffu, over);
    const u32 first_over = over_mask ? (u32)(__ffs(over_mask) - 1) : 32u;
    if (lane >= first_over) accepted = false;
    const u32 ops2 = accepted ? r.n_ops : 0u, units2 = accepted ? r.units : 0u;
    ops_incl = warp_incl_scan(ops2, lane);
    units_incl = warp_incl_scan(units2, lane);
    const u32 first_status = __shfl_sync(0xffffffffu, r.status, first_bad & 31);
    if (in) {
      r.accepted = accepted ? 1u : 0u;
      r.seq_base = seq + 1 + (ops_incl - ops2);
      r.unit_base = tail + (units_incl - units2);
      r.ord_base = cnt + (ops_incl - ops2);
      if (!accepted) {
        if (latch) r.status = latch;
        else if (lane >= first_over) r.status = mk_status(11, MSG_TOO_LARGE);
        else if (lane > first_bad) r.status = first_status;  // the latch set by an earlier batch of this tick
        r.n_ops = 0; r.units = 0;
      }
      t.bres[g.first_batch + j] = r;
      t.bstat[g.first_batch + j] = accepted ? 0u : r.status;
    }
    seq += __shfl_sync(0xffffffffu, ops_incl, 31);
    tail += __shfl_sync(0xffffffffu, units_incl, 31);
    cnt += __shfl_sync(0xffffffffu, ops_incl, 31);
    if (latch == 0 && bad_mask && first_bad < first_over) latch = first_status;
    if (over_mask && latch == 0) {
      // refuse the remainder of the group without latching: report busy
      for (u32 b2 = base + 32; b2 < g.n_batches; b2 += 32) {
        const u32 j2 = b2 + lane;
        if (j2 < g.n_batches) {
          BatchRes r2 = t.bres[g.first_batch + j2];
          r2.status = mk_status(11, MSG_TOO_LARGE); r2.n_ops = 0; r2.units = 0; r2.accepted = 0;
          t.bres[g.first_batch + j2] = r2;
          t.bstat[g.first_batch + j2] = r2.status;
        }
      }
      break;
    }
  }
  if (lane == 0) {
    sd->last_seq = seq;
    sd->mt_tail = tail;
    sd->mt_count = cnt;
    fast[g.shard_ix].mt_count = cnt;
    sd->latch = latch;
    GroupRes gr;
    gr.last_seq = seq; gr.tail = tail; gr.count = cnt; gr.latch = latch; gr.pad = 0;
    t.gres[warp] = gr;
  }
}

__global__ void __launch_bounds__(128) k_sequence(TickDev t, ShardDev* shards, ShardFast* fast) {
  const u32 warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const u32 lane = threadIdx.x & 31;
  if (warp >= t.n_groups) return;
  sequence_body(t, shards, fast, warp, lane);
}
// ------------------------------------------------------------------------------------------------
// k_insert
// ------------------------------------------------------------------------------------------------
constexpr u32 INS_LANES = 8;

// copy n bytes from an arbitrarily aligned source to a 16-byte aligned destination, zero padding
// the last unit; `lanes` lanes cooperate, one 16-byte unit each per step.
__device__ __forceinline__ void copy_to_units(u8* dst, const u8* src, u32 n, u32 lane, u32 lanes) {
  const u32 nu = units_of(n);
  for (u32 u = lane; u < nu; u += lanes) {
    const u8* s = src + 16u * u;
    const u32 rem = n - 16u * u;  // > 0
    const uintptr_t a = reinterpret_cast<uintptr_t>(s);
    const u32* w = reinterpret_cast<const u32*>(a & ~(uintptr_t)3);
    const u32 sh = (u32)(a & 3u) * 8u;
    u32 x0 = w[0], x1 = w[1], x2 = w[2], x3 = w[3];  // plain loads: the source may be global or shared memory
    uint4 o;
    if (sh) {
      u32 x4 = w[4];
      o.x = __funnelshift_r(x0, x1, sh);
      o.y = __funnelshift_r(x1, x2, sh);
      o.z = __funnelshift_r(x2, x3, sh);
      o.w = __funnelshift_r(x3, x4, sh);
    } else {
      o.x = x0; o.y = x1; o.z = x2; o.w = x3;
    }
    if (rem < 16u) {  // zero the padding bytes
      u32 words[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
      for (u32 i = 0; i < 4; i++) {
        const u32 lo = 4u * i;
        if (rem <= lo) words[i] = 0;
        else if (rem < lo + 4u) words[i] &= (1u << (8u * (rem - lo))) - 1u;
      }
      o = make_uint4(words[0], words[1], words[2], words[3]);
    }
    *reinterpret_cast<uint4*>(dst + 16u * u) = o;
  }
}

__device__ __forceinline__ u64 ld_cg_u64(const u64* p) { return __ldcg(reinterpret_cast<const unsigned long long*>(p)); }
__device__ __forceinline__ u32 ld_cg_u32(const u32* p) { return __ldcg(p); }
// memtable filter (format.cuh): the bit of an inserted key, set before the entry is published
__device__ __forceinline__ void mt_filter_set(u32* filter, u64 h) {
  const u32 b = mt_filter_bit(h);
  u32* w = filter + (b >> 5);
  const u32 m = 1u << (b & 31u);
  if (!(ld_cg_u32(w) & m)) atomicOr(w, m);  // (overwrites of a hot key find the bit set: no atomic)
}

// Link the finished entry at `unit` into the shard's table: find (or claim) the user key's slot, then insert
// the version into the key's chain in sequence order (lock-free; unit offsets grow with sequence).  Keys are
// compared through the entry's own padded heap copy, read through L2.
__device__ __forceinline__ bool eq_heap_keys_cg(const u8* a, u32 an, const u8* b, u32 bn) {
  if (an != bn) return false;
  const u32 nw = (an + 7u) >> 3;
  for (u32 i = 0; i < nw; i++)
    if (ld_cg_u64(reinterpret_cast<const u64*>(a) + i) != ld_cg_u64(reinterpret_cast<const u64*>(b) + i)) return false;
  return true;
}
// `first` is the home slot's word, loaded by the caller BEFORE its __threadfence (the probe's first round trip overlaps
// the fence's wait for the entry stores).
__device__ __noinline__ void link_into_table(ShardDev* sd, u64* slots, u32 mask, u8* heap, u8* ent, u32 unit, u32 klen, u64 h, u64 first) {
  const u32 tag = hash_tag32(h);
  const u32 P = unit + 1u;
  u32* my_link = reinterpret_cast<u32*>(ent + 16);
  u32 idx = (u32)h & mask;
  // The probe is bounded by the table size.  The reservation keeps the table at most half full, so the bound is never
  // reached; if it ever were (a table without a free slot), the entry stays unreachable and the shard latches an
  // IOError instead of the kernel spinning forever.
  for (u32 probes = 0;; probes++) {
    if (probes > mask) {
      atomicCAS(&sd->latch, 0u, mk_status(5, MSG_TOO_LARGE));
      return;
    }
    u64 cur = probes ? ld_cg_u64(slots + idx) : first;
    if (cur == 0) {
      const u64 old = atomicCAS(reinterpret_cast<unsigned long long*>(slots + idx), 0ull, ((u64)tag << 32) | P);
      if (old == 0) return;  // first version of a new key
      cur = old;
    }
    if ((u32)(cur >> 32) == tag) {
      const u8* he = heap + (u64)((u32)cur - 1u) * 16u;
      const u32 hklen = ld_cg_u32(reinterpret_cast<const u32*>(he) + 2);
      if (eq_heap_keys_cg(ent + 32, klen, he + 32, hklen)) break;
    }
    idx = (idx + 1u) & mask;
  }
  for (;;) {
    const u64 cur = ld_cg_u64(slots + idx);
    const u32 H = (u32)cur;
    if (H < P) {  // newer than the current head: become the head
      *my_link = H;
      __threadfence();
      if (atomicCAS(reinterpret_cast<unsigned long long*>(slots + idx), cur, ((u64)tag << 32) | P) == cur) return;
      continue;
    }
    u32 c = H;  // c > P: walk down to my place
    for (;;) {
      u32* clink = reinterpret_cast<u32*>(heap + (u64)(c - 1u) * 16u + 16u);
      const u32 nxt = ld_cg_u32(clink);
      if (nxt > P) {
        c = nxt;
        continue;
      }
      *my_link = nxt;
      __threadfence();
      if (atomicCAS(clink, nxt, P) == nxt) return;
      // lost a race at this link: re-read it
    }
  }
}

__global__ void __launch_bounds__(256) k_insert(TickDev t, ShardDev* shards, u32* mt_filter) {
  const u32 gid = (blockIdx.x * blockDim.x + threadIdx.x) / INS_LANES;
  const u32 lane = threadIdx.x & (INS_LANES - 1);
  const u32 gmask = ((1u << INS_LANES) - 1u) << ((threadIdx.x & 31u) & ~(INS_LANES - 1u));
  if (gid >= t.n_ops_cap) return;
  const OpRec op = t.ops[gid];
  if (op.type == kTypeInvalid) return;
  const BatchRes br = t.bres[op.batch_ix];
  if (!br.accepted) return;
  const u32 six = t.batches[op.batch_ix].shard_ix;
  ShardDev* sd = shards + six;
  u8* heap = sd->mt_heap;
  const u32 unit = br.unit_base + op.rel_units;
  const u64 seq = br.seq_base + op.op_ix;
  const u32 ord = br.ord_base + op.op_ix;
  u8* ent = heap + (u64)unit * 16u;
  u8* kdst = ent + 32u;
  u8* vdst = kdst + 16u * units_of(op.klen);
  const u8* kp = t.blob + op.koff;
  const u64 h = hash_key(kp, op.klen);  // every lane (redundant but free: the loads broadcast)
  copy_to_units(kdst, kp, op.klen, lane, INS_LANES);
  copy_to_units(vdst, t.blob + op.voff, op.vlen, lane, INS_LANES);
  if (lane == 0) {
    uint4 hd;
    const u64 st = (seq << 8) | op.type;
    hd.x = (u32)st; hd.y = (u32)(st >> 32); hd.z = op.klen; hd.w = op.vlen;
    *reinterpret_cast<uint4*>(ent) = hd;
    sd->mt_ent_off[ord] = unit;
  }
  if (lane == 1) *reinterpret_cast<uint4*>(ent + 16) = make_uint4(0u, 0u, (u32)h, (u32)(h >> 32));
  u64* slots = sd->mt_slots;
  const u32 mask = sd->mt_slot_mask;
  if (lane == 0) mt_filter_set(mt_filter + (size_t)six * MT_FILTER_WORDS, h);
  const u64 first = lane == 0 ? ld_cg_u64(slots + ((u32)h & mask)) : 0ull;
  __threadfence();  // the entry is complete before any pointer to it is published
  __syncwarp(gmask);
  if (lane != 0) return;
  link_into_table(sd, slots, mask, heap, ent, unit, op.klen, h, first);
}

// ------------------------------------------------------------------------------------------------
// k_tick_fused — the whole tick in ONE launch for ticks of small batches (the replication stream: single-Put
// WriteBatches of ~105 bytes, <= 50 per shard per pull): one CTA per shard group.
//   stage    : the group's batch bytes — contiguous in a packed tick — are pulled into shared memory with coalesced
//              16-byte vector loads (chunks of <= 128 batches / 32 KB)
//   decode   : a thread per batch walks its records in shared memory (walk_batch: RocksDB's validation, error classes)
//   sequence : block-wide — first failure latches, prefix sums assign sequence numbers / heap units / ordinals
//   insert   : the same thread walks its batch again and writes each entry (shared -> heap, 16-byte units), then links
//              it into the shard's table; per-batch results never leave the SM
//   publish  : when every insert of the group is done
// Against k_decode -> k_sequence -> k_insert -> k_publish this drops three launches and all the per-batch / per-op
// records in global memory (BatchDesc, BatchRes, OpRec: ~350 bytes of traffic per 105-byte batch).
// ------------------------------------------------------------------------------------------------
// One CTA per group: the shape for ticks whose groups are short — 64 threads / 8 KB stage when no group holds more than 64
// batches (the pull protocol's <= 50 per shard: every CTA of a 1024-shard tick is resident at once).  Longer groups go to
// k_tick_chunks below (a CTA per chunk).
constexpr u32 FT_STAGE_PER_THREAD = 128;  // bytes of stage per thread: a chunk of single-Put batches (105-116 B) fills the block

// exclusive block-wide prefix sums of two values at once: one exchange through shared memory, ONE barrier (before the
// read; the caller's next barrier protects the reuse of s_warp)
template <u32 THREADS>
__device__ __forceinline__ void block_excl_scan2(u32 a, u32 b, u32 (*s_warp)[2], u32* a_excl, u32* b_excl, u32* a_tot, u32* b_tot) {
  const u32 lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
  const u32 ai = warp_incl_scan(a, lane), bi = warp_incl_scan(b, lane);
  if (lane == 31) { s_warp[wid][0] = ai; s_warp[wid][1] = bi; }
  __syncthreads();
  u32 ab = 0, bb = 0, at = 0, bt = 0;
#pragma unroll
  for (u32 w = 0; w < THREADS / 32; w++) {
    const u32 x = s_warp[w][0], y = s_warp[w][1];
    if (w < wid) { ab += x; bb += y; }
    at += x; bt += y;
  }
  *a_excl = ab + ai - a; *b_excl = bb + bi - b;
  *a_tot = at; *b_tot = bt;
}

// the memtable of the group's shard as the insert code needs it (loaded once per CTA)
struct MtView {
  ShardDev* sd;
  u8* heap;
  u64* slots;
  u32* ent_off;
  u32* filter;  // the shard's row of the memtable filter
  u32 slot_mask;
};

// second walk of an accepted batch: every entry written (shared memory -> heap, 16-byte units) and linked
__device__ __forceinline__ void insert_batch(const Cursor& c, const MtView& m, u64 seq_base, u32 unit_base, u32 ord_base) {
  const u8* bp = c.p;
  const u32 raw_len = c.raw_len;
  const u64 ts = c.ts;
  walk_batch(c, [&](u32 type, u32 koff, u32 klen, u32 voff, u32 vlen, u32 units_before, u32 op_ix) {
    const u32 unit = unit_base + units_before;
    u8* ent = m.heap + (u64)unit * 16u;
    u8* kdst = ent + 32u;
    u8* vdst = kdst + 16u * units_of(klen);
    u64 h;
    if (koff + klen <= raw_len && voff + vlen <= raw_len) {
      h = hash_key(bp + koff, klen);
      copy_to_units(kdst, bp + koff, klen, 0, 1);
      copy_to_units(vdst, bp + voff, vlen, 0, 1);
    } else {
      // a record that reaches into the virtual LogData bytes (a truncated batch that still parses): byte by byte
      const u32 kpad = units_of(klen) * 16u, vpad = units_of(vlen) * 16u;
      for (u32 b = 0; b < kpad; b++) kdst[b] = b < klen ? (u8)batch_byte(bp, raw_len, ts, koff + b) : (u8)0;
      for (u32 b = 0; b < vpad; b++) vdst[b] = b < vlen ? (u8)batch_byte(bp, raw_len, ts, voff + b) : (u8)0;
      __threadfence();
      u64 hh = hash_init(klen);
      for (u32 i = 0; i < ((klen + 7u) >> 3); i++) hh = hash_step(hh, ld_cg_u64(reinterpret_cast<const u64*>(kdst) + i));
      h = hash_final(hh);
    }
    const u64 st = ((seq_base + op_ix) << 8) | type;
    *reinterpret_cast<uint4*>(ent) = make_uint4((u32)st, (u32)(st >> 32), klen, vlen);
    *reinterpret_cast<uint4*>(ent + 16) = make_uint4(0u, 0u, (u32)h, (u32)(h >> 32));
    m.ent_off[ord_base + op_ix] = unit;
    mt_filter_set(m.filter, h);
    const u64 first = ld_cg_u64(m.slots + ((u32)h & m.slot_mask));  // (in flight across the fence)
    __threadfence();  // the entry is complete before any pointer to it is published
    link_into_table(m.sd, m.slots, m.slot_mask, m.heap, ent, unit, klen, h, first);
  });
}

template <u32 THREADS, u32 MINB>
__global__ void __launch_bounds__(THREADS, MINB) k_tick_fused(FusedTick t, ShardDev* shards, ShardFast* fast, u32* mt_filter) {
  constexpr u32 STAGE = THREADS * FT_STAGE_PER_THREAD;
  __shared__ __align__(16) u8 s_blob[STAGE + 64];
  __shared__ u32 s_warp[THREADS / 32][2];
  __shared__ u32 s_first_bad, s_first_over, s_first_status, s_tot_ops, s_tot_units;
  const u32 tid = threadIdx.x;
  const GroupDesc g = t.groups[blockIdx.x];
  ShardDev* sd = shards + g.shard_ix;
  // group state, identical in every thread
  u32 latch = sd->latch;
  u64 seq = sd->last_seq;
  u32 tail = sd->mt_tail, cnt = sd->mt_count;
  const u32 heap_cap = sd->mt_heap_cap, ent_cap = sd->mt_ent_cap;
  MtView mt;
  mt.sd = sd; mt.heap = sd->mt_heap; mt.slots = sd->mt_slots; mt.ent_off = sd->mt_ent_off; mt.slot_mask = sd->mt_slot_mask;
  mt.filter = mt_filter + (size_t)g.shard_ix * MT_FILTER_WORDS;
  const u32 trailer = t.ts ? 10u : 0u;
  bool stop = false;  // the memtable is full: the rest of the group is refused (busy), unlatched
  if (tid == 0) { s_first_bad = 0xffffffffu; s_first_over = 0xffffffffu; s_first_status = 0; }
  for (u32 c0 = 0; c0 < g.n_batches;) {
    const u32 b0 = g.first_batch + c0;
    const u64 base = __ldg(t.off + b0);
    // ---- chunk extent: as many of the next THREADS batches as fit the stage
    const u32 j = c0 + tid;
    u64 my_off = 0, my_end = 0;
    bool fits = false;
    if (j < g.n_batches) {
      my_off = __ldg(t.off + b0 + tid);
      my_end = t.len ? my_off + __ldg(t.len + b0 + tid) : __ldg(t.off + b0 + tid + 1);
      fits = my_end - base <= STAGE;
    }
    const u32 n_in = (u32)__syncthreads_count(fits);  // offsets grow: the fitting batches are a prefix
    if (n_in == 0) {
      // a batch larger than the stage (the host routes such ticks to the general kernels; kept as a guard)
      if (tid == 0) t.bstat[b0] = latch ? latch : mk_status(11, MSG_TOO_LARGE);
      c0 += 1;
      continue;
    }
    // (the last fitting batch's own end bounds the chunk)
    const u32 chunk_bytes = (u32)((t.len ? __ldg(t.off + b0 + n_in - 1) + __ldg(t.len + b0 + n_in - 1) : __ldg(t.off + b0 + n_in)) - base);
    // ---- stage (aligned 16-byte loads; `shift` leading bytes belong to the previous batch / group)
    const u8* src = t.blob + base;
    const u32 shift = (u32)(reinterpret_cast<uintptr_t>(src) & 15u);
    const uint4* src4 = reinterpret_cast<const uint4*>(src - shift);
    const u32 n_units = (shift + chunk_bytes + 15u) >> 4;
    for (u32 u = tid; u < n_units; u += THREADS) reinterpret_cast<uint4*>(s_blob)[u] = __ldg(src4 + u);
    const bool in = tid < n_in;
    const u64 my_ts = (in && t.ts) ? __ldg(t.ts + b0 + tid) : 0ull;
    __syncthreads();
    // ---- decode (count pass)
    Cursor c{s_blob + shift + (u32)(my_off - base), 12, (u32)(my_end - my_off) + trailer, (u32)(my_end - my_off), my_ts};
    WalkResult w{0u, 0u, 0u};
    if (in) w = walk_batch(c, [](u32, u32, u32, u32, u32, u32, u32) {});
    if (in && w.status) atomicMin(&s_first_bad, tid);
    // ---- sequence: the prefix sums run over every well-formed batch of the chunk; what lies behind the first failure
    // (or the first batch without room) is cut off afterwards — a prefix does not depend on what follows it
    u32 ops_excl, units_excl, tot_ops, tot_units;
    block_excl_scan2<THREADS>(w.status ? 0u : w.n_ops, w.status ? 0u : w.units, s_warp, &ops_excl, &units_excl, &tot_ops, &tot_units);
    const u32 first_bad = s_first_bad;  // (the scan's barrier ordered the atomicMin)
    const bool stopped = stop;
    const bool live = latch == 0 && !stopped;
    // defensive capacity guard (the host reserves from an estimate): the first batch that does not fit and everything
    // after it is refused, unlatched
    const bool over = in && live && tid < first_bad && ((u64)tail + units_excl + w.units > heap_cap || (u64)cnt + ops_excl + w.n_ops > ent_cap);
    if (over) atomicMin(&s_first_over, tid);
    if (in && tid == first_bad) { s_first_status = w.status; s_tot_ops = ops_excl; s_tot_units = units_excl; }
    __syncthreads();
    const u32 first_over = s_first_over, first_status = s_first_status;
    if (first_bad != 0xffffffffu) { tot_ops = s_tot_ops; tot_units = s_tot_units; }
    if (first_over != 0xffffffffu) {  // totals of the accepted prefix only: the exclusive sums at the first refused batch
      __syncthreads();
      if (tid == first_over) { s_tot_ops = ops_excl; s_tot_units = units_excl; }
      __syncthreads();
      tot_ops = s_tot_ops;
      tot_units = s_tot_units;
    }
    if (!live) { tot_ops = 0; tot_units = 0; }
    const bool accepted = in && live && tid < first_bad && tid < first_over;
    if (in) {
      u32 st_out = 0;
      if (!accepted) {
        if (latch) st_out = latch;
        else if (stopped || tid >= first_over) st_out = mk_status(11, MSG_TOO_LARGE);
        else if (tid > first_bad) st_out = first_status;  // the latch set by an earlier batch of this tick
        else st_out = w.status;
      }
      t.bstat[b0 + tid] = st_out;
    }
    // ---- insert: the batch's thread walks it again and writes / links each entry
    if (accepted && w.n_ops) insert_batch(c, mt, seq + 1 + ops_excl, tail + units_excl, cnt + ops_excl);
    // ---- group state after this chunk (uniform)
    seq += tot_ops;
    tail += tot_units;
    cnt += tot_ops;
    const u32 lim = min(n_in, first_over);
    if (live && first_bad < lim) latch = first_status;
    if (first_over != 0xffffffffu && latch == 0) stop = true;
    c0 += n_in;
    __syncthreads();  // s_blob and the chunk scalars are reused
    if (tid == 0) { s_first_bad = 0xffffffffu; s_first_over = 0xffffffffu; s_first_status = 0; }
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    sd->last_seq = seq;
    sd->mt_tail = tail;
    sd->mt_count = cnt;
    fast[g.shard_ix].mt_count = cnt;
    sd->latch = latch;
    GroupRes gr;
    gr.last_seq = seq; gr.tail = tail; gr.count = cnt; gr.latch = latch; gr.pad = 0;
    t.gres[blockIdx.x] = gr;
    __threadfence();
    sd->pub_seq = seq;  // every insert of the group is done: readers may see the new versions
  }
}

// ------------------------------------------------------------------------------------------------
// k_tick_chunks — the fused tick for groups longer than one chunk: ONE CTA PER CHUNK (<= 128 batches / 16 KB, cut by the
// host), all chunks of a tick in flight at once.  A chunk stages and decodes on its own, then takes the group's
// sequencing state (last sequence number, heap tail, entry count, latch, stop) from its predecessor's chain record —
// the first chunk of a group from the shard descriptor — adds its own totals, publishes its record and only then
// writes its entries: the decode of chunk i + 1 overlaps the insert of chunk i, and a 1024 x 1000-batch tick is 8192
// short CTAs instead of 1024 CTAs walking eight chunks each (k_tick_fused: one wave of long latency chains).
// The chunks of a group are consecutive blocks: a waiting chunk's predecessor has a smaller block index, so it is
// resident or finished (blocks are dispatched in index order) and the chain always advances; the wait is bounded
// anyway (a chunk that gives up poisons the chain: the shard latches an IOError).  The CTA that finishes a group last
// (a counter per group) publishes the group's state and pub_seq.
// ------------------------------------------------------------------------------------------------
constexpr u32 TC_THREADS = 128;
constexpr u32 TC_STAGE = TC_THREADS * FT_STAGE_PER_THREAD;
static_assert(TC_THREADS == FUSED_CHUNK_BATCHES && TC_STAGE == FUSED_STAGE_BYTES, "the host cuts the chunks by these bounds");
constexpr u32 CHAIN_READY = 1u << 31, CHAIN_STOP = 1u << 30, CHAIN_POISON = 1u << 29;

__device__ __forceinline__ u64 ld_volatile_u64(const u64* p) { return *reinterpret_cast<const volatile u64*>(p); }
__device__ __forceinline__ void st_volatile_u64(u64* p, u64 v) { *reinterpret_cast<volatile u64*>(p) = v; }

__global__ void __launch_bounds__(TC_THREADS, 8) k_tick_chunks(FusedTick t, ShardDev* shards, ShardFast* fast, u32* mt_filter) {
  __shared__ __align__(16) u8 s_blob[TC_STAGE + 64];
  __shared__ u32 s_warp[TC_THREADS / 32][2];
  __shared__ u32 s_first_bad, s_first_over, s_first_status, s_tot_ops, s_tot_units;
  __shared__ u64 s_seq;
  __shared__ u32 s_tail, s_cnt, s_latch, s_flags;
  const u32 tid = threadIdx.x;
  const ChunkDesc ck = t.chunks[blockIdx.x];
  ShardDev* sd = shards + ck.shard_ix;
  MtView mt;
  mt.sd = sd; mt.heap = sd->mt_heap; mt.slots = sd->mt_slots; mt.ent_off = sd->mt_ent_off; mt.slot_mask = sd->mt_slot_mask;
  mt.filter = mt_filter + (size_t)ck.shard_ix * MT_FILTER_WORDS;
  const u32 heap_cap = sd->mt_heap_cap, ent_cap = sd->mt_ent_cap;
  const u32 trailer = t.ts ? 10u : 0u;
  if (tid == 0) { s_first_bad = 0xffffffffu; s_first_over = 0xffffffffu; s_first_status = 0; }
  // ---- stage
  const u32 b0 = ck.first_batch, n_in = ck.n_batches;
  const u64 base = __ldg(t.off + b0);
  const bool in = tid < n_in;
  u64 my_off = 0, my_end = 0;
  if (in) {
    my_off = __ldg(t.off + b0 + tid);
    my_end = t.len ? my_off + __ldg(t.len + b0 + tid) : __ldg(t.off + b0 + tid + 1);
  }
  const u32 chunk_bytes = (u32)((t.len ? __ldg(t.off + b0 + n_in - 1) + __ldg(t.len + b0 + n_in - 1) : __ldg(t.off + b0 + n_in)) - base);
  const u8* src = t.blob + base;
  const u32 shift = (u32)(reinterpret_cast<uintptr_t>(src) & 15u);
  const uint4* src4 = reinterpret_cast<const uint4*>(src - shift);
  const u32 n_units = (shift + chunk_bytes + 15u) >> 4;
  for (u32 u = tid; u < n_units; u += TC_THREADS) reinterpret_cast<uint4*>(s_blob)[u] = __ldg(src4 + u);
  const u64 my_ts = (in && t.ts) ? __ldg(t.ts + b0 + tid) : 0ull;
  __syncthreads();
  // ---- decode (count pass) + prefix sums over the well-formed batches
  Cursor c{s_blob + shift + (u32)(my_off - base), 12, (u32)(my_end - my_off) + trailer, (u32)(my_end - my_off), my_ts};
  WalkResult w{0u, 0u, 0u};
  if (in) w = walk_batch(c, [](u32, u32, u32, u32, u32, u32, u32) {});
  if (in && w.status) atomicMin(&s_first_bad, tid);
  u32 ops_excl, units_excl, tot_ops, tot_units;
  block_excl_scan2<TC_THREADS>(w.status ? 0u : w.n_ops, w.status ? 0u : w.units, s_warp, &ops_excl, &units_excl, &tot_ops, &tot_units);
  const u32 first_bad = s_first_bad;
  // ---- the predecessor's record, AFTER this chunk's own decode: a chunk that waits has nothing left to do but the
  // totals, so the chain advances in a few hundred nanoseconds per link (polling before the decode serialised the
  // decodes of a group, slower than the CTA-per-group kernel)
  if (tid == 0) {
    u64 seq; u32 tail, cnt, latch, flags = 0;
    if (ck.index_in_group == 0) {
      seq = sd->last_seq; tail = sd->mt_tail; cnt = sd->mt_count; latch = sd->latch;
    } else {
      const u64* rec = t.chain + 4ull * (blockIdx.x - 1u);
      u64 w2 = 0;
      u32 polls = 0;
      for (;; polls++) {
        w2 = ld_volatile_u64(rec + 2);
        if ((u32)(w2 >> 32) & CHAIN_READY) break;
        if (polls > (1u << 24)) break;  // (never expected: the predecessor is resident or finished)
        __nanosleep(polls < 64 ? 20u : 200u);
      }
      __threadfence();
      if ((u32)(w2 >> 32) & CHAIN_READY) {
        seq = ld_volatile_u64(rec + 0);
        const u64 w1 = ld_volatile_u64(rec + 1);
        tail = (u32)w1; cnt = (u32)(w1 >> 32);
        latch = (u32)w2; flags = (u32)(w2 >> 32) & (CHAIN_STOP | CHAIN_POISON);
      } else {
        seq = 0; tail = 0; cnt = 0; latch = mk_status(5, MSG_TOO_LARGE); flags = CHAIN_POISON;
      }
    }
    s_seq = seq; s_tail = tail; s_cnt = cnt; s_latch = latch; s_flags = flags;
  }
  __syncthreads();
  const u64 seq = s_seq;
  const u32 tail = s_tail, cnt = s_cnt, latch = s_latch, flags_in = s_flags;
  const bool stopped = (flags_in & CHAIN_STOP) != 0;
  const bool live = latch == 0 && !stopped;
  const bool over = in && live && tid < first_bad && ((u64)tail + units_excl + w.units > heap_cap || (u64)cnt + ops_excl + w.n_ops > ent_cap);
  if (over) atomicMin(&s_first_over, tid);
  if (in && tid == first_bad) { s_first_status = w.status; s_tot_ops = ops_excl; s_tot_units = units_excl; }
  __syncthreads();
  const u32 first_over = s_first_over, first_status = s_first_status;
  if (first_bad != 0xffffffffu) { tot_ops = s_tot_ops; tot_units = s_tot_units; }
  if (first_over != 0xffffffffu) {
    __syncthreads();
    if (tid == first_over) { s_tot_ops = ops_excl; s_tot_units = units_excl; }
    __syncthreads();
    tot_ops = s_tot_ops;
    tot_units = s_tot_units;
  }
  if (!live) { tot_ops = 0; tot_units = 0; }
  // ---- this chunk's record: the successor goes on while the entries below are written
  u32 latch_out = latch, flags_out = flags_in;
  {
    const u32 lim = min(n_in, first_over);
    if (live && first_bad < lim) latch_out = first_status;
    if (first_over != 0xffffffffu && latch_out == 0) flags_out |= CHAIN_STOP;
  }
  if (tid == 0) {
    u64* rec = t.chain + 4ull * blockIdx.x;
    st_volatile_u64(rec + 0, seq + tot_ops);
    st_volatile_u64(rec + 1, (u64)(tail + tot_units) | ((u64)(cnt + tot_ops) << 32));
    __threadfence();
    st_volatile_u64(rec + 2, (u64)latch_out | ((u64)(flags_out | CHAIN_READY) << 32));
  }
  const bool accepted = in && live && tid < first_bad && tid < first_over;
  if (in) {
    u32 st_out = 0;
    if (!accepted) {
      if (latch) st_out = latch;
      else if (stopped || tid >= first_over) st_out = mk_status(11, MSG_TOO_LARGE);
      else if (tid > first_bad) st_out = first_status;
      else st_out = w.status;
    }
    t.bstat[b0 + tid] = st_out;
  }
  if (accepted && w.n_ops) insert_batch(c, mt, seq + 1 + ops_excl, tail + units_excl, cnt + ops_excl);
  // ---- the group's last finisher publishes its state
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const u32 done = atomicAdd(t.group_done + ck.group, 1u);
    if (done + 1u == ck.group_chunks) {
      __threadfence();
      const u64* rec = t.chain + 4ull * (blockIdx.x - ck.index_in_group + ck.group_chunks - 1u);
      const u64 fseq = ld_volatile_u64(rec + 0), w1 = ld_volatile_u64(rec + 1), w2 = ld_volatile_u64(rec + 2);
      const u32 flatch = (u32)w2;
      GroupRes gr;
      if ((u32)(w2 >> 32) & CHAIN_POISON) {
        sd->latch = flatch;
        gr.last_seq = sd->last_seq; gr.tail = sd->mt_tail; gr.count = sd->mt_count; gr.latch = flatch; gr.pad = 0;
        t.gres[ck.group] = gr;
      } else {
        sd->last_seq = fseq;
        sd->mt_tail = (u32)w1;
        sd->mt_count = (u32)(w1 >> 32);
        fast[ck.shard_ix].mt_count = (u32)(w1 >> 32);
        sd->latch = flatch;
        gr.last_seq = fseq; gr.tail = (u32)w1; gr.count = (u32)(w1 >> 32); gr.latch = flatch; gr.pad = 0;
        t.gres[ck.group] = gr;
        __threadfence();
        sd->pub_seq = fseq;  // every insert of the group is done: readers may see the new versions
      }
    }
  }
}

void launch_tick_fused(const FusedTick& t, ShardDev* shards, ShardFast* fast, u32* mt_filter, cudaStream_t s) {
  if (!t.n_groups) return;
  if (fused_small_shape(t.max_group, t.max_len)) {
    k_tick_fused<64, 16><<<t.n_groups, 64, 0, s>>>(t, shards, fast, mt_filter);
  } else {
    // Long groups: a CTA per group (k_tick_fused at 128 threads, the chunks of a group one after the other) when the
    // groups alone fill the machine, a CTA per chunk (k_tick_chunks) when they do not — with enough groups the chain
    // of a group costs more than the tail of one wave; a tick of a few very long groups has no other source of
    // parallelism than its chunks.
    static const int force = [] { const char* v = getenv("RSP_TICK_CHUNKS"); return v ? (atoi(v) ? 1 : 0) : -1; }();
    const bool per_group = force < 0 ? t.n_groups >= 4u * DEVICE_SMS : force == 0;
    if (per_group) {
      k_tick_fused<128, 8><<<t.n_groups, 128, 0, s>>>(t, shards, fast, mt_filter);
      return;
    }
    // (chain records and the per-group counters sit next to each other: one clear)
    cudaMemsetAsync(t.chain, 0, (size_t)t.n_chunks * 32 + (size_t)t.n_groups * 4, s);
    k_tick_chunks<<<t.n_chunks, TC_THREADS, 0, s>>>(t, shards, fast, mt_filter);
  }
}

__global__ void k_publish(TickDev t, ShardDev* shards) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= t.n_groups) return;
  ShardDev* sd = shards + t.groups[i].shard_ix;
  sd->pub_seq = sd->last_seq;
}

void launch_decode(const TickDev& t, cudaStream_t s) {
  if (!t.n_batches) return;
  const u32 warps_per_block = 8;
  k_decode<<<(t.n_batches + warps_per_block - 1) / warps_per_block, warps_per_block * 32, 0, s>>>(t);
}
void launch_sequence(const TickDev& t, ShardDev* shards, ShardFast* fast, cudaStream_t s) {
  if (!t.n_groups) return;
  k_sequence<<<(t.n_groups + 3) / 4, 128, 0, s>>>(t, shards, fast);
}
void launch_insert(const TickDev& t, ShardDev* shards, u32* mt_filter, cudaStream_t s) {
  if (!t.n_ops_cap) return;
  const u32 per_block = 256 / INS_LANES;
  k_insert<<<(t.n_ops_cap + per_block - 1) / per_block, 256, 0, s>>>(t, shards, mt_filter);
}
void launch_publish(const TickDev& t, ShardDev* shards, cudaStream_t s) {
  if (!t.n_groups) return;
  k_publish<<<(t.n_groups + 127) / 128, 128, 0, s>>>(t, shards);
}

}  // namespace rsp
