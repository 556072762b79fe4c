// k_read.cu — Get / MultiGet / range-scan kernels.
//
// Replaces what ApplicationDB::Get / MultiGet / NewIterator hand to rocksdb::DB
// (rocksdb_admin/application_db.cpp:78-120): for each key, walk the versions newest -> oldest
// (memtable chain, then each sorted run newest first); Put answers, Delete/SingleDelete hides,
// Merge operands accumulate and are folded oldest -> newest with the AssociativeMergeOperator rules
// of examples/counter_service/merge_operator.cpp:23-45 / RocksDB's uint64add / RocksDB's StringAppendOperator on the
// device, or are handed to the host for any other operator.
//
// A query is served by a group of G lanes (8 for MultiGet): one 32-byte sector of hash slots is one
// coalesced group load, an entry is read as consecutive 16-byte units, the value leaves as
// consecutive 16-byte stores.  All lanes of a group run the same control flow.
#include <algorithm>
#include <cstddef>
#include <type_traits>

#include "kernels.h"

namespace rsp {

__device__ __forceinline__ u64 ldcg64(const void* p) { return __ldcg(reinterpret_cast<const unsigned long long*>(p)); }
__device__ __forceinline__ u32 ldcg32(const void* p) { return __ldcg(reinterpret_cast<const u32*>(p)); }

// ---- merge accumulator (device-resident operators) ------------------------------------------------
// RSP_MERGE_STRING_APPEND folds in place: the result is built where it is answered (the lookup's value slot, the scan
// record's value), which the caller names with set_out before the walk.  The walk visits the operands newest first, so
// each goes out byte-reversed followed by the delimiter, and the base, reversed, last:
// rev(o_n) d .. rev(o_1) d rev(b).  One reversal of the whole value then gives b d o_1 .. d o_n.  Bytes past the
// capacity are not written but still counted, so that res_len is the exact size needed.  The lanes of the group share
// the copies: every visit is made by all of them alike.
// CAT = false instances have none of this code and hand such a shard's operands to the host; the engine launches them
// while no string-append shard is open.  The fold costs the scan instances 16 to 20 registers, and the fast path, which
// never folds, a block per SM.
struct CatState {
  u8* out;     // the destination
  u64 cap;     // its capacity
  u32 len;     // bytes folded so far (counted past the capacity)
  u32 delim;   // 0x100 | c, 0 = none
  u32 gmask;   // the lanes of the group
};
struct NoCat {};

// the string-append copies stay out of line: they run once per operand, and inlined at every visit they cost the
// walks' registers
// n bytes of src, reversed, at out + at .. (the bytes below cap), then the delimiter byte (0x100 | c; 0 = none)
__device__ __noinline__ void cat_put_reversed(u8* out, u64 cap, u64 at, const u8* src, u32 n, u32 delim, u32 gmask) {
  const u32 lanes = __popc(gmask), lane = __popc(gmask & ((1u << (threadIdx.x & 31u)) - 1u));
  for (u32 b = lane; b < n; b += lanes) {
    const u64 p = at + n - 1u - b;
    if (p < cap) out[p] = __ldcg(src + b);
  }
  if (delim && lane == 0 && at + n < cap) out[at + n] = (u8)delim;
}
// reverse out[0 .. len) in place, after every lane of the group has written its bytes
__device__ __noinline__ void cat_reverse(u8* out, u32 len, u32 gmask) {
  const u32 lanes = __popc(gmask), lane = __popc(gmask & ((1u << (threadIdx.x & 31u)) - 1u));
  __syncwarp(gmask);
  for (u32 i = lane; i < len / 2u; i += lanes) {
    const u8 x = out[i];
    out[i] = out[len - 1u - i];
    out[len - 1u - i] = x;
  }
  __syncwarp(gmask);
}

template <bool CAT>
struct Acc : std::conditional_t<CAT, CatState, NoCat> {  // (a base: NoCat takes no room)
  u32 n_ops, n_bad;
  u64 sum;             // wrapping sum of the 8-byte operands seen so far
  const u8* last_ptr;  // oldest operand seen so far
  u32 last_len;
  u32 merge_op;
  // result
  bool done, imm;
  i32 status;
  u32 msg;
  const u8* res_ptr;   // (string append: == cat().out, the value is already in place)
  u32 res_len;
  u64 res_imm;
  __device__ void init(u32 op, u32 delim) {
    n_ops = n_bad = 0; sum = 0; last_ptr = nullptr; last_len = 0; merge_op = op;
    done = false; imm = false; status = 1; msg = 0; res_ptr = nullptr; res_len = 0; res_imm = 0;
    if constexpr (CAT) { cat().out = nullptr; cat().cap = 0; cat().len = 0; cat().delim = delim; cat().gmask = 0; }
  }
  __device__ CatState& cat() { return *this; }
  __device__ void set_out(u8* out, u64 cap, u32 gmask) {
    if constexpr (CAT) { cat().out = out; cat().cap = cap; cat().gmask = gmask; }
  }
  __device__ bool in_place(const u8* dst) const {
    if constexpr (CAT) return res_ptr == dst;
    return false;
  }
  __device__ void fail(i32 st, u32 m) { status = st; msg = m; done = true; }
  // string append: n bytes at src, reversed, at the end of the fold (an operand: and the delimiter after them)
  __device__ void cat_piece(const u8* src, u32 n, bool operand) {
    if constexpr (CAT) {
      const u32 d = operand ? cat().delim : 0u;
      if (cat().len < cat().cap) cat_put_reversed(cat().out, cat().cap, cat().len, src, n, d, cat().gmask);
      cat().len += n + (d ? 1u : 0u);
    }
  }
  __device__ void cat_finish(const u8* base, u32 base_len) {
    if constexpr (CAT) {
      if (base) cat_piece(base, base_len, false);
      else if (cat().delim) cat().len--;  // no existing value: the oldest operand's delimiter goes
      status = 0; res_ptr = cat().out; res_len = cat().len;
      if (cat().len <= cat().cap) cat_reverse(cat().out, cat().len, cat().gmask);
    }
  }
  // fold the collected operands onto `base` (nullptr = no existing value)
  __device__ void finish(const u8* base, u32 base_len) {
    done = true;
    if constexpr (CAT) {
      if (merge_op == MERGE_OP_STRING_APPEND) return cat_finish(base, base_len);
    }
    if (merge_op == 1) {  // RSP_MERGE_COUNTER
      if (base) {
        if (base_len != 8 || n_bad) return fail(2, MSG_MERGE_FAILED);
        res_imm = sum + ldcg64(base);
      } else if (n_ops == 1) {  // existing == nullptr -> the operand itself, any size
        status = 0; res_ptr = last_ptr; res_len = last_len;
        return;
      } else {
        if (n_bad) return fail(2, MSG_MERGE_FAILED);
        res_imm = sum;
      }
    } else {  // RSP_MERGE_UINT64ADD: malformed operands count as 0
      res_imm = sum + ((base && base_len == 8) ? ldcg64(base) : 0ull);
    }
    status = 0; imm = true; res_len = 8;
  }
  // one version, newest first.  returns done.
  __device__ bool visit(u32 type, const u8* vptr, u32 vlen) {
    if (type == kTypeValue) {
      if (n_ops == 0) { status = 0; res_ptr = vptr; res_len = vlen; done = true; }
      else finish(vptr, vlen);
    } else if (type == kTypeMerge) {
      if (merge_op == 0) fail(4, MSG_MERGE_NOT_INIT);
      else if (CAT && merge_op == MERGE_OP_STRING_APPEND) { cat_piece(vptr, vlen, true); n_ops++; }
      else if (merge_op > 2) fail(ST_NEED_HOST_MERGE, 0);
      else {
        n_ops++;
        if (vlen == 8) sum += ldcg64(vptr); else n_bad++;
        last_ptr = vptr; last_len = vlen;
      }
    } else {  // Delete / SingleDelete
      if (n_ops == 0) { status = 1; done = true; }
      else finish(nullptr, 0);
    }
    return done;
  }
  __device__ void end_of_versions() {
    if (done) return;
    if (n_ops) finish(nullptr, 0);
    else { status = 1; done = true; }
  }
};

// ---- version walk over one shard ---------------------------------------------------------------------
// V: visitor with bool visit(u32 type, const u8* vptr, u32 vlen) (true = stop).
template <u32 G, class V>
__device__ __forceinline__ void walk_memtable(const ShardDev* sd, const u8* kp, u32 klen, u64 h, u64 snap,
                                              u32 lane, u32 gmask, u32 gbase, V& v) {
  const u64* slots = sd->mt_slots;
  const u8* heap = sd->mt_heap;
  const u32 mask = sd->mt_slot_mask;
  const u32 tag = hash_tag32(h);
  u32 idx = (u32)h & mask;
  for (u32 probes = 0; probes <= mask; probes += G) {
    const u64 sv = ldcg64(slots + ((idx + lane) & mask));
    const u32 empty_m = (__ballot_sync(gmask, sv == 0) >> gbase) & ((1u << G) - 1u);
    u32 match_m = (__ballot_sync(gmask, (u32)(sv >> 32) == tag && sv != 0) >> gbase) & ((1u << G) - 1u);
    const u32 first_empty = empty_m ? (u32)(__ffs(empty_m) - 1) : G;
    match_m &= (first_empty >= 32u) ? 0xffffffffu : ((1u << first_empty) - 1u);
    while (match_m) {
      const u32 m = (u32)(__ffs(match_m) - 1);
      match_m &= match_m - 1;
      u32 c = (u32)__shfl_sync(gmask, (u32)sv, gbase + m);
      const u8* he = heap + (u64)(c - 1u) * 16u;
      const u32 hklen = ldcg32(he + 8);
      if (!eq_key_vs_padded_cg(kp, klen, reinterpret_cast<const u64*>(he + 32), hklen)) continue;
      // my key: walk the chain newest -> oldest, skipping versions newer than the published snapshot
      while (c) {
        const u8* e = heap + (u64)(c - 1u) * 16u;
        const uint4 hd = __ldcg(reinterpret_cast<const uint4*>(e));
        const u64 st = ((u64)hd.y << 32) | hd.x;
        if ((st >> 8) <= snap) {
          if (v.visit((u32)(st & 0xffu), e + 32u + 16u * units_of(hd.z), hd.w)) return;
        }
        c = ldcg32(e + 16);
      }
      return;  // chain exhausted, older versions live in the runs
    }
    if (empty_m) return;
    idx = (idx + G) & mask;
  }
}

__device__ __forceinline__ const u8* run_entry(const RunDev& r, u32 ord) {
  const u32 unit = r.uniform_units ? ord * r.uniform_units : __ldg(r.ent_off + ord);
  return r.heap + (u64)unit * 16u;
}

template <u32 G, class V>
__device__ __forceinline__ bool walk_run(const RunDev& r, const u8* kp, u32 klen, u64 h, u32 lane, u32 gmask,
                                         u32 gbase, V& v) {
  if (r.n_ent == 0) return false;
  const u32 tag = (u32)(h >> 32) >> r.ord_bits;
  const u32 ord_mask = (1u << r.ord_bits) - 1u;
  u32 bucket = (u32)(((u64)(u32)h * r.n_buckets) >> 32);
  for (u32 nb = 0; nb < r.n_buckets; nb++) {
    // one 32-byte sector of slots per bucket; with G < 8 lanes each lane covers several slots
    u32 sv[RUN_BUCKET_SLOTS / G > 0 ? RUN_BUCKET_SLOTS / G : 1];
    bool any_empty = false;
#pragma unroll
    for (u32 i = 0; i < RUN_BUCKET_SLOTS / G; i++) {
      sv[i] = __ldg(r.hslots + (u64)bucket * RUN_BUCKET_SLOTS + i * G + lane);
      any_empty |= sv[i] == 0;
    }
    const bool grp_empty = __ballot_sync(gmask, any_empty) != 0;
#pragma unroll
    for (u32 i = 0; i < RUN_BUCKET_SLOTS / G; i++) {
      u32 match_m = (__ballot_sync(gmask, sv[i] != 0 && (sv[i] >> r.ord_bits) == tag) >> gbase) & ((1u << G) - 1u);
      while (match_m) {
        const u32 m = (u32)(__ffs(match_m) - 1);
        match_m &= match_m - 1;
        u32 ord = (__shfl_sync(gmask, sv[i], gbase + m) & ord_mask) - 1u;
        const u8* e = run_entry(r, ord);
        uint4 hd = __ldg(reinterpret_cast<const uint4*>(e));
        if (!eq_key_vs_padded(kp, klen, reinterpret_cast<const u64*>(e + 16), hd.z)) continue;
        // first (newest) version of my key in this run; older versions follow in sort order
        for (;;) {
          if (v.visit(hd.x & 0xffu, e + 16u + 16u * units_of(hd.z), hd.w)) return true;
          if (++ord >= r.n_ent) return true;
          e = run_entry(r, ord);
          hd = __ldg(reinterpret_cast<const uint4*>(e));
          if (!eq_key_vs_padded(kp, klen, reinterpret_cast<const u64*>(e + 16), hd.z)) return true;
        }
      }
    }
    if (grp_empty) return false;
    bucket = bucket + 1 == r.n_buckets ? 0 : bucket + 1;
  }
  return false;
}

// the sorted runs newest first, until the visitor is done.  n_runs is read before each run: a caller that wants it read
// once passes a local copy.
template <u32 G, class V>
__device__ __forceinline__ void walk_runs(const RunDev* runs, const u32& n_runs, const u8* kp, u32 klen, u64 h, u32 lane,
                                          u32 gmask, u32 gbase, V& v) {
  for (u32 ri = 0; ri < n_runs && !v.done; ri++) walk_run<G>(runs[ri], kp, klen, h, lane, gmask, gbase, v);
}

// the memtable, then the sorted runs; the walk stops right after the visit that finishes
template <u32 G, class V>
__device__ __forceinline__ void walk_shard(const ShardDev* sd, const u8* kp, u32 klen, u32 lane, u32 gmask,
                                           u32 gbase, V& v) {
  const u64 h = hash_key(kp, klen);
  const u64 snap = ldcg64(&sd->pub_seq);
  if (ldcg32(&sd->mt_count) != 0) {
    walk_memtable<G>(sd, kp, klen, h, snap, lane, gmask, gbase, v);
    if (v.done) return;
  }
  const u32 n_runs = sd->n_runs;
  for (u32 ri = 0; ri < n_runs; ri++) {
    walk_run<G>(sd->runs[ri], kp, klen, h, lane, gmask, gbase, v);
    if (v.done) return;
  }
}

// ------------------------------------------------------------------------------------------------
// k_multi_get
// ------------------------------------------------------------------------------------------------
constexpr u32 MG_LANES = 8;

__device__ __forceinline__ void group_copy_out(u8* dst, const u8* src, u32 n, u32 lane, u32 lanes) {
  if ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0) {
    const u32 full = n >> 4;
    for (u32 u = lane; u < full; u += lanes)
      reinterpret_cast<uint4*>(dst)[u] = __ldcg(reinterpret_cast<const uint4*>(src) + u);
    for (u32 b = (full << 4) + lane; b < n; b += lanes) dst[b] = src[b];
  } else {
    for (u32 b = lane; b < n; b += lanes) dst[b] = src[b];
  }
}

// The eight-lane lookups of k_multi_get / k_multi_get_pending (GetArgs) and k_multi_get_at (GetAtArgs) share these
// steps; both argument structs name the key and result fields alike.
template <class Args>
__device__ __forceinline__ const u8* lookup_key(const Args& a, u32 q, u32& klen) {
  if (a.klen_fixed) {
    klen = a.klen_fixed;
    return a.keys + (u64)q * klen;
  }
  const u64 o = __ldg(a.koff + q);
  klen = (u32)(__ldg(a.koff + q + 1) - o);
  return a.keys + o;
}

// an unknown or closed shard, or a null, released or foreign snapshot: InvalidArgument
template <class Args>
__device__ __forceinline__ void answer_invalid(const Args& a, u32 q, u32 lane) {
  if (lane == 0) {
    a.st[q] = 4;
    a.vlen[q] = 0;
    if (a.n_special) atomicAdd(a.n_special, 1u);
  }
}

// status, value and value length (the message id for error statuses) of a walk that has seen every version it needs
template <class Args, bool CAT>
__device__ __forceinline__ void answer(const Args& a, u32 q, u32 lane, Acc<CAT>& acc) {
  acc.end_of_versions();
  i32 st = acc.status;
  const u32 msg = acc.msg;
  u32 vlen = 0;
  if (st == 0) {
    vlen = acc.res_len;
    if ((u64)vlen > a.val_stride) {
      st = 7;  // RSP_INCOMPLETE: vlen reports the size needed
    } else {
      u8* dst = a.vals + (u64)q * a.val_stride;
      if (acc.imm) {
        if (lane == 0) {
#pragma unroll
          for (u32 b = 0; b < 8; b++) dst[b] = (u8)(acc.res_imm >> (8u * b));
        }
      } else if (!acc.in_place(dst)) {  // (a string-append fold is already there)
        group_copy_out(dst, acc.res_ptr, vlen, lane, MG_LANES);
      }
    }
  } else if (st != 1 && st != ST_NEED_HOST_MERGE) {
    vlen = msg;  // message id rides in vlen for error statuses
  }
  if (lane == 0) {
    a.st[q] = st;
    a.vlen[q] = vlen;
    if (st != 0 && st != 1 && st != 7 && a.n_special) atomicAdd(a.n_special, 1u);
  }
}

// generic path: any key length, any entry shape, memtable chains, merges, multiple runs
template <bool CAT>
__device__ __noinline__ void lookup_generic(const GetArgs& a, u32 q, u32 lane, u32 gmask, u32 gbase) {
  const u32 six = __ldg(a.shard_ix + q);
  if (six >= a.max_shards || !a.shards[six].live) return answer_invalid(a, q, lane);
  const ShardDev* sd = a.shards + six;
  u32 klen;
  const u8* kp = lookup_key(a, q, klen);
  Acc<CAT> acc;
  acc.init(sd->merge_op, sd->merge_delim);
  acc.set_out(a.vals + (u64)q * a.val_stride, a.val_stride, gmask);
  walk_shard<MG_LANES>(sd, kp, klen, lane, gmask, gbase, acc);
  answer(a, q, lane, acc);
}

template <bool CAT>
__global__ void __launch_bounds__(256) k_multi_get(GetArgs a) {
  const u32 q = (blockIdx.x * blockDim.x + threadIdx.x) / MG_LANES;
  const u32 lane = threadIdx.x & (MG_LANES - 1);
  const u32 gbase = (threadIdx.x & 31u) & ~(MG_LANES - 1u);
  const u32 gmask = ((1u << MG_LANES) - 1u) << gbase;
  if (q >= a.n) return;
  lookup_generic<CAT>(a, q, lane, gmask, gbase);
}

// Tried and dropped: hash-addressed entry slots instead of the index, and software prefetch of later lookups' sectors
// (both slower than the index probe below).
// ---- the hot kernels: 16-byte keys, TWO lanes per lookup, three dependent memory round trips ----------
//   1. shard id + query key (coalesced across the warp) and the 32-byte ShardFast descriptor
//      (32 B x #shards: L1/L2-resident); both lanes load the same words (one broadcast transaction)
//   2. the hash bucket: one 32-byte sector of run 0's index, four u32 slots (one 16-byte load) per lane
//      (when the memtable is not empty: eight u64 memtable slots first, four per lane)
//   3. the entry: both lanes read the header and key units (same sector, broadcast) and decide alike with
//      no shuffles; lane L then moves value units L, L+2, .. straight from its registers to the output
//      (2 lanes x 2 x 16 B = the 64-byte value)
// The kernels are issue-bound before they are HBM-bound, so the lane count per lookup is what the instruction
// budget allows: 8 lanes cost ~70 warp instructions per lookup, 2 lanes ~1/4 of that.
// Tag false positives and probes that spill past a full home bucket (wrapping at the last bucket) are served here
// too.  Anything else — a memtable window with two tag matches or no empty slot, Delete / Merge, version chains,
// several runs (k_multi_get16), entries of 255 units or more, values beyond the template's size — is appended to the
// pending list and served by the generic path (k_multi_get_pending).
static_assert(offsetof(ShardDev, mt_slot_mask) == 24 && offsetof(ShardDev, pub_seq) == 56, "ShardDev units 0-3");
static_assert(sizeof(ShardFast) == 32, "ShardFast");

constexpr u32 FL = 2;  // lanes per lookup
// 20 blocks of 64 threads per SM leave 48 registers per thread.  At 24 blocks (40 registers) ptxas for sm_90a spills
// k_multi_get16<false> to local memory (60 bytes per thread), and the launch of 8.4 M lookups takes 1.04 ms instead of
// 0.91 ms on an H100 80GB HBM3 at a 400 W power limit: the spill traffic costs more than the extra lookups in flight buy.
constexpr u32 MG16_THREADS = 64;
constexpr u32 MG16_MIN_BLOCKS = 20;

// L2 residency control (createpolicy + ld .L2::cache_hint): the hash-index sectors are the only data with reuse
// across lookups (80 MB at 10 M keys against a 50 MB L2), so they are loaded evict_last; entries, query keys and
// results stream through once.
__device__ __forceinline__ u64 pol_evict_last() {
  u64 p;
#ifdef RSP_EMUL  // tests/emul: cache policies have no meaning on the CPU
  p = 0;
#else
  asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
#endif
  return p;
}
__device__ __forceinline__ uint4 ldg_pol(const uint4* p, u64 pol) {
  uint4 v;
#ifdef RSP_EMUL
  (void)pol;
  v = *p;
#else
  asm("ld.global.nc.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
      : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p), "l"(pol));
#endif
  return v;
}

// Candidate entry at `ent`: header unit 0, key unit KU, value units KU+1.. (U units in all).  CG: a memtable entry
// (read through L2, its size known only from its header), otherwise a run entry.
// Returns 0 = served, 1 = not my key (tag false positive), 2 = needs the generic path.
template <bool CG>
__device__ __forceinline__ uint4 ld_entry_unit(const uint4* p) {
  if (CG) return __ldcg(p);
  return __ldg(p);
}
template <bool CG, bool BIG>
__device__ __forceinline__ u32 fast_entry(const u8* ent, u32 U, u32 KU, const uint4& kq, u64 snap, u8* dst,
                                          u64 val_stride, u32 lane, u32& vlen_out) {
  const uint4* ep = reinterpret_cast<const uint4*>(ent);
  const uint4 hd = ld_entry_unit<CG>(ep);
  const uint4 ek = ld_entry_unit<CG>(ep + KU);
  const u32 fv = KU + 1;  // first value unit; lane L owns value units L, L+2, L+4, ...
  uint4 v0 = make_uint4(0, 0, 0, 0), v1 = v0, v2 = v0;
  if (!CG) {
    // a run: the entry size U is known before the header arrives, so the first six value units are
    // requested together with header and key (one round trip for values up to 96 bytes)
    if (fv + lane < U) v0 = ld_entry_unit<CG>(ep + fv + lane);
    if (fv + lane + 2 < U) v1 = ld_entry_unit<CG>(ep + fv + lane + 2);
    if (fv + lane + 4 < U) v2 = ld_entry_unit<CG>(ep + fv + lane + 4);
  }
  if (ek.x != kq.x || ek.y != kq.y || ek.z != kq.z || ek.w != kq.w || hd.z != 16) return 1;
  const u64 seq = (((u64)hd.y << 32) | hd.x) >> 8;
  const u32 vu = (hd.w + 15u) >> 4;
  if ((hd.x & 0xffu) != kTypeValue || seq > snap || (!CG && fv + vu > U) || (u64)vu * 16u > val_stride || (!BIG && vu > 6)) return 2;
  uint4* out = reinterpret_cast<uint4*>(dst);
  if (CG) {
    // the memtable: the entry's size is only known from its header, so the value follows in a second trip
    for (u32 u = lane; u < vu; u += FL) out[u] = ld_entry_unit<CG>(ep + fv + u);
  } else {
    if (lane < vu) out[lane] = v0;
    if (lane + 2 < vu) out[lane + 2] = v1;
    if (lane + 4 < vu) out[lane + 4] = v2;
    if (BIG)
      for (u32 u = lane + 6; u < vu; u += FL) out[u] = ld_entry_unit<CG>(ep + fv + u);  // values > 96 bytes
  }
  vlen_out = hd.w;
  return 0;
}

// One sorted run through its hash index: g0/g1 are the run's 32-byte descriptor in ShardFast's layout (heap pointer,
// index pointer, bucket count, meta).  One bucket = one 32-byte sector, four slots per lane.  Walks the tag matches in
// probe order; a false positive (18-bit tags at 16 K entries: ~1 per 60 K lookups) just moves on to the next
// candidate, a full bucket to the next bucket.  Returns 0 = served, 2 = generic path, 4 = not in this run.
template <bool BIG>
__device__ __forceinline__ u32 probe_one_run(const uint4& g0, const uint4& g1, const uint4& kq, u64 h, u8* dst, u64 val_stride,
                                             u32 lane, u32 pmask, u32 pbase, u32& vlen) {
  const u8* heap = reinterpret_cast<const u8*>(((u64)g0.y << 32) | g0.x);
  const u32 n_buckets = g1.x, ord_bits = g1.y & 0xffu, U = (g1.y >> FAST_META_UNITS_SHIFT) & 0xffu;
  if (U == 0 || U >= 255) return 2;
  const uint4* hs = reinterpret_cast<const uint4*>(((u64)g0.w << 32) | g0.z);
  u32 bucket = (u32)(((u64)(u32)h * n_buckets) >> 32);
  const u32 tag = (u32)(h >> 32) >> ord_bits;
  u32 m8 = 0, e8 = 1, probe = 0;  // e8 != 0 before the first load only so that the loop loads first
  uint4 sv = make_uint4(0, 0, 0, 0);
#pragma unroll 1
  for (;;) {
    if (!m8) {
      if (probe && e8) return 4;           // an empty slot ends the probe: not here
      if (probe == n_buckets) return 4;    // (a table without an empty slot)
      if (probe) bucket = bucket + 1 == n_buckets ? 0 : bucket + 1;
      probe++;
      sv = ldg_pol(hs + (u64)bucket * 2u + lane, pol_evict_last());
      const u32 m = ((sv.x && (sv.x >> ord_bits) == tag) ? 1u : 0u) | ((sv.y && (sv.y >> ord_bits) == tag) ? 2u : 0u) |
                    ((sv.z && (sv.z >> ord_bits) == tag) ? 4u : 0u) | ((sv.w && (sv.w >> ord_bits) == tag) ? 8u : 0u);
      const u32 e = (sv.x == 0 || sv.y == 0 || sv.z == 0 || sv.w == 0) ? 1u : 0u;
      const u32 mine = m | (e << 4);
      const u32 other = __shfl_xor_sync(pmask, mine, 1);
      m8 = lane ? ((other & 15u) | ((mine & 15u) << 4)) : ((mine & 15u) | ((other & 15u) << 4));
      e8 = (mine | other) >> 4;
      if (!m8) continue;
    }
    const u32 p = __ffs(m8) - 1;
    m8 &= m8 - 1;
    const u32 pick = (p & 2u) ? ((p & 1u) ? sv.w : sv.z) : ((p & 1u) ? sv.y : sv.x);
    const u32 val = __shfl_sync(pmask, pick, pbase + (p >> 2));
    // run entry: unit0 header, unit1 key, units 2.. value
    const u32 r = fast_entry<false, BIG>(heap + (u64)((val & ((1u << ord_bits) - 1u)) - 1u) * U * 16u, U, 1, kq, ~0ull, dst,
                                         val_stride, lane, vlen);
    if (r == 0) return 0;
    if (r == 2) return 2;
  }
}

// One lookup of the 16-byte-key kernels.  MULTI = false (k_multi_get16): a shard with several sorted runs takes the
// pending list.  MULTI = true (k_multi_get16m, for engines where some shard has several runs, between a flush and the
// next merge): the runs are walked newest first, a run that does not hold the key hands over to the next older one
// (per-run descriptors behind the ShardFast array).  The two stay separate kernels and the host picks one per launch:
// one kernel with a runtime choice between them changes k_multi_get16's register allocation at the same instruction mix.
// BIG = false: values up to 96 bytes (larger ones take the pending list); BIG = true adds the tail loop for
// larger values at the price of a few registers — the host picks by the caller's value stride.
template <bool BIG, bool MULTI>
__device__ __forceinline__ void multi_get16(GetArgs a) {
  const u32 q = (blockIdx.x * blockDim.x + threadIdx.x) / FL;
  const u32 lane = threadIdx.x & (FL - 1);
  const u32 pbase = (threadIdx.x & 31u) & ~1u;
  const u32 pmask = 3u << pbase;  // the two lanes of this lookup always branch together
  if (q >= a.n) return;
  // (1)
  u32 six = __ldg(a.shard_ix + q);
  const bool bad_shard = six >= a.max_shards;
  if (bad_shard) six = 0;
  const uint4 kq = __ldg(reinterpret_cast<const uint4*>(a.keys) + q);
  const uint4 f0 = __ldg(reinterpret_cast<const uint4*>(a.fast + six));
  const uint4 f1 = __ldg(reinterpret_cast<const uint4*>(a.fast + six) + 1);
  const u32 n_runs = (f1.y >> FAST_META_RUNS_SHIFT) & 0xffu;
  const u64 k0 = ((u64)kq.y << 32) | kq.x, k1 = ((u64)kq.w << 32) | kq.z;
  const u64 h = hash_final(hash_step(hash_step(hash_init(16), k0), k1));
  u8* dst = a.vals + (u64)q * a.val_stride;
  u32 state = 3;  // 0 served, 2 generic path, 3 undecided, 4 not found
  u32 vlen = 0;
  if ((!MULTI && n_runs > 1) || ((a.val_stride | reinterpret_cast<uintptr_t>(a.vals)) & 15u) || bad_shard || !(f1.y & FAST_META_LIVE)) state = 2;
  bool in_mem = false;
  if (state == 3 && f1.z /* mt_count */) {
    // the shard's memtable filter (L2-resident, behind the descriptors): a clear bit = the key is not in the memtable
    const u32 fb = mt_filter_bit(h);
    const u32 fw = __ldcg(reinterpret_cast<const u32*>(a.fast + (size_t)a.max_shards * (1u + RSP_MAX_RUNS)) + (size_t)six * MT_FILTER_WORDS + (fb >> 5));
    in_mem = (fw >> (fb & 31u)) & 1u;
  }
  if (in_mem) {
    // ---- (2) memtable: eight u64 slots from the home position, four per lane; descriptor through L2
    const uint4* dp = reinterpret_cast<const uint4*>(a.shards + six);
    const uint4 d0 = __ldcg(dp), d1 = __ldcg(dp + 1), d3 = __ldcg(dp + 3);
    const u8* heap = reinterpret_cast<const u8*>(((u64)d0.y << 32) | d0.x);
    const u64* sp = reinterpret_cast<const u64*>(((u64)d0.w << 32) | d0.z);
    const u32 mask = d1.z;
    const u64 snap = ((u64)d3.w << 32) | d3.z;
    const u32 tag = hash_tag32(h);
    u32 cand = 0, info = 0;  // info: matches | (position of my first empty + 1) << 8
#pragma unroll
    for (u32 i = 0; i < 4; i++) {
      const u64 sv = ldcg64(sp + (((u32)h + 4u * lane + i) & mask));
      if (sv == 0) { if (!(info >> 8)) info |= (4u * lane + i + 1u) << 8; }
      else if ((u32)(sv >> 32) == tag && !(info >> 8)) { if (!cand) cand = (u32)sv; info++; }
    }
    const u32 o_cand = __shfl_xor_sync(pmask, cand, 1), o_info = __shfl_xor_sync(pmask, info, 1);
    // lane 1's slots come after lane 0's in probe order: they count only if lane 0 saw no empty slot
    const u32 lo_info = lane ? o_info : info, hi_info = lane ? info : o_info;
    const u32 lo_cand = lane ? o_cand : cand, hi_cand = lane ? cand : o_cand;
    const bool lo_empty = (lo_info >> 8) != 0;
    const u32 n_match = (lo_info & 0xffu) + (lo_empty ? 0u : (hi_info & 0xffu));
    const bool any_empty = lo_empty || (hi_info >> 8) != 0;
    if (n_match == 1) {
      const u32 c = (lo_info & 0xffu) ? lo_cand : hi_cand;
      // memtable entry: unit0 header, unit1 link, unit2 key, units 3.. value
      const u32 r = fast_entry<true, BIG>(heap + (u64)(c - 1u) * 16u, 7, 2, kq, snap, dst, a.val_stride, lane, vlen);
      state = r == 0 ? 0 : 2;
    } else if (n_match > 1 || !any_empty) {
      state = 2;
    }
  }
  if (state == 3) {
    // (2), (3): the sorted runs, newest first
    state = 4;
    for (u32 r = 0; r < n_runs; r++) {
      uint4 g0 = f0, g1 = f1;
      if (MULTI && r) {
        const uint4* fr = reinterpret_cast<const uint4*>(a.fast + a.max_shards) + ((u64)six * RSP_MAX_RUNS + r) * 2u;
        g0 = __ldg(fr);
        g1 = __ldg(fr + 1);
      }
      const u32 rs = probe_one_run<BIG>(g0, g1, kq, h, dst, a.val_stride, lane, pmask, pbase, vlen);
      if (rs != 4 || !MULTI) { state = rs; break; }
    }
  }
  if (lane == 0) {
    if (state == 2) {
      a.pending[atomicAdd(a.n_pending + a.parity, 1u)] = q;
    } else {
      a.st[q] = state == 0 ? 0 : 1;
      a.vlen[q] = vlen;
    }
  }
}

template <bool BIG>
__global__ void __launch_bounds__(MG16_THREADS, MG16_MIN_BLOCKS) k_multi_get16(GetArgs a) { multi_get16<BIG, false>(a); }
template <bool BIG>
__global__ void __launch_bounds__(MG16_THREADS, MG16_MIN_BLOCKS) k_multi_get16m(GetArgs a) { multi_get16<BIG, true>(a); }

// generic path over the queries the fast kernel deferred; a small fixed grid strides over the list
template <bool CAT>
__global__ void __launch_bounds__(256) k_multi_get_pending(GetArgs a) {
  const u32 lane = threadIdx.x & (MG_LANES - 1);
  const u32 gbase = (threadIdx.x & 31u) & ~(MG_LANES - 1u);
  const u32 gmask = ((1u << MG_LANES) - 1u) << gbase;
  const u32 n = __ldcg(a.n_pending + a.parity);
  const u32 groups = gridDim.x * (blockDim.x / MG_LANES);
  for (u32 i = (blockIdx.x * blockDim.x + threadIdx.x) / MG_LANES; i < n; i += groups)
    lookup_generic<CAT>(a, __ldcg(a.pending + i), lane, gmask, gbase);
}

bool launch_multi_get(const GetArgs& a, bool cat, cudaStream_t s) {
  if (!a.n) return false;
  const u32 per_block = 256 / MG_LANES;
  const u32 grid = (a.n + per_block - 1) / per_block;
  if (a.klen_fixed == 16 && (reinterpret_cast<uintptr_t>(a.keys) & 15u) == 0 && a.pending && a.fast) {
    // this launch counts in n_pending[parity]; a memset node clears it (clearing the other parity's counter inside
    // the kernel instead is slower end to end)
    cudaMemsetAsync(a.n_pending + a.parity, 0, 4, s);
    const u32 g16 = (a.n + MG16_THREADS / FL - 1) / (MG16_THREADS / FL);
    const bool multi = a.multirun != 0;
    if (a.val_stride > 96) {
      if (multi) k_multi_get16m<true><<<g16, MG16_THREADS, 0, s>>>(a); else k_multi_get16<true><<<g16, MG16_THREADS, 0, s>>>(a);
    } else {
      if (multi) k_multi_get16m<false><<<g16, MG16_THREADS, 0, s>>>(a); else k_multi_get16<false><<<g16, MG16_THREADS, 0, s>>>(a);
    }
    if (cat) k_multi_get_pending<true><<<std::min<u32>(grid, DEVICE_SMS), 256, 0, s>>>(a);
    else k_multi_get_pending<false><<<std::min<u32>(grid, DEVICE_SMS), 256, 0, s>>>(a);
    return true;
  }
  if (cat) k_multi_get<true><<<grid, 256, 0, s>>>(a);
  else k_multi_get<false><<<grid, 256, 0, s>>>(a);
  return false;
}

// ------------------------------------------------------------------------------------------------
// k_get_versions — slow path for host-folded merge operators: dump the version stack
// ------------------------------------------------------------------------------------------------
struct DumpVisitor {
  u8* out;
  u64 cap;
  u32 used, n_rec;
  bool done;
  __device__ bool visit(u32 type, const u8* vptr, u32 vlen) {
    const u32 rec = 8u + ((vlen + 3u) & ~3u);
    if ((u64)used + rec <= cap) {
      *reinterpret_cast<u32*>(out + used) = type;
      *reinterpret_cast<u32*>(out + used + 4) = vlen;
      for (u32 b = 0; b < vlen; b++) out[used + 8 + b] = __ldcg(vptr + b);
      n_rec++;
    }
    used += rec;
    if (type != kTypeMerge) done = true;
    return done;
  }
};

__global__ void k_get_versions(VersionsArgs a) {
  const u32 q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= a.n) return;
  const u32 lane_in_warp = threadIdx.x & 31u;
  const ShardDev* sd = a.views ? nullptr : a.shards + a.shard_ix[q];
  const u64 o = a.koff[q];
  const u32 klen = (u32)(a.koff[q + 1] - o);
  DumpVisitor v{a.out + (u64)q * a.out_stride, a.out_stride, 0, 0, false};
  if (a.views) {  // a pinned iterator snapshot: sorted runs only
    const ScanView& vw = a.views[q];
    const u64 h = hash_key(a.keys + o, klen);
    walk_runs<1>(vw.runs, vw.n_runs, a.keys + o, klen, h, 0, 1u << lane_in_warp, lane_in_warp, v);
  } else {
    walk_shard<1>(sd, a.keys + o, klen, 0, 1u << lane_in_warp, lane_in_warp, v);
  }
  a.n_rec[q] = v.n_rec;
  a.need[q] = v.used;
}

void launch_get_versions(const VersionsArgs& a, cudaStream_t s) {
  if (!a.n) return;
  k_get_versions<<<(a.n + 63) / 64, 64, 0, s>>>(a);
}

// ------------------------------------------------------------------------------------------------
// k_multi_get_at — MultiGet at snapshots: the generic eight-lane walk over a pinned view instead of a live shard
// ------------------------------------------------------------------------------------------------
template <bool CAT>
__global__ void __launch_bounds__(256) k_multi_get_at(GetAtArgs a) {
  const u32 q = (blockIdx.x * blockDim.x + threadIdx.x) / MG_LANES;
  const u32 lane = threadIdx.x & (MG_LANES - 1);
  const u32 gbase = (threadIdx.x & 31u) & ~(MG_LANES - 1u);
  const u32 gmask = ((1u << MG_LANES) - 1u) << gbase;
  if (q >= a.n) return;
  const u32 slot = __ldg(a.slot + q);
  if (slot >= a.n_views || !a.views[slot].live) return answer_invalid(a, q, lane);
  const ScanView& vw = a.views[slot];
  u32 klen;
  const u8* kp = lookup_key(a, q, klen);
  Acc<CAT> acc;
  acc.init(vw.merge_op, vw.merge_delim);
  acc.set_out(a.vals + (u64)q * a.val_stride, a.val_stride, gmask);
  const u64 h = hash_key(kp, klen);
  const u32 n_runs = vw.n_runs;
  walk_runs<MG_LANES>(vw.runs, n_runs, kp, klen, h, lane, gmask, gbase, acc);
  answer(a, q, lane, acc);
}

void launch_multi_get_at(const GetAtArgs& a, bool cat, cudaStream_t s) {
  if (!a.n) return;
  const u32 per_block = 256 / MG_LANES;
  const u32 grid = (a.n + per_block - 1) / per_block;
  if (cat) k_multi_get_at<true><<<grid, 256, 0, s>>>(a);
  else k_multi_get_at<false><<<grid, 256, 0, s>>>(a);
}

// ------------------------------------------------------------------------------------------------
// k_multi_scan — Seek + N x Next/Prev over the sorted runs (one warp per scan)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int cmp_run_key(const RunDev& r, u32 ord, const u8* kp, u32 klen) {
  const u8* e = run_entry(r, ord);
  const u32 eklen = __ldg(reinterpret_cast<const u32*>(e) + 2);
  return -cmp_key_vs_padded(kp, klen, reinterpret_cast<const u64*>(e + 16), eklen);  // sign of (entry - key)
}
// first ordinal whose key is >= key (strict: > key)
__device__ u32 run_lower_bound(const RunDev& r, const u8* kp, u32 klen, bool strict) {
  u32 lo = 0, hi = r.n_ent;
  // block index first: 8-byte big-endian prefixes of every RSP_BLOCK_ENTRIES-th entry
  if (r.n_blocks > 1 && klen) {
    const u64 pfx = key_prefix_be(kp, klen);
    u32 bl = 0, bh = r.n_blocks;  // last block whose first prefix < pfx bounds the answer from below
    while (bl < bh) {
      const u32 m = (bl + bh) >> 1;
      if (__ldg(r.blk_pfx + m) < pfx) bl = m + 1; else bh = m;
    }
    lo = bl ? (bl - 1) * RSP_BLOCK_ENTRIES : 0;
    // first block whose prefix > pfx bounds it from above
    u32 cl = bl, ch = r.n_blocks;
    while (cl < ch) {
      const u32 m = (cl + ch) >> 1;
      if (__ldg(r.blk_pfx + m) <= pfx) cl = m + 1; else ch = m;
    }
    hi = min(r.n_ent, cl * RSP_BLOCK_ENTRIES);
  }
  while (lo < hi) {
    const u32 m = (lo + hi) >> 1;
    const int c = cmp_run_key(r, m, kp, klen);
    if (c < 0 || (strict && c == 0)) lo = m + 1; else hi = m;
  }
  return lo;
}

struct EntRef {
  const u8* e;
  u32 klen, vlen, type;
  __device__ const u64* key() const { return reinterpret_cast<const u64*>(e + 16); }
  __device__ const u8* val() const { return e + 16u + 16u * units_of(klen); }
};
__device__ __forceinline__ EntRef load_ent(const RunDev& r, u32 ord) {
  EntRef x;
  x.e = run_entry(r, ord);
  const uint4 hd = __ldg(reinterpret_cast<const uint4*>(x.e));
  x.type = hd.x & 0xffu; x.klen = hd.z; x.vlen = hd.w;
  return x;
}

__device__ __forceinline__ void warp_copy_bytes(u8* dst, const u8* src, u32 n, u32 lane) {
  for (u32 b = lane; b < n; b += 32) dst[b] = src[b];
}

// ---- TMA-staged block index + warp-ballot search (Seek on a sorted run) --------------------------------
// The run's block index (8-byte big-endian first-key prefix per RSP_BLOCK_ENTRIES entries) is pulled into
// shared memory with ONE bulk asynchronous copy (cp.async.bulk global -> shared, completion on an mbarrier:
// the TMA engine, SASS UBLKCP) instead of a dependent chain of ~log2(n_blocks) global loads; the warp then
// counts prefixes below / not above the target 32 at a time with ballots, and resolves the final position
// inside the 1-2 candidate blocks by comparing 32 entry keys at once.
// independent loads per lane in the streaming loop: 4 gives 181 M scans/s, the plain loop (one load in flight per
// warp: LDG, STG, LDG, ...) leaves the load latency exposed
#define RSP_SCAN_UNROLL 4
constexpr u32 SCAN_WARPS = 4;
constexpr u32 SCAN_STAGE_PFX = 512;  // prefixes staged per warp (4 KB): runs up to 16 K entries

#ifdef RSP_EMUL
// tests/emul: the bulk copy completes at issue; the mbarrier word counts completed phases
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, u32 bytes, u64* mbar) {
  memcpy(smem_dst, gmem_src, bytes);
  *mbar += 1;
}
__device__ __forceinline__ void mbar_init(u64* mbar, u32) { *mbar = 0; }
__device__ __forceinline__ bool mbar_wait(u64* mbar, u32 parity) {
  while ((*mbar & 1u) == parity) emul_yield();
  return true;
}
#else
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, u32 bytes, u64* mbar) {
  const u32 dst = (u32)__cvta_generic_to_shared(smem_dst);
  const u32 bar = (u32)__cvta_generic_to_shared(mbar);
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(gmem_src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_init(u64* mbar, u32 count) {
  const u32 bar = (u32)__cvta_generic_to_shared(mbar);
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// Bounded wait: try_wait itself blocks for a hardware time slice per attempt, so 2^20 attempts are seconds, not a
// hang.  false = the bulk copy never completed (never seen; the caller then searches the index in global memory).
__device__ __forceinline__ bool mbar_wait(u64* mbar, u32 parity) {
  const u32 bar = (u32)__cvta_generic_to_shared(mbar);
  for (u32 tries = 0; tries < (1u << 20); tries++) {
    u32 ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    if (ok) return true;
  }
  return false;
}
#endif

// warp-cooperative lower bound: first ordinal of R whose key is >= key (strict: > key).  mbar: R's block index is being
// copied into s_pfx by the bulk copy that completes the mbarrier's phase 0 (issued once per scan; later searches find
// the phase complete); nullptr: a run of several blocks is searched in global memory.
__device__ u32 run_lower_bound_warp(const RunDev& R, const u8* kp, u32 klen, bool strict, const u64* s_pfx, u64* mbar,
                                    u32 lane) {
  u32 lo = 0, hi = R.n_ent;
  if (R.n_blocks > 1 && klen) {
    if (!mbar) return run_lower_bound(R, kp, klen, strict);
    const u64 pfx = key_prefix_be(kp, klen);  // (the key's load overlaps the bulk copy)
    if (!__all_sync(0xffffffffu, mbar_wait(mbar, 0))) return run_lower_bound(R, kp, klen, strict);
    u32 n_lt = 0, n_le = 0;
    for (u32 b = 0; b < R.n_blocks; b += 32) {
      const u64 p = b + lane < R.n_blocks ? s_pfx[b + lane] : ~0ull;
      const u32 in = b + lane < R.n_blocks;
      n_lt += __popc(__ballot_sync(0xffffffffu, in && p < pfx));
      n_le += __popc(__ballot_sync(0xffffffffu, in && p <= pfx));
    }
    lo = n_lt ? (n_lt - 1) * RSP_BLOCK_ENTRIES : 0;
    hi = min(R.n_ent, n_le * RSP_BLOCK_ENTRIES);
  }
  // entries [lo, hi) are sorted: the answer is lo + #(entries below the target)
  u32 below = 0;
  for (u32 b = lo; b < hi; b += 32) {
    bool is_below = false;
    if (b + lane < hi) {
      const int c = cmp_run_key(R, b + lane, kp, klen);
      is_below = c < 0 || (strict && c == 0);
    }
    const u32 m = __ballot_sync(0xffffffffu, is_below);
    below += __popc(m);
    if (m != 0xffffffffu) break;  // sorted: once an entry is not below, none after it is
  }
  return lo + below;
}

// BOUNDED: the requests carry end keys (a.ends; the low, for reverse scans); the unbounded instance has none of the
// end-key code.  REVERSE: SeekForPrev + Prev (descending keys); the forward instances have none of the reverse code.
// CAT: the string-append fold (Acc).
template <bool BOUNDED, bool REVERSE, bool CAT>
__device__ __forceinline__ void multi_scan_body(const ScanArgs& a) {
  __shared__ __align__(16) u64 s_pfx_all[SCAN_WARPS][SCAN_STAGE_PFX];
  __shared__ __align__(8) u64 s_mbar[SCAN_WARPS];
  {
    const u32 wi = threadIdx.x >> 5;
    if ((threadIdx.x & 31u) == 0) mbar_init(&s_mbar[wi], 1);
    __syncwarp();
  }
  const u32 q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const u32 lane = threadIdx.x & 31u;
  if (q >= a.n) return;
  const RunDev* runs;
  u32 n_runs, merge_op, merge_delim = 0;
  if (a.flags & SCAN_AT_SLOT) {
    // without a snapshot table (views == nullptr, n_views == 0) every slot is refused
    const u32 slot = a.shard_ix[q];
    if (slot >= a.n_views || !a.views[slot].live) {
      if (lane == 0) { a.n_out[q] = 0; a.st[q] = 4; }  // InvalidArgument, as k_multi_get_at
      return;
    }
    const ScanView& vw = a.views[slot];
    runs = vw.runs; n_runs = vw.n_runs; merge_op = vw.merge_op;
    if constexpr (CAT) merge_delim = vw.merge_delim;
  } else {
    const ShardDev* sd = a.shards + a.shard_ix[q];
    runs = sd->runs; n_runs = sd->n_runs; merge_op = sd->merge_op;
    if constexpr (CAT) merge_delim = sd->merge_delim;
  }
  const u8* kp;
  u32 klen;
  if (a.klen_fixed) { klen = a.klen_fixed; kp = a.keys + (u64)q * klen; }
  else { const u64 o = a.koff[q]; klen = (u32)(a.koff[q + 1] - o); kp = a.keys + o; }
  const bool exclusive = a.flags & SCAN_EXCLUSIVE, extreme = a.flags & SCAN_FROM_EXTREME;
  // the end key: forward scans stop before it, reverse scans before the first key below it
  const bool has_end = BOUNDED;
  const u8* ekp = nullptr;
  u32 eklen = 0;
  if (has_end) {
    if (a.eoff) { const u64 o = a.eoff[q]; eklen = (u32)(a.eoff[q + 1] - o); ekp = a.ends + o; }
    else { eklen = a.elen; ekp = a.ends + (u64)q * eklen; }
  }
  u8* out = a.out + (u64)q * a.out_stride;
  u64 used = 0;
  u32 n_out = 0;
  i32 st = 0;

  // ---- fast path: one fully compacted run of fixed-size Puts.  Seek (block index + binary search), then the warp
  // streams the consecutive entries out as 8-byte words: record i = [u32 klen][u32 vlen][key][value] at
  // out + i * (8 + klen + vlen) is entry start + i (forward) or start - i (reverse, start = the last entry <= key).
  if (n_runs == 1 && (runs[0].flags & RUN_ALL_PUT_FIXED)) {
    const RunDev& R = runs[0];
    const u32 kl = R.kv_len & 0xffffu, vl = R.kv_len >> 16;
    const u32 rec = 8u + kl + vl;
    if ((kl & 15u) == 0 && (vl & 7u) == 0 && ((reinterpret_cast<uintptr_t>(out) | a.out_stride) & 7u) == 0) {
      // ONE bulk copy of the block index (when a search needs it) serves the start and the end search
      const u32 wi = threadIdx.x >> 5;
      u64* mbar = nullptr;
      if (R.n_blocks > 1 && R.n_blocks <= SCAN_STAGE_PFX && ((!extreme && klen) || (has_end && eklen))) {
        mbar = &s_mbar[wi];
        if (lane == 0) tma_load_1d(s_pfx_all[wi], R.blk_pfx, (R.n_blocks * 8u + 15u) & ~15u, mbar);
      }
      const u64* s_pfx = s_pfx_all[wi];
      u32 start, cnt;
      if constexpr (REVERSE) {
        // entries [lo, p) are <= key (< key when exclusive) and >= the low; they go out from p - 1 down
        const u32 p = extreme ? R.n_ent : run_lower_bound_warp(R, kp, klen, !exclusive, s_pfx, mbar, lane);
        const u32 lo = has_end ? run_lower_bound_warp(R, ekp, eklen, false, s_pfx, mbar, lane) : 0u;
        start = p - 1u;  // (unused when p == 0: cnt is 0)
        cnt = p > lo ? min(a.max_entries, p - lo) : 0u;
      } else {
        start = extreme ? 0u : run_lower_bound_warp(R, kp, klen, exclusive, s_pfx, mbar, lane);
        cnt = min(a.max_entries, R.n_ent - start);
        if (has_end) {
          const u32 end = run_lower_bound_warp(R, ekp, eklen, false, s_pfx, mbar, lane);
          cnt = end > start ? min(cnt, end - start) : 0u;
        }
      }
      i32 fst = 0;
      if ((u64)cnt * rec > a.out_stride) { cnt = (u32)(a.out_stride / rec); fst = 7; }
      const u32 wpr = rec >> 3;  // 8-byte words per record
      const u64* src = reinterpret_cast<const u64*>(R.heap) + (u64)start * R.uniform_units * 2u;
      u64* dst = reinterpret_cast<u64*>(out);
      const u32 total = cnt * wpr;
      // RSP_SCAN_UNROLL loads are issued before the first of their stores: with one load in flight per warp (what
      // the plain loop compiles to: LDG, STG, LDG, ...) the kernel is bound by latency x occupancy, not by HBM
      for (u32 w0 = lane; w0 < total; w0 += 32u * RSP_SCAN_UNROLL) {
        u64 v[RSP_SCAN_UNROLL];
#pragma unroll
        for (u32 u = 0; u < RSP_SCAN_UNROLL; u++) {
          const u32 w = w0 + 32u * u;
          if (w < total) {
            const u32 r = w / wpr, jw = w - r * wpr;
            // source words of record r: word 1 = (klen, vlen); key from word 2; value follows (klen % 16 == 0)
            const u64 off = (u64)r * R.uniform_units * 2u;
            v[u] = __ldg((REVERSE ? src - off : src + off) + 1 + jw);
          }
        }
#pragma unroll
        for (u32 u = 0; u < RSP_SCAN_UNROLL; u++) {
          const u32 w = w0 + 32u * u;
          if (w < total) dst[w] = v[u];
        }
      }
      if (lane == 0) {
        a.n_out[q] = cnt;
        a.st[q] = fst;
      }
      return;
    }
  }

  // ---- general path: k-way newest-wins merge over the pinned runs, lane-parallel.  Lane r owns run r's cursor and
  // keeps its head entry cached (pointer, lengths, type, 8-byte big-endian key prefix).  Every lane seeks its own run at
  // the same time; per output key the warp takes the minimum (reverse: maximum) prefix by shuffles, settles prefix ties
  // by full-key compares done in parallel by the tied lanes, and the runs that hold the key are visited newest first
  // while their lanes already load their next heads.  Forward, the head is entry my_cur.  Reverse, it is entry
  // my_cur - 1 (my_cur = the number of entries <= key, or < key when exclusive), the oldest version of its key.
  u32 my_cur = 0, h_klen = 0, h_vlen = 0, h_type = 0;
  const u8* h_e = nullptr;
  u64 h_pfx = 0;
  bool h_valid = false;
  auto load_head = [&]() {
    h_valid = lane < n_runs && (REVERSE ? my_cur > 0 : my_cur < runs[lane].n_ent);
    if (h_valid) {
      h_e = run_entry(runs[lane], REVERSE ? my_cur - 1u : my_cur);
      const uint4 hd = __ldg(reinterpret_cast<const uint4*>(h_e));
      h_type = hd.x & 0xffu; h_klen = hd.z; h_vlen = hd.w;
      h_pfx = h_klen ? bswap64(__ldg(reinterpret_cast<const u64*>(h_e + 16))) : 0ull;
    }
  };
  if (lane < n_runs) {
    if constexpr (REVERSE) my_cur = extreme ? runs[lane].n_ent : run_lower_bound(runs[lane], kp, klen, !exclusive);
    else my_cur = extreme ? 0u : run_lower_bound(runs[lane], kp, klen, exclusive);
  }
  load_head();

  while (n_out < a.max_entries) {
    EntRef bk;
    Acc<CAT> acc;
    acc.init(merge_op, merge_delim);
    const u32 vmask = __ballot_sync(0xffffffffu, h_valid);
    if (!vmask) break;
    // minimum (reverse: maximum) prefix over the valid heads (lanes 0 .. 7 hold the runs: three butterfly steps)
    u64 mp = h_valid ? h_pfx : (REVERSE ? 0ull : ~0ull);
#pragma unroll
    for (u32 d = 1; d < RSP_MAX_RUNS; d <<= 1) {
      const u64 o = __shfl_xor_sync(0xffffffffu, mp, d);
      mp = (REVERSE ? o > mp : o < mp) ? o : mp;
    }
    mp = __shfl_sync(0xffffffffu, mp, 0);
    u32 cand = __ballot_sync(0xffffffffu, h_valid && h_pfx == mp);
    u32 group, w;
    for (;;) {  // the smallest (reverse: largest) full key among the tied prefixes, and every run whose head is that key
      w = (u32)__ffs(cand) - 1u;
      const u64 wk = __shfl_sync(0xffffffffu, (u64)reinterpret_cast<uintptr_t>(h_e), w);
      const u32 wkl = __shfl_sync(0xffffffffu, h_klen, w);
      int c = 0;
      const bool mine = ((cand >> lane) & 1u) && lane != w;
      if (mine) c = cmp_padded(reinterpret_cast<const u64*>(h_e + 16), h_klen, reinterpret_cast<const u64*>(reinterpret_cast<const u8*>(wk) + 16), wkl);
      const u32 ahead = __ballot_sync(0xffffffffu, mine && (REVERSE ? c > 0 : c < 0));
      if (ahead) { cand = ahead; continue; }
      group = __ballot_sync(0xffffffffu, mine && c == 0) | (1u << w);
      break;
    }
    bk.e = reinterpret_cast<const u8*>(__shfl_sync(0xffffffffu, (u64)reinterpret_cast<uintptr_t>(h_e), w));
    bk.klen = __shfl_sync(0xffffffffu, h_klen, w);
    bk.vlen = 0; bk.type = 0;
    // a string-append fold is built in place, at the value of this key's record
    if constexpr (CAT) {
      const u64 voff = used + 8 + bk.klen;
      acc.set_out(out + voff, voff < a.out_stride ? a.out_stride - voff : 0ull, 0xffffffffu);
    }
    // the end key (reverse: the low): checked before any version is visited, so that deleted keys, merge operands and
    // host-folded keys at or beyond the end (below the low) are never walked, folded or reported
    if (has_end) {
      const u64 epfx = key_prefix_be(ekp, eklen);
      if constexpr (REVERSE) {
        if (mp < epfx || (mp == epfx && cmp_key_vs_padded(ekp, eklen, bk.key(), bk.klen) > 0)) break;
      } else {
        if (mp > epfx || (mp == epfx && cmp_key_vs_padded(ekp, eklen, bk.key(), bk.klen) <= 0)) break;
      }
    }
    if constexpr (REVERSE) {
      // the versions of a key lie together in a run, newest first, so the head is the oldest: each run that holds the
      // key walks down to the group's first (newest) entry, and the entry below it becomes its next head.  The group is
      // then [my_cur, top); its last entry is the old head, kept in o_e / o_type / o_vlen.
      const u32 top = my_cur, o_type = h_type, o_vlen = h_vlen;
      const u8* o_e = h_e;
      if ((group >> lane) & 1u) {
        do {
          my_cur--;
          load_head();
        } while (h_valid && h_pfx == mp &&
                 cmp_padded(reinterpret_cast<const u64*>(h_e + 16), h_klen, bk.key(), bk.klen) == 0);
      }
      const u32 voff = 16u + 16u * units_of(bk.klen);
      // newest run first, newest version first
      for (u32 g = group; g && !acc.done;) {
        const u32 r = (u32)__ffs(g) - 1u;
        g &= g - 1u;
        const u32 lo = __shfl_sync(0xffffffffu, my_cur, r), hi = __shfl_sync(0xffffffffu, top, r);
        for (u32 o = lo; o + 1u < hi && !acc.done; o++) {
          const EntRef x = load_ent(runs[r], o);
          acc.visit(x.type, x.val(), x.vlen);
        }
        const u32 t = __shfl_sync(0xffffffffu, o_type, r), vl = __shfl_sync(0xffffffffu, o_vlen, r);
        const u64 ep = __shfl_sync(0xffffffffu, (u64)reinterpret_cast<uintptr_t>(o_e), r);
        if (!acc.done) acc.visit(t, reinterpret_cast<const u8*>(ep) + voff, vl);
      }
    } else {
      // newest run first; inside a run the versions of a key follow each other, newest first
      for (u32 g = group; g;) {
        const u32 r = (u32)__ffs(g) - 1u;
        g &= g - 1u;
        for (;;) {
          const u32 t = __shfl_sync(0xffffffffu, h_type, r), vl = __shfl_sync(0xffffffffu, h_vlen, r);
          const u64 ep = __shfl_sync(0xffffffffu, (u64)reinterpret_cast<uintptr_t>(h_e), r);
          const u32 kl = __shfl_sync(0xffffffffu, h_klen, r);
          if (!acc.done) acc.visit(t, reinterpret_cast<const u8*>(ep) + 16u + 16u * units_of(kl), vl);
          bool same = false;
          if (lane == r) {
            my_cur++;
            load_head();
            same = h_valid && cmp_padded(reinterpret_cast<const u64*>(h_e + 16), h_klen, bk.key(), bk.klen) == 0;
          }
          if (!__shfl_sync(0xffffffffu, (u32)same, r)) break;
        }
      }
    }
    acc.end_of_versions();
    if (acc.status == 1) continue;  // deleted
    u32 vlen = 0;
    bool host_fold = false, merge_failed = false;
    if (acc.status == ST_NEED_HOST_MERGE) {
      // the operator lives on the host: hand back the key alone (vlen marker 0xffffffff)
      if (st == 0) st = ST_NEED_HOST_MERGE;
      host_fold = true;
    } else if (acc.status != 0) {
      // DBIter keeps the key with an empty value and records the (sticky) status; the record carries the marker
      // SCAN_VLEN_MERGE_FAILED so that an iterator can raise the status when it REACHES this key, as DBIter does
      st = (i32)mk_status((u32)acc.status, acc.msg);
      merge_failed = true;
    } else {
      vlen = acc.res_len;
    }
    const u64 rec = 8ull + bk.klen + vlen;
    // out of room: INCOMPLETE, or its flag on top of a status that is already there (host-fold request, failed merge)
    if (used + rec > a.out_stride) { st = st == 0 ? 7 : (st | SCAN_ST_TRUNCATED); break; }
    if (lane == 0) {
      u8 hdr[8];
      const u32 vl_out = host_fold ? SCAN_VLEN_HOST_FOLD : (merge_failed ? SCAN_VLEN_MERGE_FAILED : vlen);
      for (u32 b = 0; b < 4; b++) { hdr[b] = (u8)(bk.klen >> (8 * b)); hdr[4 + b] = (u8)(vl_out >> (8 * b)); }
      for (u32 b = 0; b < 8; b++) out[used + b] = hdr[b];
    }
    warp_copy_bytes(out + used + 8, reinterpret_cast<const u8*>(bk.key()), bk.klen, lane);
    if (vlen) {
      if (acc.imm) {
        if (lane < 8) out[used + 8 + bk.klen + lane] = (u8)(acc.res_imm >> (8u * lane));
      } else if (!acc.in_place(out + used + 8 + bk.klen)) {
        warp_copy_bytes(out + used + 8 + bk.klen, acc.res_ptr, vlen, lane);
      }
    }
    used += rec;
    n_out++;
  }
  if (lane == 0) {
    a.n_out[q] = n_out;
    a.st[q] = st;
  }
}

// (a minimum of one block: with __launch_bounds__(128) alone ptxas holds the instances to 64 or 72 registers and spills
// three of them; with it none spills)
template <bool BOUNDED, bool REVERSE, bool CAT>
__global__ void __launch_bounds__(128, 1) k_multi_scan(ScanArgs a) { multi_scan_body<BOUNDED, REVERSE, CAT>(a); }

template <bool CAT>
static void launch_multi_scan_t(const ScanArgs& a, bool reverse, cudaStream_t s) {
  const u32 blocks = (a.n + 3) / 4;
  if (reverse) {
    if (a.ends) k_multi_scan<true, true, CAT><<<blocks, 128, 0, s>>>(a);
    else k_multi_scan<false, true, CAT><<<blocks, 128, 0, s>>>(a);
  } else {
    if (a.ends) k_multi_scan<true, false, CAT><<<blocks, 128, 0, s>>>(a);
    else k_multi_scan<false, false, CAT><<<blocks, 128, 0, s>>>(a);
  }
}
void launch_multi_scan(const ScanArgs& a, bool reverse, bool cat, cudaStream_t s) {
  if (!a.n) return;
  if (cat) launch_multi_scan_t<true>(a, reverse, s);
  else launch_multi_scan_t<false>(a, reverse, s);
}
}  // namespace rsp
