// arena.h — the engine's device-memory arena (std only: the slab allocator is a callback, so that tests/cpp/arena_test.cpp
// can drive it over malloc).
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <iterator>
#include <map>
#include <mutex>
#include <vector>

namespace rsp {

// best-fit blocks with splitting and coalescing, carved from large slabs
// Requests are rounded to 256 bytes and served from the smallest free block that fits (the remainder stays free); a
// released block merges with its free neighbours inside its slab.  (Power-of-two size classes with per-class free
// lists do not work here: a shard's runs grow from generation to generation, so the classes of the earlier generations
// fill up with blocks nobody asks for again.)
struct Arena {
  std::mutex mu;
  size_t slab_bytes = 0;
  std::vector<void*> slabs;
  struct Block { size_t size; uint32_t slab; bool free; };
  // how slabs are obtained / returned (the engine: cudaMalloc / cudaFree, throwing on failure)
  void* (*slab_alloc)(size_t) = nullptr;
  void (*slab_free)(void*) = nullptr;
  std::map<uintptr_t, Block> blocks;                 // every block of every slab, by address
  std::multimap<size_t, uintptr_t> free_by_size;     // the free ones, by size
  size_t in_use = 0, reserved = 0, free_bytes = 0;

  static size_t round_up(size_t n) { return (std::max<size_t>(n, 1) + 255) & ~(size_t)255; }
#ifdef RSP_EMUL
  // tests/emul under AddressSanitizer: every request is its own exactly-sized allocation, freed on release, so an
  // access past the requested size or after release is reported instead of landing in a neighbour
  static bool exact() { static const bool on = getenv("RSP_EMUL_EXACT_ALLOC") != nullptr; return on; }
#endif
  void drop_free(std::map<uintptr_t, Block>::iterator it) {  // mu held: *it leaves the size index
    auto r = free_by_size.equal_range(it->second.size);
    for (auto f = r.first; f != r.second; ++f)
      if (f->second == it->first) { free_by_size.erase(f); break; }
    free_bytes -= it->second.size;
  }
  void add_free(std::map<uintptr_t, Block>::iterator it) {
    it->second.free = true;
    free_by_size.emplace(it->second.size, it->first);
    free_bytes += it->second.size;
  }
  void* alloc(size_t n) {
#ifdef RSP_EMUL
    if (exact()) return slab_alloc(n ? n : 1);
#endif
    const size_t c = round_up(n);
    std::lock_guard<std::mutex> g(mu);
    auto f = free_by_size.lower_bound(c);
    if (f == free_by_size.end()) {
      // nothing fits: one more slab (a request beyond the slab size gets a slab of its own size)
      const size_t sb = std::max(slab_bytes, c);
      void* s = slab_alloc(sb);
      slabs.push_back(s);
      reserved += sb;
      auto it = blocks.emplace((uintptr_t)s, Block{sb, (uint32_t)(slabs.size() - 1), true}).first;
      add_free(it);
      f = free_by_size.lower_bound(c);
    }
    auto it = blocks.find(f->second);
    drop_free(it);
    it->second.free = false;
    if (it->second.size > c) {  // the tail stays free
      const size_t rest = it->second.size - c;
      it->second.size = c;
      auto tail = blocks.emplace(it->first + c, Block{rest, it->second.slab, true}).first;
      add_free(tail);
    }
    in_use += c;
    return (void*)it->first;
  }
  // (the block map knows every block's size: a size passed by a caller is not needed and not read)
  void release(void* p, size_t /*unused*/ = 0) {
    if (!p) return;
#ifdef RSP_EMUL
    if (exact()) { slab_free(p); return; }
#endif
    std::lock_guard<std::mutex> g(mu);
    auto it = blocks.find((uintptr_t)p);
    if (it == blocks.end() || it->second.free) return;  // (not ours / released twice: ignored)
    in_use -= it->second.size;
    // merge with the free neighbours of the same slab
    auto nx = std::next(it);
    if (nx != blocks.end() && nx->second.free && nx->second.slab == it->second.slab && it->first + it->second.size == nx->first) {
      drop_free(nx);
      it->second.size += nx->second.size;
      blocks.erase(nx);
    }
    if (it != blocks.begin()) {
      auto pv = std::prev(it);
      if (pv->second.free && pv->second.slab == it->second.slab && pv->first + pv->second.size == it->first) {
        drop_free(pv);
        pv->second.size += it->second.size;
        blocks.erase(it);
        it = pv;
      }
    }
    add_free(it);
  }
  // invariants (tests): the blocks of a slab tile it exactly, no two neighbours of a slab are both free, the size index
  // holds exactly the free blocks, the counters add up
  bool check() {
    std::lock_guard<std::mutex> g(mu);
    size_t used = 0, fre = 0, n_free = 0;
    std::vector<size_t> per_slab(slabs.size(), 0);
    const Block* prev = nullptr;
    uintptr_t prev_end = 0;
    for (auto& kv : blocks) {
      const Block& b = kv.second;
      if (b.slab >= slabs.size() || b.size == 0 || (kv.first & 255) || (b.size & 255)) return false;
      if (prev && prev->slab == b.slab) {
        if (prev_end != kv.first) return false;          // a hole or an overlap inside a slab
        if (prev->free && b.free) return false;          // not coalesced
      }
      per_slab[b.slab] += b.size;
      (b.free ? fre : used) += b.size;
      n_free += b.free ? 1 : 0;
      prev = &b;
      prev_end = kv.first + b.size;
    }
    size_t total = 0;
    for (size_t v : per_slab) total += v;
    if (total != reserved || used != in_use || fre != free_bytes || n_free != free_by_size.size()) return false;
    for (auto& f : free_by_size) {
      auto it = blocks.find(f.second);
      if (it == blocks.end() || !it->second.free || it->second.size != f.first) return false;
    }
    return true;
  }
  void destroy() {
    for (void* s : slabs) slab_free(s);
    slabs.clear();
    blocks.clear();
    free_by_size.clear();
    in_use = reserved = free_bytes = 0;
  }
};

// One arena block and the duty to give it back: released when the handle is destroyed or assigned over, handed on by
// move.  An empty handle owns nothing and its get() is null.
class ArenaBlock {
 public:
  ArenaBlock() = default;
  ArenaBlock(Arena& a, size_t n) : a_(&a), p_(a.alloc(n)) {}
  ArenaBlock(ArenaBlock&& o) noexcept : a_(o.a_), p_(o.p_) { o.p_ = nullptr; }
  ArenaBlock& operator=(ArenaBlock&& o) noexcept {
    if (this != &o) {
      reset();
      a_ = o.a_;
      p_ = o.p_;
      o.p_ = nullptr;
    }
    return *this;
  }
  ~ArenaBlock() { reset(); }
  template <class T = void>
  T* get() const { return static_cast<T*>(p_); }
  explicit operator bool() const { return p_ != nullptr; }
  void reset() {
    if (p_) a_->release(p_);
    p_ = nullptr;
  }

 private:
  Arena* a_ = nullptr;
  void* p_ = nullptr;
};

}  // namespace rsp
