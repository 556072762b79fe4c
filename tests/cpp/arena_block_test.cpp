// rsp::ArenaBlock (csrc/arena.h) over malloc'ed "slabs": the handle gives its block back exactly once however it is
// moved — destruction releases, a move hands the block on and leaves the source empty, move-assignment releases what
// the target held, an empty handle releases nothing — and the arena's invariants hold throughout
#include <cstdio>
#include <cstring>
#include <random>
#include <utility>
#include <vector>
#include "../../rocksplicator_b200/csrc/arena.h"
int main() {
  rsp::Arena a;
  a.slab_bytes = 1 << 20;
  a.slab_alloc = [](size_t n) -> void* { void* p = nullptr; if (posix_memalign(&p, 4096, n)) abort(); return p; };
  a.slab_free = [](void* p) { free(p); };
  long bad = 0;
  auto expect = [&](bool ok, const char* what) {
    if (!ok) { bad++; printf("failed: %s\n", what); }
  };
  {
    rsp::ArenaBlock e0;
    expect(!e0 && e0.get() == nullptr, "an empty handle holds nothing");
    rsp::ArenaBlock x(a, 1000);
    expect(x && a.in_use == 1024, "a handle holds its rounded block");
    memset(x.get<unsigned char>(), 7, 1000);
    rsp::ArenaBlock y(std::move(x));
    expect(!x && x.get() == nullptr, "a moved-from handle is empty");
    expect(y && a.in_use == 1024 && y.get<unsigned char>()[999] == 7, "a move hands the same block on");
    rsp::ArenaBlock z(a, 300);
    void* zp = z.get();
    z = std::move(y);
    expect(!y && a.in_use == 1024 && z.get<unsigned char>()[0] == 7 && a.check(), "move-assignment releases the target's block");
    rsp::ArenaBlock w(a, 300);
    expect(w.get() == zp, "the released block is found again");
    z = std::move(z);
    expect(z && a.in_use == 1024 + 512, "self-move changes nothing");
    w.reset();
    w.reset();
    expect(!w && a.in_use == 1024, "reset releases once");
    e0 = std::move(w);
    expect(!e0 && a.in_use == 1024 && a.check(), "empty into empty");
  }
  expect(a.in_use == 0 && a.check(), "every handle released its block on leaving the scope");
  // handles in a growing vector (moves on reallocation), dropped in random order
  std::mt19937_64 rng(7);
  std::vector<rsp::ArenaBlock> v;
  for (int i = 0; i < 2000; i++) {
    v.emplace_back(a, 1 + rng() % 5000);
    if (rng() % 3 == 0) v.erase(v.begin() + rng() % v.size());
    if (i % 128 == 0 && !a.check()) expect(false, "arena invariants");
  }
  v.clear();
  expect(a.in_use == 0 && a.check() && a.free_bytes == a.reserved, "a vector of handles gives every block back");
  printf("arena blocks: bad %ld\n", bad);
  a.destroy();
  return bad != 0;
}
