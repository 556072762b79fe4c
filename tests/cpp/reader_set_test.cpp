// csrc/reader_set.h with fake streams and events: a mutation waits for the latest read on every stream read since the
// last wait, however many reads on other streams came after it (a ring of eight events forgot such a stream), one
// stream keeps one event, a wait clears the pending set, and destroy releases every event it created
#include <cstdio>
#include <set>
#include <utility>
#include <vector>
#include "../../rocksplicator_b200/csrc/reader_set.h"

struct Fake {
  using Stream = int;
  using Event = int;
  static int created, destroyed;
  static std::vector<std::pair<int, int>> records;  // (event, stream)
  static std::vector<std::pair<int, int>> waits;    // (waiting stream, event)
  static std::set<int> live;
  static Event create() { live.insert(created); return created++; }
  static void record(Event ev, Stream s) { records.push_back({ev, s}); }
  static void wait(Stream on, Event ev) { waits.push_back({on, ev}); }
  static void destroy(Event ev) { destroyed++; live.erase(ev); }
};
int Fake::created = 0, Fake::destroyed = 0;
std::vector<std::pair<int, int>> Fake::records, Fake::waits;
std::set<int> Fake::live;

static int bad = 0;
#define CHECK(c)                                              \
  do {                                                        \
    if (!(c)) { printf("FAILED line %d: %s\n", __LINE__, #c); bad++; } \
  } while (0)

// the stream whose latest record the event `ev` holds
static int stream_of(int ev) {
  int s = -1;
  for (auto& r : Fake::records)
    if (r.first == ev) s = r.second;
  return s;
}

int main() {
  const int ENGINE = 0, A = 1, B = 2, C = 3;
  rsp::ReaderSet<Fake> rs;
  // one read on A, then nine on B: the wait covers A and B
  rs.note(A);
  for (int i = 0; i < 9; i++) rs.note(B);
  CHECK(rs.streams() == 2);
  CHECK(rs.pending() == 2);
  rs.wait(ENGINE);
  std::set<int> covered;
  for (auto& w : Fake::waits) {
    CHECK(w.first == ENGINE);
    covered.insert(stream_of(w.second));
  }
  CHECK(covered == std::set<int>({A, B}));
  CHECK(Fake::waits.size() == 2);
  // the wait cleared the pending set: a second wait issues nothing
  CHECK(rs.pending() == 0);
  rs.wait(ENGINE);
  CHECK(Fake::waits.size() == 2);
  // repeated reads on one stream keep one entry, re-recording its event on that stream
  const size_t rec0 = Fake::records.size();
  for (int i = 0; i < 40; i++) rs.note(A);
  CHECK(rs.streams() == 2);
  CHECK(Fake::created == 2);
  CHECK(Fake::records.size() == rec0 + 40);
  CHECK(rs.pending() == 1);
  // a third stream after the first two: only the streams read since the last wait are waited for
  rs.note(C);
  Fake::waits.clear();
  rs.wait(ENGINE);
  covered.clear();
  for (auto& w : Fake::waits) covered.insert(stream_of(w.second));
  CHECK(covered == std::set<int>({A, C}));
  // many streams, one read each, then many reads on one of them: every stream is still waited for
  for (int s = 10; s < 30; s++) rs.note(s);
  for (int i = 0; i < 100; i++) rs.note(29);
  Fake::waits.clear();
  rs.wait(ENGINE);
  covered.clear();
  for (auto& w : Fake::waits) covered.insert(stream_of(w.second));
  CHECK(covered.size() == 20 && *covered.begin() == 10 && *covered.rbegin() == 29);
  // destroy releases every event it created
  rs.destroy();
  CHECK(rs.streams() == 0);
  CHECK(Fake::destroyed == Fake::created);
  CHECK(Fake::live.empty());
  printf("reader_set: events %d, bad %d\n", Fake::created, bad);
  return bad ? 1 : 0;
}
