// reader_set.h — which reads on callers' streams a mutation of the engine must wait for (std only: the stream and
// event operations come from a policy type, so that tests/cpp/reader_set_test.cpp can drive it with fakes).
#pragma once
#include <cstddef>
#include <vector>

namespace rsp {

// One event per distinct caller stream, re-recorded after every read launched on it: a later record on a stream covers
// every earlier read on that stream, so waiting on the events of the streams read since the last wait covers every
// read, however many came after it on other streams.  (A fixed ring of events forgets a stream once that many reads on
// other streams have followed its last one.)  Not thread-safe: the engine calls it with its mutex held.
//
// Api: types Stream, Event; static Event create(); static void record(Event, Stream); static void wait(Stream on,
// Event); static void destroy(Event).
template <class Api>
class ReaderSet {
 public:
  using Stream = typename Api::Stream;
  using Event = typename Api::Event;

  // a read was launched on `s`
  void note(Stream s) {
    for (Entry& x : ents_) {
      if (x.s == s) {
        Api::record(x.ev, s);
        x.pending = true;
        return;
      }
    }
    Entry x{s, Api::create(), true};
    ents_.push_back(x);
    Api::record(x.ev, s);
  }
  // make `on` wait for every read noted since the last wait
  void wait(Stream on) {
    for (Entry& x : ents_) {
      if (!x.pending) continue;
      Api::wait(on, x.ev);
      x.pending = false;
    }
  }
  size_t streams() const { return ents_.size(); }
  size_t pending() const {
    size_t n = 0;
    for (const Entry& x : ents_) n += x.pending;
    return n;
  }
  void destroy() {
    for (Entry& x : ents_) Api::destroy(x.ev);
    ents_.clear();
  }

 private:
  struct Entry {
    Stream s;
    Event ev;
    bool pending;
  };
  std::vector<Entry> ents_;
};

}  // namespace rsp
