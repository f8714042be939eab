// ccm_relay.h — the accounting rule of the relayed whole-HBM gate (ccm-scrub --relay, DESIGN.md §5n) and the rule that
// decides when a GPU's free memory has settled after the first leg's process ended.  Plain C++17, no CUDA: a CPU test
// compiles it on its own.
//
// Leg A scrubs everything its context can map and hands its mapping back; while A's context still exists, the process
// that runs leg B creates its own, so B's footprint can only come from memory A just scrubbed.  A then exits, and leg B
// scrubs everything free, which now includes A's footprint.  account() says, per GPU, how much of the device neither
// leg reached.
#pragma once
#include <cstdint>

namespace ccm_relay {

// The settle rule: free memory is read every kSettlePollMs after A was reaped, until kSettleFlat reads in a row are
// equal or kSettleDeadlineMs have passed.
constexpr double kSettlePollMs = 5.0;
constexpr int kSettleFlat = 4;
constexpr double kSettleDeadlineMs = 2000.0;

// What the two legs measured on one GPU, in bytes (cudaMemGetInfo's numbers and the gate reports').
struct Inputs {
  uint64_t total = 0;            // cudaMemGetInfo total (leg B's report)
  uint64_t a_free_before = 0;    // leg A's report: free when its gate started
  uint64_t a_unreached = 0;      // leg A's report: free, but not mappable
  uint64_t b_free_held = 0;      // free once leg B's context existed and was armed, A still alive
  uint64_t b_free_settled = 0;   // free once A had exited and the reads settled
  uint64_t b_free_before = 0;    // leg B's report: free when its gate started
  uint64_t b_unreached = 0;      // leg B's report: free, but not mappable
  uint64_t marked = 0;           // bytes A held with a known content until it exited (a drill; 0 otherwise)
};

struct Relay {
  Inputs in;
  uint64_t footprint_a = 0;   // what the device held beside leg A's mapping when A started
  uint64_t freed = 0;         // what A's exit gave back
  uint64_t held = 0;          // what neither leg could map: another process's memory, or what the driver kept
  uint64_t growth = 0;        // what leg B's process allocated after the hand-over (it may sit on A's freed memory)
  uint64_t unreached = 0;     // held + growth + both legs' unmappable granules
  double coverage = 0;        // 1 - unreached / total
};

inline uint64_t minus(uint64_t a, uint64_t b) { return a > b ? a - b : 0; }
inline uint64_t plus(uint64_t a, uint64_t b) { return a + b < a ? UINT64_MAX : a + b; }

// Every difference is clamped at 0 and every sum saturates: nonsense inputs (free > total) never wrap.
inline Relay account(const Inputs& in) {
  Relay r;
  r.in = in;
  r.footprint_a = minus(in.total, in.a_free_before);
  r.freed = minus(in.b_free_settled, in.b_free_held);
  r.held = minus(r.footprint_a, r.freed);
  r.growth = minus(in.b_free_settled, in.b_free_before);
  r.unreached = plus(plus(r.held, r.growth), plus(in.a_unreached, in.b_unreached));
  const uint64_t miss = r.unreached < in.total ? r.unreached : in.total;
  r.coverage = in.total ? 1.0 - (double)miss / (double)in.total : 0.0;
  return r;
}

// One GPU's wait for its free memory to settle: read() takes each read and the ms since the wait began, and returns
// true once the wait is over.  `free_bytes` is then the last read; `settled` says whether the reads went flat or the
// deadline ended the wait.
struct Settle {
  uint64_t free_bytes = 0;
  int polls = 0;
  int flat = 0;
  bool settled = false;
  bool done = false;

  bool read(uint64_t free_now, double ms) {
    if (done) return true;
    flat = polls && free_now == free_bytes ? flat + 1 : 1;
    free_bytes = free_now;
    ++polls;
    settled = flat >= kSettleFlat;
    done = settled || ms >= kSettleDeadlineMs;
    return done;
  }
};

}  // namespace ccm_relay
