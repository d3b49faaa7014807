// pipe_state.cuh -- a position in a ring of N mbarrier-guarded buffers (tc::TmaRing).  Plain C++ (device code calls the constexpr
// members under --expt-relaxed-constexpr), so a host program can check it against a model of the mbarrier protocol.
#pragma once

#include <stdint.h>

namespace kdb {

// Position n is slot n % N in round n / N.  Consumers wait on `full` at the round's parity; the producer waits on `empty` at the other
// one, for the releases of the round before (in round 0 the phase before the first, which counts as complete from init on).
template <int N>
struct PipeState {
  int slot;
  uint32_t phase;
  static constexpr PipeState at(int n) { return PipeState{n % N, (uint32_t)(n / N) & 1u}; }
  constexpr void advance() {
    if (++slot == N) {
      slot = 0;
      phase ^= 1u;
    }
  }
  constexpr uint32_t consumer_parity() const { return phase; }
  constexpr uint32_t producer_parity() const { return phase ^ 1u; }
};

}  // namespace kdb
