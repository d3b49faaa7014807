// Host check of csrc/pipe_state.cuh (compiled as plain C++ by tests/test_pipe_state_host.py).  For ring sizes 1..4 over a few thousand
// positions: advance() and at(n) agree, both equal the slot / parity arithmetic the tensor-core kernels wrote out by hand before, and a
// model of mbarrier phases run under many random interleavings never lets the producer refill a slot before all its releases, never lets
// a consumer read a slot before it holds that position, and never deadlocks.  Prints one line per failure and "ok" at the end.
#include <cstdio>
#include <random>
#include <vector>

#include "pipe_state.cuh"

using kdb::PipeState;

static int failures = 0;
#define CHECK(cond, ...)                   \
  do {                                     \
    if (!(cond)) {                         \
      if (failures++ < 50) {               \
        std::printf(__VA_ARGS__);          \
        std::printf("\n");                 \
      }                                    \
    }                                      \
  } while (0)

constexpr int POSITIONS = 5000;

template <int N>
void check_arithmetic() {
  PipeState<N> s{};
  uint32_t su = 0, pu = 0;  // the hand-wrapped counters of the feed-forward kernel's weight rings
  for (int n = 0; n < POSITIONS; ++n, s.advance()) {
    const PipeState<N> a = PipeState<N>::at(n);
    CHECK(a.slot == s.slot && a.phase == s.phase, "N=%d n=%d: at() {%d,%u} != advance() {%d,%u}", N, n, a.slot, a.phase, s.slot, s.phase);
    // the GEMM's ring and the window / global attention's Q and K/V rings: n % N, (n / N) & 1, producer ((n / N) & 1) ^ 1
    CHECK(s.slot == n % N && s.consumer_parity() == (uint32_t)((n / N) & 1) && s.producer_parity() == (uint32_t)(((n / N) & 1) ^ 1),
          "N=%d n=%d: differs from n %% N, (n / N) & 1", N, n);
    CHECK((int)su == s.slot && pu == s.consumer_parity() && (pu ^ 1u) == s.producer_parity(), "N=%d n=%d: differs from the wrapped counters", N, n);
    if (++su == (uint32_t)N) {
      su = 0;
      pu ^= 1u;
    }
    if (N == 2)  // the fused kernels' X buffers: i & 1, (i >> 1) & 1, producer ((i >> 1) & 1) ^ 1
      CHECK(s.slot == (n & 1) && s.consumer_parity() == (uint32_t)((n >> 1) & 1) && s.producer_parity() == (uint32_t)(((n >> 1) & 1) ^ 1),
            "N=2 n=%d: differs from n & 1, (n >> 1) & 1", n);
    if (N == 1)  // the neighbourhood kernel's single K/V buffer: consumer it & 1, producer (it - 1) & 1 for it > 0
      CHECK(s.slot == 0 && s.consumer_parity() == (uint32_t)(n & 1) && (n == 0 || s.producer_parity() == (uint32_t)((n - 1) & 1)),
            "N=1 n=%d: differs from it & 1, (it - 1) & 1", n);
  }
}

// mbarrier: a phase completes when its pending arrivals reach zero; waiting on parity p succeeds once the phase with parity p has
// completed, i.e. while the current (incomplete) phase's parity differs from p.  At init phase 0 is current, so parity 1 passes.
struct MBar {
  int count, pending, phase = 0;
  explicit MBar(int c) : count(c), pending(c) {}
  bool ready(uint32_t parity) const { return (uint32_t)(phase & 1) != parity; }
  void arrive() {
    if (--pending == 0) {
      ++phase;
      pending = count;
    }
  }
};

// One producer, `releasers` consumers that each read every position and release it, random interleaving.
template <int N>
void check_protocol(int releasers, unsigned seed) {
  std::vector<MBar> full(N, MBar(1)), empty(N, MBar(releasers));
  std::vector<int> filled(N, -1);           // position a slot holds
  std::vector<int> released(N, 0);          // releases of the slot's current position
  int prod = 0;
  std::vector<int> cons(releasers, 0);
  std::vector<bool> holding(releasers, false);  // consumer has passed `full` and not yet released
  std::mt19937 rng(seed);
  const int total = 300;
  for (;;) {
    bool done = prod == total;
    for (int c = 0; c < releasers; ++c) done = done && cons[c] == total;
    if (done) return;
    // agents that can make progress now
    std::vector<int> can;
    if (prod < total && empty[PipeState<N>::at(prod).slot].ready(PipeState<N>::at(prod).producer_parity())) can.push_back(-1);
    for (int c = 0; c < releasers; ++c) {
      if (cons[c] == total) continue;
      const PipeState<N> s = PipeState<N>::at(cons[c]);
      if (holding[c] || full[s.slot].ready(s.consumer_parity())) can.push_back(c);
    }
    CHECK(!can.empty(), "N=%d releasers=%d seed=%u: deadlock at producer %d", N, releasers, seed, prod);
    if (can.empty()) return;
    const int who = can[rng() % can.size()];
    if (who < 0) {
      const PipeState<N> s = PipeState<N>::at(prod);
      CHECK(prod < N || (filled[s.slot] == prod - N && released[s.slot] == releasers), "N=%d releasers=%d: slot %d refilled for %d before its releases",
            N, releasers, s.slot, prod);
      filled[s.slot] = prod;
      released[s.slot] = 0;
      full[s.slot].arrive();  // the expect_tx arrival and the TMA bytes landing, taken together
      ++prod;
    } else if (!holding[who]) {
      const PipeState<N> s = PipeState<N>::at(cons[who]);
      CHECK(filled[s.slot] == cons[who], "N=%d releasers=%d: consumer read slot %d for %d while it holds %d", N, releasers, s.slot, cons[who],
            filled[s.slot]);
      holding[who] = true;
    } else {
      const PipeState<N> s = PipeState<N>::at(cons[who]);
      ++released[s.slot];
      empty[s.slot].arrive();
      holding[who] = false;
      ++cons[who];
    }
  }
}

template <int N>
void check_all() {
  check_arithmetic<N>();
  for (int releasers : {1, 2, 4, 8})
    for (unsigned seed = 0; seed < 20; ++seed) check_protocol<N>(releasers, seed);
}

int main() {
  check_all<1>();
  check_all<2>();
  check_all<3>();
  check_all<4>();
  if (failures) {
    std::printf("%d failures\n", failures);
    return 1;
  }
  std::printf("ok\n");
  return 0;
}
