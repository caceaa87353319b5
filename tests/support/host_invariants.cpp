// Test harness (NOT a product path): a lowered model.h and its invariants.h compiled for the host, for the tests of the
// per-invariant report (tests/test_invariant_reports_host.py builds it, one library per header pair):
//   g++ -O2 -std=c++17 -shared -fPIC -DKMC_MODEL_HEADER='"model.h"' -DKMC_INVARIANTS_HEADER='"invariants.h"' host_invariants.cpp
//   hi_mask / hi_first   violated_invariants and first_violated_invariant of one state
//   hi_bfs               a level-ordered BFS past violations that reports, per invariant, what kmc_invariant_reports does
#include <stdint.h>
#include <string.h>

#include <unordered_set>
#include <vector>
#include KMC_MODEL_HEADER
#include KMC_INVARIANTS_HEADER

namespace M = kmc_model;
using M::State;
namespace {
constexpr int W = M::W;

struct StateHash {
  size_t operator()(const State& s) const {
    uint64_t h = 0x9E3779B97F4A7C15ull;
    for (int i = 0; i < W; ++i) {
      h ^= s.w[i] + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2);
      h *= 0xff51afd7ed558ccdull;
      h ^= h >> 33;
    }
    return (size_t)h;
  }
};
struct StateEq {
  bool operator()(const State& a, const State& b) const { return memcmp(a.w, b.w, sizeof(a.w)) == 0; }
};
struct Sink {
  std::vector<State> out;
  int failed = 0;
  void emit(const State& n, int) { out.push_back(n); }
  void fail(int code) { failed = code; }
};
State load(const uint64_t* p) {
  State s;
  memcpy(s.w, p, sizeof(s.w));
  return s;
}
State canon(const State& s) {
  State c;
  M::canonicalize(s, c);
  return c;
}
// the engine's set-identity fingerprint (kmc_engine.cu)
uint64_t fmix64(uint64_t x) {
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdull;
  x ^= x >> 33;
  x *= 0xc4ceb9fe1a85ec53ull;
  x ^= x >> 33;
  return x;
}
uint64_t fingerprint(const State& s) {
  if (M::STATE_BITS <= 63) return fmix64(s.w[0] + 1);
  uint64_t h = fmix64(s.w[0] + 0x9E3779B97F4A7C15ull);
  for (int i = 1; i < W; ++i) h = fmix64(h ^ (s.w[i] + 0x9E3779B97F4A7C15ull * (uint64_t)(i + 1)));
  return h ? h : 1;
}
}  // namespace

extern "C" {
uint64_t hi_mask(const uint64_t* w) { return M::violated_invariants(load(w)); }
int hi_first(const uint64_t* w) { return M::first_violated_invariant(load(w)); }
int hi_num_invariants() { return M::NUM_INVARIANTS; }

// Level-ordered BFS past violations.  Checked states: every initial state, every stored state (at its level) and every
// successor a CONSTRAINT discards (at its parent's level + 1, each time it is generated).  Per invariant i (arrays of
// NUM_INVARIANTS): first_level[i] (0: never violated), the violators at that level, the violators over the run and the
// smallest set-identity fingerprint among the first level's violators.  Returns the number of checked states on which
// violated_invariants and first_violated_invariant disagree (ctz of a non-zero mask, or a zero mask and -1), or -1 on a
// layout trap.
int64_t hi_bfs(uint64_t* first_level, uint64_t* first_count, uint64_t* total, uint64_t* pick_fp) {
  const int n_inv = M::NUM_INVARIANTS;
  for (int i = 0; i < n_inv; ++i) first_level[i] = first_count[i] = total[i] = 0, pick_fp[i] = ~0ull;
  int64_t mismatches = 0;
  auto check = [&](const State& s, uint64_t level) {
    const uint64_t m = M::violated_invariants(s);
    const int first = M::first_violated_invariant(s);
    if (m ? first != __builtin_ctzll(m) : first != -1) ++mismatches;
    for (int i = 0; i < n_inv; ++i) {
      if (!((m >> i) & 1)) continue;
      total[i]++;
      if (!first_level[i]) first_level[i] = level;
      if (first_level[i] != level) continue;
      first_count[i]++;
      const uint64_t fp = fingerprint(canon(s));
      if (fp < pick_fp[i]) pick_fp[i] = fp;
    }
  };
  std::unordered_set<State, StateHash, StateEq> seen;
  std::vector<State> store;
  auto reach = [&](const State& s, uint64_t level) {
    if (M::NUM_CONSTRAINTS > 0 && !M::in_model(s)) return check(s, level);
    if (!seen.insert(canon(s)).second) return;
    store.push_back(s);
    check(s, level);
  };
  for (int i = 0; i < M::NUM_INIT; ++i) reach(load(M::INIT_STATES[i]), 1);
  Sink sink;
  for (size_t first = 0, level = 1; first < store.size(); ++level) {
    const size_t end = store.size();
    for (size_t k = first; k < end; ++k) {
      sink.out.clear();
      M::expand(store[k], sink);
      if (sink.failed) return -1;
      for (const State& t : sink.out) reach(t, level + 1);
    }
    first = end;
  }
  return mismatches;
}
}  // extern "C"
