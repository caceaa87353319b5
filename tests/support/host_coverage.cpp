// Test harness (NOT a product path): per-emit-site coverage of a lowered model on the host.  A sequential BFS
// (past violations, like -continue) that enumerates successors through the two-phase form the expand kernel runs:
// for every expanded state and site group, each set bit of site_mask counts one successor of that emit site, and
// the site bodies produce the successors.  Build: g++ -O2 -shared -fPIC -DKMC_MODEL_HEADER='"model.h"' host_coverage.cpp
#include <stdint.h>
#include <string.h>
#include <unordered_set>
#include <vector>
#include KMC_MODEL_HEADER

namespace M = kmc_model;
using M::State;
namespace {
struct StateHash {
  size_t operator()(const State& s) const {
    uint64_t h = 0x9E3779B97F4A7C15ull;
    for (int i = 0; i < M::W; ++i) {
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
template <int G>
struct Groups {
  static void run(const State& s, uint64_t* site_gen, Sink& sink) {
    const uint64_t m = M::site_mask(M::SiteGroupTag<G>{}, s);
    for (int b = 0; b < M::SITE_GROUP_BEGIN[G + 1] - M::SITE_GROUP_BEGIN[G]; ++b)
      if ((m >> b) & 1) site_gen[M::SITE_GROUP_BEGIN[G] + b]++;
    M::SiteLoop<M::SITE_GROUP_BEGIN[G], M::SITE_GROUP_BEGIN[G + 1]>::run(m, 0, s, sink);
    Groups<G + 1>::run(s, site_gen, sink);
  }
};
template <>
struct Groups<M::NUM_SITE_GROUPS> {
  static void run(const State&, uint64_t*, Sink&) {}
};
}  // namespace

extern "C" int kmc_cov_num_sites() { return M::NUM_SITES; }
extern "C" int kmc_cov_site_action(int i) { return M::SITE_ACTION[i]; }

// stats: [0] distinct  [1] generated (initial states included)  [2] fail code (0 = complete);  site_gen[NUM_SITES]
extern "C" int kmc_cov_bfs(uint64_t* stats, uint64_t* site_gen) {
  memset(stats, 0, 3 * sizeof(uint64_t));
  memset(site_gen, 0, sizeof(uint64_t) * (M::NUM_SITES > 0 ? M::NUM_SITES : 1));
  std::unordered_set<State, StateHash, StateEq> seen;
  std::vector<State> frontier, next;
  for (int i = 0; i < M::NUM_INIT; ++i) {
    State s, c;
    memcpy(s.w, M::INIT_STATES[i], sizeof(s.w));
    stats[1]++;
    if (!M::in_model(s)) continue;
    M::canonicalize(s, c);
    if (seen.insert(c).second) frontier.push_back(s);
  }
  Sink sink;
  while (!frontier.empty()) {
    next.clear();
    for (const State& s : frontier) {
      sink.out.clear();
      Groups<0>::run(s, site_gen, sink);
      if (sink.failed) {
        stats[2] = (uint64_t)sink.failed;
        stats[0] = seen.size();
        return 1;
      }
      stats[1] += sink.out.size();
      for (const State& n : sink.out) {
        if (!M::in_model(n)) continue;
        State c;
        M::canonicalize(n, c);
        if (seen.insert(c).second) next.push_back(n);
      }
    }
    frontier.swap(next);
  }
  stats[0] = seen.size();
  return 0;
}
