// Test harness (NOT a product path): whole-store audit of a finished or stopped GPU run against the lowered Next,
// compiled for the host from the same model.h the engine was built from.  Input: the stored states and parent words
// (of one rank, or the union of several ranks' stores), each state's BFS level and the number of expanded levels.
// The audit checks, state by state, what the engine's bookkeeping claims:
//   init        level 1 = the in-model INIT_STATES, one per identity, parent word NO_PARENT
//   edges       a state of level L >= 2 names a parent of level L-1 (rank, index), an action id < NUM_ACTIONS, and its
//               exact words are a successor of that parent labelled with that action, under expand() AND expand_sites()
//   uniqueness  canonical identities are pairwise distinct
//   closure     every in-model successor of every expanded state of level L is stored at a level <= L+1
// and recomputes the run's totals (generated, deadlocks, out-of-model, per action, per emit site) and the violators the
// engine records at each level end.  A level-ordered host BFS writes a store in the same format (CPU tests).
// Build: g++ -O2 -std=c++17 -shared -fPIC -DKMC_MODEL_HEADER='"model.h"' host_audit.cpp
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>
#include KMC_MODEL_HEADER

namespace M = kmc_model;
using M::State;
namespace {
constexpr uint64_t NO_PARENT = 0x0000FFFFFFFFFFFFull;
constexpr uint64_t IDX_MASK = 0x000000FFFFFFFFFFull;

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
  std::vector<int> act;
  int failed = 0;
  void emit(const State& n, int a) {
    out.push_back(n);
    act.push_back(a);
  }
  void fail(int code) { failed = code; }
  void clear() {
    out.clear();
    act.clear();
  }
};
// the two-phase form the expand kernel runs: per site group, the popcount of site_mask counts each site's successors
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
bool kept(const State& s) { return M::NUM_CONSTRAINTS == 0 || M::in_model(s); }   // passes every CONSTRAINT
bool has_edge(const Sink& sink, const State& s, int action) {
  for (size_t k = 0; k < sink.out.size(); ++k)
    if (sink.act[k] == action && StateEq()(sink.out[k], s)) return true;
  return false;
}
std::string words_text(const State& s) {
  std::string t;
  char b[24];
  for (int i = 0; i < M::W; ++i) {
    snprintf(b, sizeof(b), "%s%016llx", i ? " " : "", (unsigned long long)s.w[i]);
    t += b;
  }
  return t;
}
int report(char* msg, size_t cap, const std::string& text) {
  if (msg && cap) {
    strncpy(msg, text.c_str(), cap - 1);
    msg[cap - 1] = 0;
  }
  return 1;
}

// The store as the audit sees it: the union of `n_ranks` ranks' stores, rank r at [rank_off[r], rank_off[r+1]).
struct Store {
  const uint64_t* states;
  const uint64_t* parents;
  const uint32_t* level;
  uint64_t n;
  const uint64_t* rank_off;
  uint32_t n_ranks;
  State at(uint64_t i) const { return load(states + i * M::W); }
  uint32_t rank_of(uint64_t i) const {
    uint32_t r = 0;
    while (r + 1 < n_ranks && i >= rank_off[r + 1]) ++r;
    return r;
  }
  // the parent word the engine gives a successor of state i (its index in its own rank's store, and that rank)
  uint64_t parent_ref(uint64_t i) const {
    const uint32_t r = rank_of(i);
    return (i - rank_off[r]) | ((uint64_t)r << 40);
  }
};

// Violators the engine records at the end of level `e` (0 = the insert of the initial states):
//   e = 0   stored level-1 states that violate an invariant, in-model or not (the initial states go through the insert)
//   e >= 1  deadlocks of level e (when deadlocks are checked), stored level-(e+1) states that violate an invariant,
//           and the out-of-model successors of level e that violate one (every generation of one, not deduplicated)
// Row: W words, parent word, invariant (~0 = deadlock), 1 if the engine fingerprints the canonical state (the
// out-of-model rows: the insert's identity) else 0 (k_invariants and deadlocks fingerprint the stored state).
struct ViolationSink {
  std::vector<uint64_t>* rows;   // the rows of the first level end that has any (so far)
  uint64_t* counts;              // [n_expanded + 1] violators per level end
  uint64_t first = ~0ull;
  void add(uint64_t e, const State& s, uint64_t meta, uint64_t inv, uint64_t canonical) {
    counts[e]++;
    if (e > first) return;
    if (e < first) {
      rows->clear();
      first = e;
    }
    for (int k = 0; k < M::W; ++k) rows->push_back(s.w[k]);
    rows->push_back(meta);
    rows->push_back(inv);
    rows->push_back(canonical);
  }
};
}  // namespace

extern "C" {
int audit_words() { return M::W; }
int audit_state_bits() { return M::STATE_BITS; }
int audit_all_ones_possible() { return M::ALL_ONES_POSSIBLE ? 1 : 0; }
int audit_has_symmetry() { return M::HAS_SYMMETRY ? 1 : 0; }
int audit_num_actions() { return M::NUM_ACTIONS; }
int audit_num_sites() { return M::NUM_SITES; }
int audit_num_invariants() { return M::NUM_INVARIANTS; }
int audit_num_init() { return M::NUM_INIT; }
int audit_check_deadlock() { return M::CHECK_DEADLOCK ? 1 : 0; }
const char* audit_digest() { return KMC_MODEL_DIGEST; }

void audit_canonicalize(const uint64_t* states, uint64_t n, uint64_t* out) {
  for (uint64_t i = 0; i < n; ++i) {
    const State c = canon(load(states + i * M::W));
    memcpy(out + i * M::W, c.w, sizeof(c.w));
  }
}

// Returns 0 when every check passes, else 1 with "<check>: <what>" in msg.  level[i] is state i's BFS level (1 = Init);
// levels 1..n_expanded were expanded.  Outputs (also on failure, as far as computed):
//   totals[0] generated (NUM_INIT + successors of the expanded states)   totals[1] deadlocks of the expanded states
//   totals[2] out-of-model (initial states and successors)
//   act_gen[NUM_ACTIONS], site_gen[NUM_SITES]: successors per action / per emit site
//   viol_counts[n_expanded + 1]: violators recorded at each level end; audit_violator_rows then returns those of the
//   first level end that has any
static std::vector<uint64_t> g_viol_rows;
int audit_store(const uint64_t* states, const uint64_t* parents, const uint32_t* level, uint64_t n, const uint64_t* rank_off,
                uint32_t n_ranks, uint32_t n_expanded, int check_deadlock, uint64_t* totals,
                uint64_t* act_gen, uint64_t* site_gen, uint64_t* viol_counts, char* msg, size_t msg_cap) {
  const Store S{states, parents, level, n, rank_off, n_ranks};
  memset(totals, 0, 3 * sizeof(uint64_t));
  memset(act_gen, 0, sizeof(uint64_t) * M::NUM_ACTIONS);
  memset(site_gen, 0, sizeof(uint64_t) * (M::NUM_SITES > 0 ? M::NUM_SITES : 1));
  memset(viol_counts, 0, sizeof(uint64_t) * (n_expanded + 1));
  g_viol_rows.clear();
  ViolationSink V{&g_viol_rows, viol_counts};
  char b[512];
  for (uint64_t i = 1; i < n; ++i)
    if (level[i] < level[i - 1] && S.rank_of(i) == S.rank_of(i - 1))
      return report(msg, msg_cap, "levels: the level bounds are not ordered");

  // ---- init: level 1 is the set of in-model initial states, one per identity
  std::unordered_set<State, StateHash, StateEq> init_ids;
  totals[0] = M::NUM_INIT;
  for (int i = 0; i < M::NUM_INIT; ++i) {
    const State s = load(M::INIT_STATES[i]);
    if (!kept(s)) {
      totals[2]++;
      if (M::NUM_INVARIANTS > 0) {
        const int inv = M::first_violated_invariant(s);
        if (inv >= 0) V.add(0, s, NO_PARENT, (uint64_t)inv, 1);
      }
      continue;
    }
    init_ids.insert(canon(s));
  }
  uint64_t n_level1 = 0;
  for (uint64_t i = 0; i < n; ++i) {
    const bool no_parent = (parents[i] & NO_PARENT) == NO_PARENT;
    if (level[i] != 1) {
      if (no_parent) {
        snprintf(b, sizeof(b), "init: state %llu of level %u has no parent", (unsigned long long)i, level[i]);
        return report(msg, msg_cap, b);
      }
      continue;
    }
    ++n_level1;
    const State s = S.at(i);
    bool is_init = false;
    for (int k = 0; k < M::NUM_INIT && !is_init; ++k) is_init = memcmp(s.w, M::INIT_STATES[k], sizeof(s.w)) == 0;
    if (!is_init || parents[i] != NO_PARENT || !init_ids.count(canon(s))) {
      snprintf(b, sizeof(b), "init: level-1 state %llu [%s] parent word %016llx is not an in-model initial state with NO_PARENT",
               (unsigned long long)i, words_text(s).c_str(), (unsigned long long)parents[i]);
      return report(msg, msg_cap, b);
    }
  }
  if (n_level1 != init_ids.size()) {
    snprintf(b, sizeof(b), "init: level 1 holds %llu states, the model has %zu initial identities", (unsigned long long)n_level1,
             init_ids.size());
    return report(msg, msg_cap, b);
  }

  // ---- edges: every non-initial state is a successor of its parent under the action its parent word names
  Sink sink;
  std::vector<uint64_t> scratch(M::NUM_SITES > 0 ? M::NUM_SITES : 1);
  for (uint64_t i = 0; i < n; ++i) {
    if (level[i] < 2) continue;
    const uint64_t pw = parents[i];
    const uint32_t prank = (uint32_t)((pw >> 40) & 0xFF), act = (uint32_t)(pw >> 56);
    const uint64_t idx = pw & IDX_MASK;
    const char* bad = nullptr;
    uint64_t pos = 0;
    if (prank >= n_ranks) bad = "names a rank outside the run";
    else if ((pw >> 48) & 0xFF) bad = "has bits 48..55 set";
    else if (idx >= rank_off[prank + 1] - rank_off[prank]) bad = "names an index outside the parent rank's store";
    else if (level[pos = rank_off[prank] + idx] != level[i] - 1) bad = "names a parent outside the previous level";
    else if (act >= (uint32_t)M::NUM_ACTIONS) bad = "names an action id >= NUM_ACTIONS";
    if (!bad) {
      const State p = S.at(pos), s = S.at(i);
      sink.clear();
      M::expand(p, sink);
      if (!has_edge(sink, s, (int)act)) bad = "names a parent whose expand() has no such successor under that action";
      sink.clear();
      M::expand_sites(p, sink);
      if (!bad && !has_edge(sink, s, (int)act)) bad = "names a parent whose expand_sites() has no such successor under that action";
    }
    if (bad) {
      snprintf(b, sizeof(b), "edges: state %llu (level %u) parent word %016llx (rank %u, index %llu, action %u) %s",
               (unsigned long long)i, level[i], (unsigned long long)pw, prank, (unsigned long long)idx, act, bad);
      return report(msg, msg_cap, b);
    }
  }

  // ---- uniqueness of the canonical identities
  std::unordered_map<State, uint64_t, StateHash, StateEq> where;
  where.reserve(n * 2);
  for (uint64_t i = 0; i < n; ++i) {
    auto ins = where.emplace(canon(S.at(i)), i);
    if (!ins.second) {
      snprintf(b, sizeof(b), "uniqueness: states %llu (level %u) and %llu (level %u) have the same canonical identity",
               (unsigned long long)ins.first->second, level[ins.first->second], (unsigned long long)i, level[i]);
      return report(msg, msg_cap, b);
    }
  }

  // ---- closure, totals and violators, over the expanded levels
  for (uint64_t i = 0; i < n; ++i) {
    const uint32_t L = level[i];
    const State s = S.at(i);
    // invariants of the stored states: checked by k_invariants at the end of the level that added them
    if (M::NUM_INVARIANTS > 0 && L - 1 <= n_expanded) {
      const int inv = M::first_violated_invariant(s);
      if (inv >= 0) V.add(L - 1, s, parents[i], (uint64_t)inv, 0);
    }
    if (L > n_expanded) continue;
    sink.clear();
    Groups<0>::run(s, site_gen, sink);
    if (sink.failed) {
      snprintf(b, sizeof(b), "closure: state %llu traps the layout (code %d)", (unsigned long long)i, sink.failed);
      return report(msg, msg_cap, b);
    }
    totals[0] += sink.out.size();
    if (sink.out.empty()) {
      totals[1]++;
      if (check_deadlock) V.add(L, s, parents[i], ~0ull, 0);
    }
    for (size_t k = 0; k < sink.out.size(); ++k) {
      const State& t = sink.out[k];
      act_gen[sink.act[k]]++;
      if (!kept(t)) {
        totals[2]++;
        if (M::NUM_INVARIANTS > 0) {
          const int inv = M::first_violated_invariant(t);
          if (inv >= 0) V.add(L, t, S.parent_ref(i) | ((uint64_t)sink.act[k] << 56), (uint64_t)inv, 1);
        }
        continue;
      }
      auto it = where.find(canon(t));
      if (it == where.end() || level[it->second] > L + 1) {
        snprintf(b, sizeof(b), "closure: successor [%s] (action %d) of state %llu (level %u) is %s", words_text(t).c_str(),
                 sink.act[k], (unsigned long long)i, L,
                 it == where.end() ? "not in the store" : ("stored at level " + std::to_string(level[it->second])).c_str());
        return report(msg, msg_cap, b);
      }
    }
  }
  return 0;
}

// the violator rows of the first level end with any, from the last audit_store call; returns the number of rows
uint64_t audit_violator_rows(uint64_t* out, uint64_t cap) {
  const uint64_t row = M::W + 3, n = g_viol_rows.size() / row;
  memcpy(out, g_viol_rows.data(), std::min(n, cap) * row * 8);
  return n;
}

// Level-ordered sequential BFS that writes its store like the engine: states in BFS order (level k contiguous), parent
// words index | action << 56 (NO_PARENT for initial states); the first member of an orbit found is the one stored.
// Stops at the first level end holding >= stop_after states (0: never).  Returns the number of stored states, or -1
// when `cap` is too small or the layout traps.  widths[] gets each level's size, *n_levels their number and
// *n_expanded how many of them were expanded.
int64_t audit_host_bfs(uint64_t* states, uint64_t* parents, uint64_t cap, uint64_t stop_after, uint64_t* widths,
                       uint32_t widths_cap, uint32_t* n_levels, uint32_t* n_expanded) {
  std::unordered_set<State, StateHash, StateEq> seen;
  uint64_t n = 0;
  auto push = [&](const State& s, uint64_t pw) {
    if (n >= cap) return false;
    memcpy(states + n * M::W, s.w, sizeof(s.w));
    parents[n++] = pw;
    return true;
  };
  for (int i = 0; i < M::NUM_INIT; ++i) {
    const State s = load(M::INIT_STATES[i]);
    if (kept(s) && seen.insert(canon(s)).second && !push(s, NO_PARENT)) return -1;
  }
  *n_levels = *n_expanded = 0;
  uint64_t first = 0;
  Sink sink;
  while (n > first) {
    if (*n_levels >= widths_cap) return -1;
    widths[(*n_levels)++] = n - first;
    if (stop_after && n >= stop_after) break;
    const uint64_t end = n;
    for (uint64_t i = first; i < end; ++i) {
      sink.clear();
      M::expand(load(states + i * M::W), sink);
      if (sink.failed) return -1;
      for (size_t k = 0; k < sink.out.size(); ++k)
        if (kept(sink.out[k]) && seen.insert(canon(sink.out[k])).second &&
            !push(sink.out[k], i | ((uint64_t)sink.act[k] << 56)))
          return -1;
    }
    (*n_expanded)++;
    first = end;
  }
  return (int64_t)n;
}
}  // extern "C"
