// Test harness (NOT a product path): a lowered model.h and its invariants.h compiled for the host, so that the tests can
// run the headers the CUDA engine includes on a machine without a GPU.  tests/support/hostmodel.py builds one library
// per header pair:
//   g++ -O2 -std=c++17 -shared -fPIC -DKMC_MODEL_HEADER='"model.h"' -DKMC_INVARIANTS_HEADER='"invariants.h"' host_model.cpp
// It holds
//   hm_*     the model's facts and per-state calls: successors under either form of Next, invariants (first violated and
//            the mask of all violated), constraints, initial states (either form of Init), canonical forms
//   hm_bfs   a level-ordered sequential BFS that stores its states as the engine does, with the run's statistics
//   audit_*  the whole-store audit of a finished or stopped GPU run
//   hs_*     a stand-in for one rank of the sharded engine (kafka_specification_b200/sharded.py's CPU tests)
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>
#include KMC_MODEL_HEADER
#include KMC_INVARIANTS_HEADER

namespace M = kmc_model;
using M::State;
namespace {
constexpr int W = M::W;
constexpr uint64_t NO_PARENT = 0x0000FFFFFFFFFFFFull;
constexpr uint64_t IDX_MASK = 0x000000FFFFFFFFFFull;

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
using StateSet = std::unordered_set<State, StateHash, StateEq>;

// successors and their action ids; `failed` keeps the code of a layout trap
struct Sink {
  std::vector<State> out;
  std::vector<int> act;
  int failed = 0;
  void emit(const State& n, int a) {
    out.push_back(n);
    act.push_back(a);
  }
  void fail(int code) { failed = code; }
};
// the two-phase form the expand kernel runs; with site_gen, each set bit of site_mask counts one successor of its site
template <int G>
struct Groups {
  static void run(const State& s, uint64_t* site_gen, Sink& sink) {
    const uint64_t m = M::site_mask(M::SiteGroupTag<G>{}, s);
    if (site_gen)
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
// the successors of s under expand() (sites = false) or the two-phase form, in place of sink's previous ones
void successors(const State& s, bool sites, Sink& sink, uint64_t* site_gen = nullptr) {
  sink.out.clear();
  sink.act.clear();
  if (sites) Groups<0>::run(s, site_gen, sink);
  else M::expand(s, sink);
}

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

// the engine's fingerprint and owner (kmc_engine.cu)
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
uint32_t owner_of(uint64_t fp, uint32_t world) { return (uint32_t)(((fp >> 32) * (uint64_t)world) >> 32); }
}  // namespace

// ================================================================================================ facts and one state
extern "C" {
int hm_words() { return W; }
int hm_state_bits() { return M::STATE_BITS; }
int hm_all_ones_possible() { return M::ALL_ONES_POSSIBLE ? 1 : 0; }
int hm_has_symmetry() { return M::HAS_SYMMETRY ? 1 : 0; }
int hm_num_actions() { return M::NUM_ACTIONS; }
int hm_num_sites() { return M::NUM_SITES; }
int hm_num_invariants() { return M::NUM_INVARIANTS; }
int hm_num_init() { return M::NUM_INIT; }
int hm_check_deadlock() { return M::CHECK_DEADLOCK ? 1 : 0; }
const char* hm_digest() { return KMC_MODEL_DIGEST; }
int hm_site_action(int i) { return M::SITE_ACTION[i]; }

// Returns the number of successors (also when it exceeds cap; then only cap rows are written), or -1 on a layout trap.
int hm_successors(const uint64_t* state, int sites, uint64_t* out, int* actions, int cap) {
  Sink sink;
  successors(load(state), sites != 0, sink);
  if (sink.failed) return -1;
  for (size_t k = 0; k < sink.out.size() && (int)k < cap; ++k) {
    memcpy(out + k * W, sink.out[k].w, sizeof(uint64_t) * W);
    actions[k] = sink.act[k];
  }
  return (int)sink.out.size();
}
int hm_first_violated(const uint64_t* state) { return M::first_violated_invariant(load(state)); }
uint64_t hm_mask(const uint64_t* state) { return M::violated_invariants(load(state)); }
int hm_in_model(const uint64_t* state) { return M::in_model(load(state)) ? 1 : 0; }
void hm_init_state(int i, uint64_t* out) { memcpy(out, M::INIT_STATES[i], sizeof(uint64_t) * W); }
void hm_canonicalize(const uint64_t* states, uint64_t n, uint64_t* out) {
  for (uint64_t i = 0; i < n; ++i) {
    const State c = canon(load(states + i * W));
    memcpy(out + i * W, c.w, sizeof(c.w));
  }
}
}  // extern "C"

// ================================================================================================ Init
// Both forms of Init as one list of generated initial states (duplicates included, as TLC counts them): the host
// form's INIT_STATES table, or every solution of every candidate of every branch of the device form, in branch and
// candidate order -- the order k_init counts them in, though it inserts them in any order.
namespace {
#ifdef KMC_HAS_DEVICE_INIT
constexpr int INIT_BRANCHES = M::INIT_BRANCHES;
uint64_t init_space(int b) { return M::INIT_SPACE[b]; }
#else
constexpr int INIT_BRANCHES = 0;
uint64_t init_space(int) { return 0; }
#endif
// 1: a solution, packed into s; 0: rejected by a filter; -code: a solution that traps the layout
int init_candidate(int b, uint64_t idx, State& s) {
#ifdef KMC_HAS_DEVICE_INIT
  unsigned fail = 0;
  memset(s.w, 0, sizeof(s.w));
  const bool ok = M::init_candidate(b, idx, s, fail);
  if (fail) return -(int)fail;
  return ok ? 1 : 0;
#else
  (void)b, (void)idx, (void)s;
  return 0;
#endif
}
// Calls f(state) for every generated initial state; returns 0, or the code of the first layout trap (and stops there).
template <class F>
int for_each_init(F&& f) {
  for (int i = 0; i < M::NUM_INIT; ++i) f(load(M::INIT_STATES[i]));
  State s;
  for (int b = 0; b < INIT_BRANCHES; ++b)
    for (uint64_t i = 0; i < init_space(b); ++i) {
      const int r = init_candidate(b, i, s);
      if (r < 0) return -r;
      if (r > 0) f(s);
    }
  return 0;
}
}  // namespace

extern "C" {
int hm_init_branches() { return INIT_BRANCHES; }
uint64_t hm_init_space(int b) { return b >= 0 && b < INIT_BRANCHES ? init_space(b) : 0; }
// Candidate idx of branch b of the device form: 1 (a solution, its words in out), 0 (rejected) or -code (a solution
// that does not fit the layout).
int hm_init_candidate(int b, uint64_t idx, uint64_t* out) {
  State s;
  const int r = init_candidate(b, idx, s);
  if (r > 0) memcpy(out, s.w, sizeof(s.w));
  return r;
}
// Every generated initial state of either form: the first `cap` of them into out, their number into *n; returns 0 or
// the code of a layout trap.
int hm_init_solutions(uint64_t* out, uint64_t cap, uint64_t* n) {
  *n = 0;
  return for_each_init([&](const State& s) {
    if (*n < cap) memcpy(out + *n * W, s.w, sizeof(s.w));
    ++*n;
  });
}
}  // extern "C"

// ================================================================================================ the BFS
namespace {
enum { T_GENERATED, T_DEADLOCKS, T_FAIL, T_COMPLETE, T_EXPANDED, T_MAX_FANOUT, T_FIRST_INV, T_FIRST_LEVEL, T_MISMATCHES,
       T_COUNT };
// The last hm_bfs run, which the caller copies out with hm_bfs_array.
struct Bfs {
  // generated (initial states included), deadlocks, fail code, complete, levels expanded, max fan-out,
  // first violated invariant (~0: none) and its level, checked states on which the mask and first_violated_invariant
  // disagree
  std::vector<uint64_t> totals;
  std::vector<uint64_t> states, parents, widths;   // the store: W words per state, parent words, level widths
  std::vector<uint64_t> act_gen, site_gen;         // successors generated per action / per emit site
  // per invariant, by first_violated_invariant: first violating level (0: never), violators
  std::vector<uint64_t> inv_level, inv_count;
  // per invariant, by the mask (what kmc_invariant_reports reports): first violating level (0: never), violators at
  // that level, violators over the run, smallest set-identity fingerprint among that level's violators
  std::vector<uint64_t> mask_level, mask_first_count, mask_count, mask_pick_fp;
};
Bfs g_bfs;
}  // namespace

extern "C" {
// Level-ordered sequential BFS (past violations, like -continue) that stores its states like the engine: in BFS order
// (level k contiguous), the first member of an orbit found, parent words index | action << 56 (NO_PARENT for initial
// states).  Successors come from expand() or, with sites, from the two-phase form, which also counts them per emit
// site.  Every initial state, stored state and out-of-model successor (at its parent's level + 1, each time it is
// generated) is checked against the invariants.  Stops, as incomplete, at the first level end that holds >= stop_at
// states (0: never) or at a layout trap.
void hm_bfs(int sites, uint64_t stop_at) {
  Bfs& B = g_bfs = Bfs();
  B.totals.assign(T_COUNT, 0);
  B.totals[T_COMPLETE] = 1;
  B.totals[T_FIRST_INV] = ~0ull;
  B.act_gen.assign(M::NUM_ACTIONS, 0);
  B.site_gen.assign(M::NUM_SITES, 0);
  B.inv_level.assign(M::NUM_INVARIANTS, 0);
  B.inv_count.assign(M::NUM_INVARIANTS, 0);
  for (auto* v : {&B.mask_level, &B.mask_first_count, &B.mask_count}) v->assign(M::NUM_INVARIANTS, 0);
  B.mask_pick_fp.assign(M::NUM_INVARIANTS, ~0ull);
  uint64_t* t = B.totals.data();
  StateSet seen;
  auto check = [&](const State& s, uint64_t level) {
    const uint64_t m = M::violated_invariants(s);
    const int inv = M::first_violated_invariant(s);
    if (m ? inv != __builtin_ctzll(m) : inv != -1) t[T_MISMATCHES]++;
    for (uint64_t b = m; b; b &= b - 1) {
      const int i = __builtin_ctzll(b);
      B.mask_count[i]++;
      if (!B.mask_level[i]) B.mask_level[i] = level;
      if (B.mask_level[i] != level) continue;
      B.mask_first_count[i]++;
      B.mask_pick_fp[i] = std::min(B.mask_pick_fp[i], fingerprint(canon(s)));
    }
    if (inv < 0) return;
    if (!B.inv_level[inv]) B.inv_level[inv] = level;
    B.inv_count[inv]++;
    if (t[T_FIRST_INV] == ~0ull) {
      t[T_FIRST_INV] = (uint64_t)inv;
      t[T_FIRST_LEVEL] = level;
    }
  };
  auto reach = [&](const State& s, uint64_t pw, uint64_t level) {
    if (!kept(s)) return check(s, level);
    if (!seen.insert(canon(s)).second) return;
    B.states.insert(B.states.end(), s.w, s.w + W);
    B.parents.push_back(pw);
    check(s, level);
  };
  // every solution of the device form is generated; one that does not fit the layout traps like a successor
  const int init_fail = for_each_init([&](const State& s) {
    t[T_GENERATED]++;
    reach(s, NO_PARENT, 1);
  });
  if (init_fail) {
    t[T_FAIL] = (uint64_t)init_fail;
    t[T_COMPLETE] = 0;
    return;
  }
  Sink sink;
  for (uint64_t first = 0; first < B.parents.size();) {
    const uint64_t end = B.parents.size(), level = B.widths.size() + 1;
    B.widths.push_back(end - first);
    if (stop_at && end >= stop_at) {
      t[T_COMPLETE] = 0;
      return;
    }
    for (uint64_t i = first; i < end; ++i) {
      successors(load(&B.states[i * W]), sites != 0, sink, B.site_gen.data());
      if (sink.failed) {
        t[T_FAIL] = (uint64_t)sink.failed;
        t[T_COMPLETE] = 0;
        return;
      }
      t[T_GENERATED] += sink.out.size();
      t[T_MAX_FANOUT] = std::max<uint64_t>(t[T_MAX_FANOUT], sink.out.size());
      if (sink.out.empty()) t[T_DEADLOCKS]++;
      for (size_t k = 0; k < sink.out.size(); ++k) {
        B.act_gen[sink.act[k]]++;
        reach(sink.out[k], i | ((uint64_t)sink.act[k] << 56), level + 1);
      }
    }
    t[T_EXPANDED]++;
    first = end;
  }
}
// One array of the last run, in the order of Bfs's fields (hostmodel.py's BFS_ARRAYS): its length in *n and its words,
// valid until the next hm_bfs or hm_bfs_clear.
const uint64_t* hm_bfs_array(int which, uint64_t* n) {
  std::vector<uint64_t>* v[] = {&g_bfs.totals,     &g_bfs.states,           &g_bfs.parents,    &g_bfs.widths,
                                &g_bfs.act_gen,    &g_bfs.site_gen,         &g_bfs.inv_level,  &g_bfs.inv_count,
                                &g_bfs.mask_level, &g_bfs.mask_first_count, &g_bfs.mask_count, &g_bfs.mask_pick_fp};
  *n = v[which]->size();
  return v[which]->data();
}
void hm_bfs_clear() { g_bfs = Bfs(); }
}  // extern "C"

// ================================================================================================ the store audit
// The audit checks, state by state, what the engine's bookkeeping claims about a store (the stored states and parent
// words of one rank, or the union of several ranks' stores, each state's BFS level and the number of expanded levels):
//   init        level 1 = the in-model initial states (INIT_STATES, or the device form's solutions), one per identity,
//               parent word NO_PARENT
//   edges       a state of level L >= 2 names a parent of level L-1 (rank, index), an action id < NUM_ACTIONS, and its
//               exact words are a successor of that parent labelled with that action, under expand() AND the two-phase
//               form
//   uniqueness  canonical identities are pairwise distinct
//   closure     every in-model successor of every expanded state of level L is stored at a level <= L+1
// and recomputes the run's totals (generated, deadlocks, out-of-model, per action, per emit site) and the violators the
// engine records at each level end.
namespace {
bool has_edge(const Sink& sink, const State& s, int action) {
  for (size_t k = 0; k < sink.out.size(); ++k)
    if (sink.act[k] == action && StateEq()(sink.out[k], s)) return true;
  return false;
}
std::string words_text(const State& s) {
  std::string t;
  char b[24];
  for (int i = 0; i < W; ++i) {
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
  State at(uint64_t i) const { return load(states + i * W); }
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
// Row: W words, parent word, invariant (~0 = deadlock).  The engine fingerprints every row by its canonical state.
struct ViolationSink {
  std::vector<uint64_t>* rows;   // the rows of the first level end that has any (so far)
  uint64_t* counts;              // [n_expanded + 1] violators per level end
  uint64_t first = ~0ull;
  void add(uint64_t e, const State& s, uint64_t meta, uint64_t inv) {
    counts[e]++;
    if (e > first) return;
    if (e < first) {
      rows->clear();
      first = e;
    }
    for (int k = 0; k < W; ++k) rows->push_back(s.w[k]);
    rows->push_back(meta);
    rows->push_back(inv);
  }
};
std::vector<uint64_t> g_viol_rows;
}  // namespace

// Above this many candidates the audit does not enumerate the device form of Init: the caller passes the initial states.
constexpr uint64_t AUDIT_MAX_INIT_CANDIDATES = 1ull << 32;

extern "C" {
// Returns 0 when every check passes, else 1 with "<check>: <what>" in msg.  level[i] is state i's BFS level (1 = Init);
// levels 1..n_expanded were expanded.  The generated initial states (duplicates included) are init_rows[n_init_rows]
// when init_rows is given, else the model's own (INIT_STATES, or every candidate of the device form up to
// AUDIT_MAX_INIT_CANDIDATES).  Outputs (also on failure, as far as computed):
//   totals[0] generated (initial states + successors of the expanded states)   totals[1] deadlocks of the expanded states
//   totals[2] out-of-model (initial states and successors)
//   act_gen[NUM_ACTIONS], site_gen[NUM_SITES]: successors per action / per emit site
//   viol_counts[n_expanded + 1]: violators recorded at each level end; audit_violator_rows then returns those of the
//   first level end that has any
int audit_store(const uint64_t* states, const uint64_t* parents, const uint32_t* level, uint64_t n, const uint64_t* rank_off,
                uint32_t n_ranks, uint32_t n_expanded, int check_deadlock, const uint64_t* init_rows, uint64_t n_init_rows,
                uint64_t* totals, uint64_t* act_gen, uint64_t* site_gen, uint64_t* viol_counts, char* msg, size_t msg_cap) {
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
  StateSet init_ids, init_words;
  auto add_init = [&](const State& s) {
    totals[0]++;
    if (!kept(s)) {
      totals[2]++;
      if (M::NUM_INVARIANTS > 0) {
        const int inv = M::first_violated_invariant(s);
        if (inv >= 0) V.add(0, s, NO_PARENT, (uint64_t)inv);
      }
      return;
    }
    init_words.insert(s);
    init_ids.insert(canon(s));
  };
  if (init_rows) {
    for (uint64_t i = 0; i < n_init_rows; ++i) add_init(load(init_rows + i * W));
  } else {
    uint64_t candidates = 0;
    for (int br = 0; br < INIT_BRANCHES; ++br) candidates += init_space(br);
    if (candidates > AUDIT_MAX_INIT_CANDIDATES) {
      snprintf(b, sizeof(b), "init: the device form has %llu candidates, more than the audit enumerates: pass the initial states",
               (unsigned long long)candidates);
      return report(msg, msg_cap, b);
    }
    if (const int code = for_each_init(add_init)) {
      snprintf(b, sizeof(b), "init: a solution of the device form traps the layout (code %d)", code);
      return report(msg, msg_cap, b);
    }
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
    if (!init_words.count(s) || parents[i] != NO_PARENT || !init_ids.count(canon(s))) {
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
      successors(p, false, sink);
      if (!has_edge(sink, s, (int)act)) bad = "names a parent whose expand() has no such successor under that action";
      successors(p, true, sink);
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
      if (inv >= 0) V.add(L - 1, s, parents[i], (uint64_t)inv);
    }
    if (L > n_expanded) continue;
    successors(s, true, sink, site_gen);
    if (sink.failed) {
      snprintf(b, sizeof(b), "closure: state %llu traps the layout (code %d)", (unsigned long long)i, sink.failed);
      return report(msg, msg_cap, b);
    }
    totals[0] += sink.out.size();
    if (sink.out.empty()) {
      totals[1]++;
      if (check_deadlock) V.add(L, s, parents[i], ~0ull);
    }
    for (size_t k = 0; k < sink.out.size(); ++k) {
      const State& t = sink.out[k];
      act_gen[sink.act[k]]++;
      if (!kept(t)) {
        totals[2]++;
        if (M::NUM_INVARIANTS > 0) {
          const int inv = M::first_violated_invariant(t);
          if (inv >= 0) V.add(L, t, S.parent_ref(i) | ((uint64_t)sink.act[k] << 56), (uint64_t)inv);
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
  const uint64_t row = W + 2, n = g_viol_rows.size() / row;
  memcpy(out, g_viol_rows.data(), std::min(n, cap) * row * 8);
  return n;
}
}  // extern "C"

// ================================================================================================ one sharded rank
// Stand-in for ONE RANK of the sharded engine: it gives the multi-rank driver (kafka_specification_b200/sharded.py)
// something to drive in the CPU-only gloo tests.  Same row format, set identity (the canonical form) and owner function
// as kmc_engine.cu, std::unordered_set instead of the HBM hash set.
namespace {
constexpr int ROW = W + 1;
struct Rank {
  uint32_t rank, world;
  StateSet seen;
  std::vector<State> store;
  std::vector<uint64_t> parent;
  State viol_state;
  uint64_t viol_meta = 0, viol_fp = ~0ull, viol_level = 0, level = 0;
  std::vector<std::vector<uint64_t>> cand;
  uint64_t generated = 0, deadlocks = 0, level_first = 0, level_count = 0;
  int64_t viol_inv = -1;
  int fail = 0;
  // one candidate row for the rank that owns s
  void send(const State& s, uint64_t meta) {
    const uint32_t d = world > 1 ? owner_of(fingerprint(canon(s)), world) : 0;
    cand[d].insert(cand[d].end(), s.w, s.w + W);
    cand[d].push_back(meta);
  }
};
}  // namespace

extern "C" {
void* hs_create(uint32_t rank, uint32_t world) {
  Rank* r = new Rank();
  r->rank = rank;
  r->world = world;
  r->cand.resize(world);
  return r;
}
void hs_destroy(void* h) { delete (Rank*)h; }
void hs_begin(void* h) {
  Rank* r = (Rank*)h;
  r->seen.clear();
  r->store.clear();
  r->parent.clear();
  r->viol_fp = ~0ull;
  r->viol_level = 0;
  r->level = 0;
  for (auto& c : r->cand) c.clear();
  r->generated = r->deadlocks = r->level_first = r->level_count = 0;
  r->viol_inv = -1;
  r->fail = 0;
}
void hs_seed_init(void* h) {
  Rank* r = (Rank*)h;
  if (r->rank != 0) return;
  for (int i = 0; i < M::NUM_INIT; ++i) {
    r->send(load(M::INIT_STATES[i]), NO_PARENT);
    r->generated++;
  }
}
void hs_reset_cand(void* h) {
  for (auto& c : ((Rank*)h)->cand) c.clear();
}
void hs_expand(void* h, uint64_t first, uint64_t count) {
  Rank* r = (Rank*)h;
  Sink sink;
  for (uint64_t i = first; i < first + count; ++i) {
    successors(r->store[i], false, sink);
    for (size_t k = 0; k < sink.out.size(); ++k) r->send(sink.out[k], i | ((uint64_t)r->rank << 40) | ((uint64_t)sink.act[k] << 56));
    r->generated += sink.out.size();
    if (sink.out.empty()) r->deadlocks++;
  }
  if (sink.failed) r->fail = sink.failed;
}
void hs_counts(void* h, uint64_t* out) {
  Rank* r = (Rank*)h;
  for (uint32_t d = 0; d < r->world; ++d) out[d] = r->cand[d].size() / ROW;
}
uint64_t* hs_send_ptr(void* h, uint32_t dest) { return ((Rank*)h)->cand[dest].data(); }
void hs_insert(void* h, const uint64_t* rows, uint64_t n) {
  Rank* r = (Rank*)h;
  for (uint64_t i = 0; i < n; ++i) {
    const State s = load(rows + i * ROW);
    const bool inmodel = M::in_model(s);
    const bool is_new = inmodel && r->seen.insert(canon(s)).second;
    const uint64_t meta = rows[i * ROW + W];
    if (is_new) {
      r->store.push_back(s);
      r->parent.push_back(meta);
    }
    if (is_new || !inmodel) {
      const int inv = M::first_violated_invariant(s);
      const uint64_t fp = fingerprint(canon(s));   // the engine's pick: by set identity, the orbit's under SYMMETRY
      if (inv >= 0 && (r->viol_inv < 0 || r->viol_level == r->level + 1) && fp < r->viol_fp) {
        if (r->viol_inv < 0) r->viol_level = r->level + 1;
        r->viol_inv = inv;
        r->viol_fp = fp;
        r->viol_state = s;
        r->viol_meta = meta;
      }
    }
  }
}
void hs_level_done(void* h, uint64_t* first, uint64_t* count) {
  Rank* r = (Rank*)h;
  r->level_first += r->level_count;
  r->level_count = r->store.size() - r->level_first;
  r->level++;
  *first = r->level_first;
  *count = r->level_count;
}
void hs_stats(void* h, uint64_t* out) {
  Rank* r = (Rank*)h;
  out[0] = r->store.size();
  out[1] = r->generated;
  out[2] = r->deadlocks;
  out[3] = (uint64_t)r->fail;
  out[4] = (uint64_t)r->viol_inv;
}
int hs_row_words() { return ROW; }
// violation record: out[0..W) words, out[W] parent word, out[W+1] fingerprint, out[W+2] level; returns invariant or -1
int hs_violation_record(void* h, uint64_t* out) {
  Rank* r = (Rank*)h;
  if (r->viol_inv < 0) return -1;
  memcpy(out, r->viol_state.w, sizeof(r->viol_state.w));
  out[W] = r->viol_meta;
  out[W + 1] = r->viol_fp;
  out[W + 2] = r->viol_level;
  return (int)r->viol_inv;
}
void hs_state_and_parent(void* h, uint64_t idx, uint64_t* out) {
  Rank* r = (Rank*)h;
  memcpy(out, r->store[idx].w, sizeof(uint64_t) * W);
  out[W] = r->parent[idx];
}
}  // extern "C"
