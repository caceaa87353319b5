// cpu_bfs.cpp -- the CPU arm of the benchmark (bench.py --impl reference, and bench.py's cpu_baseline leg).
//
// NOT a product path and not a checker: it exists to put an honest CPU number beside the GPU's.  The reference
// (hachikuji/kafka-specification) is TLA+ text whose executor, TLC (Java, third-party, not vendored, no JVM in this
// image), cannot run here; this file stands in for TLC's Worker loop the way TLC itself is organised
// (tlc2.tool.Worker.run: StateQueue.sDequeue -> Tool.getNextStates -> TLCState.fingerPrint -> FPSet.put ->
// invariants -> sEnqueue), with everything a fair CPU implementation would do:
//   * the SAME lowered Next / invariants / constraints the GPU runs (build/models/<m>/model.h compiled for the
//     host with -O3 -march=native), packed W-word states, no per-state allocation;
//   * a lock-free open-addressing table of 64-bit fingerprints (one CAS per new state, like TLC's OffHeapDiskFPSet);
//   * a persistent pool of worker threads, level-synchronous BFS, per-thread output buffers (no shared queue tail),
//     work handed out in chunks of 256 states.
// It keeps no state store and no parent links (a throughput run), so its memory is the table plus two frontiers.
//
// Build (bench.py does this):  g++ -O3 -march=native -std=c++20 -pthread -shared -fPIC
//                                  -DKMC_MODEL_HEADER='"build/models/<m>/model.h"' baseline/cpu_bfs.cpp -o ...
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <barrier>
#include <chrono>
#include <thread>
#include <vector>

#include KMC_MODEL_HEADER

namespace M = kmc_model;
using M::State;

namespace {

inline uint64_t mix64(uint64_t x) {
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdull;
  x ^= x >> 33;
  x *= 0xc4ceb9fe1a85ec53ull;
  x ^= x >> 33;
  return x;
}
inline uint64_t fingerprint(const State& s) {
  uint64_t h = 0x243F6A8885A308D3ull;
  for (int i = 0; i < M::W; ++i) h = mix64(h ^ s.w[i]) + 0x9E3779B97F4A7C15ull * (uint64_t)(i + 1);
  return h ? h : 1;
}

struct Table {
  std::atomic<uint64_t>* slots = nullptr;
  uint64_t mask = 0;
  // 1 = new, 0 = present, -1 = full
  int put(uint64_t fp) {
    uint64_t i = (fp ^ (fp >> 29)) & mask;
    for (uint64_t n = 0; n <= mask; ++n) {
      uint64_t v = slots[i].load(std::memory_order_relaxed);
      if (v == fp) return 0;
      if (v == 0) {
        uint64_t expect = 0;
        if (slots[i].compare_exchange_strong(expect, fp, std::memory_order_relaxed)) return 1;
        if (expect == fp) return 0;
      }
      i = (i + 1) & mask;
    }
    return -1;
  }
};

struct Sink {
  State out[M::MAX_FANOUT + 1];
  int n = 0;
  int failed = 0;
  void emit(const State& s, int) { if (n < M::MAX_FANOUT + 1) out[n++] = s; else failed = 99; }
  void fail(int code) { failed = code; }
};

struct Worker {
  std::vector<State> next;
  uint64_t generated = 0, fresh = 0, deadlocks = 0, out_of_model = 0;
  uint64_t viol[16] = {};
  int failed = 0;
};

}  // namespace

// stats: [0] distinct [1] generated [2] depth [3] deadlocks [4] fail code [5] complete [6] out_of_model
//        [7] nanoseconds of the search (first Init to empty queue; table allocation excluded)
//        [8] threads used   [16+i] states violating invariant i   [64+l] width of level l+1 (l < 192)
extern "C" int kmc_cpu_bfs(uint64_t* st, int threads, int table_log2, uint64_t stop_after_states) {
  memset(st, 0, 320 * sizeof(uint64_t));
  if (threads < 1) threads = (int)std::thread::hardware_concurrency();
  if (threads < 1) threads = 1;
  Table table;
  table.mask = (1ull << table_log2) - 1;
  table.slots = static_cast<std::atomic<uint64_t>*>(aligned_alloc(4096, (size_t)8 << table_log2));
  if (!table.slots) { st[4] = 3; return 1; }
  {
    // first touch in parallel (outside the timed region: the GPU arm's cudaMemset is outside its timing too)
    std::vector<std::thread> th;
    const size_t bytes = (size_t)8 << table_log2, per = bytes / threads;
    for (int t = 0; t < threads; ++t)
      th.emplace_back([&, t] { memset(reinterpret_cast<char*>(table.slots) + t * per, 0, t == threads - 1 ? bytes - t * per : per); });
    for (auto& x : th) x.join();
  }
  std::vector<Worker> ws(threads);
  std::vector<State> frontier;
  std::atomic<uint64_t> cursor{0};
  std::atomic<int> stop{0};
  uint64_t level = 1, distinct = 0;
  bool complete = true;

  auto t0 = std::chrono::steady_clock::now();
  // initial states (sequential): the table, or every solution of the device form of Init
  auto seed = [&](const State& s) {
    ws[0].generated++;
    if (M::NUM_CONSTRAINTS && !M::in_model(s)) { ws[0].out_of_model++; return; }
    State c;
    M::canonicalize(s, c);
    if (table.put(fingerprint(c)) == 1) {
      frontier.push_back(s);
      int inv = M::first_violated_invariant(s);
      if (inv >= 0 && inv < 16) ws[0].viol[inv]++;
    }
  };
#ifdef KMC_HAS_DEVICE_INIT
  for (int b = 0; b < M::INIT_BRANCHES; ++b)
    for (uint64_t i = 0; i < M::INIT_SPACE[b]; ++i) {
      State s;
      unsigned fail = 0;
      if (M::init_candidate(b, i, s, fail)) seed(s);
      if (fail) { st[4] = KMC_FAIL_LAYOUT; free(table.slots); return 1; }
    }
#else
  for (int i = 0; i < M::NUM_INIT; ++i) {
    State s;
    memcpy(s.w, M::INIT_STATES[i], sizeof(s.w));
    seed(s);
  }
#endif
  distinct = frontier.size();

  auto on_level_end = [&]() noexcept {
    // runs in exactly one thread while the others wait at the barrier
    uint64_t total = 0;
    for (auto& w : ws) total += w.next.size();
    if (level <= 192) st[64 + level - 1] = frontier.size();
    frontier.clear();
    frontier.reserve(total);
    for (auto& w : ws) {
      frontier.insert(frontier.end(), w.next.begin(), w.next.end());
      w.next.clear();
      if (w.failed && !st[4]) st[4] = (uint64_t)w.failed;
    }
    distinct += total;
    cursor.store(0, std::memory_order_relaxed);
    if (total == 0 || st[4]) stop.store(1);
    else {
      ++level;
      if (stop_after_states && distinct >= stop_after_states) { complete = false; stop.store(1); }
    }
  };
  std::barrier bar(threads, on_level_end);

  auto work = [&](int tid) {
    Worker& w = ws[tid];
    Sink sink;
    constexpr uint64_t CHUNK = 256;
    while (!stop.load(std::memory_order_relaxed)) {
      const uint64_t n = frontier.size();
      for (;;) {
        uint64_t b = cursor.fetch_add(CHUNK, std::memory_order_relaxed);
        if (b >= n) break;
        uint64_t e = b + CHUNK < n ? b + CHUNK : n;
        for (uint64_t i = b; i < e; ++i) {
          sink.n = 0;
          M::expand(frontier[i], sink);
          if (sink.failed) { w.failed = sink.failed; break; }
          w.generated += (uint64_t)sink.n;
          if (sink.n == 0) w.deadlocks++;
          for (int k = 0; k < sink.n; ++k) {
            const State& s = sink.out[k];
            if (M::NUM_CONSTRAINTS && !M::in_model(s)) {
              w.out_of_model++;
              int inv = M::first_violated_invariant(s);
              if (inv >= 0 && inv < 16) w.viol[inv]++;
              continue;
            }
            uint64_t fp;
            if (M::HAS_SYMMETRY) {
              State c;
              M::canonicalize(s, c);
              fp = fingerprint(c);
            } else {
              fp = fingerprint(s);
            }
            int r = table.put(fp);
            if (r < 0) { w.failed = 2; break; }
            if (r == 1) {
              int inv = M::first_violated_invariant(s);
              if (inv >= 0 && inv < 16) w.viol[inv]++;
              w.next.push_back(s);
            }
          }
        }
        if (w.failed) break;
      }
      bar.arrive_and_wait();
    }
  };
  if (distinct == 0) stop.store(1);
  std::vector<std::thread> pool;
  for (int t = 1; t < threads; ++t) pool.emplace_back(work, t);
  work(0);
  for (auto& x : pool) x.join();
  auto t1 = std::chrono::steady_clock::now();

  for (auto& w : ws) {
    st[1] += w.generated;
    st[3] += w.deadlocks;
    st[6] += w.out_of_model;
    for (int i = 0; i < 16; ++i) st[16 + i] += w.viol[i];
  }
  st[0] = distinct;
  st[2] = level;                     // levels expanded (Init = level 1); the last one produced no new state
  st[5] = (complete && !st[4]) ? 1 : 0;
  st[7] = (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(t1 - t0).count();
  st[8] = (uint64_t)threads;
  free(table.slots);
  return st[4] ? 1 : 0;
}
extern "C" int kmc_cpu_words() { return M::W; }
