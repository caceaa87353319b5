// kmc_engine.cu -- the BFS frontier-expansion engine, compiled once per lowered model:
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -shared -Xcompiler -fPIC \
//        -DKMC_NO_ONE_PHASE -include <model>.h kmc_engine.cu -o libkmc_<model>.so
//
// It replaces TLC's Worker next-state loop, FPSet and StateQueue (SURVEY.md section 8):
//
//   k_expand  (K1)  lowered Next over the frontier, in two phases per site group: every lane evaluates the
//                   complete path conditions of its states (site_mask), then warps run the straight-line
//                   bodies of the enabled (state, site) pairs one site at a time (site_body).  Successor
//                   rows (state words + parent/action word) are staged per warp in shared memory and
//                   flushed in bulk: straight into the set by the warp itself (kmc_run, one rank: K2's
//                   insert path runs inside K1, see Params::fused), into the local candidate buffer (the
//                   shard calls at world 1), into per-owner regions (NCCL exchange), or -- fused
//                   exchange -- straight into the owner rank's inbox through a peer mapping (NVLink stores).
//   k_insert  (K2)  one thread per candidate: identity (see state_ident), open-addressing hash set in HBM
//                   with 32-byte buckets (one DRAM sector), CAS insertion, warp ballot/popc compaction of
//                   the winners into the state store (= next frontier), parent link.  k_insert_inbox is
//                   the same over the regions the peers filled.
//   k_invariants (K3) the cfg's INVARIANTs on the new states of a level (compacted => every lane busy).
//                   Violating states (rare, terminal) go to a small ring; the host reports the one with
//                   the smallest fingerprint, so the counterexample is deterministic.  Under "continue",
//                   k_invariant_report then passes a level's violators through record_invariants: violators
//                   per invariant, and a second ring that holds the violators of invariants not reported
//                   yet, so that every invariant gets its own first level and counterexample.
//   k_edges (K5)    after a run (kmc_edges, TLC -dump dot): the candidate rows of a non-fused K1 over stored states
//                   turned into compacted edge rows (source index, source and successor fingerprints, action).
//
// DESIGN.md sections 3-4 give the layout, the kernels and their measurements.
//
// HBM layout (per rank):   table  2^table_log2 slots           8-byte fingerprints or 16-byte keys (see KEY128)
//                          store  u64[max_states][W]           all distinct states, BFS order;
//                                                              level k is a contiguous range
//                          parent u64[max_states]              parent ref | action << 56
//                          cand   u64[world][region_rows][W+1] successors of one frontier chunk
//
// There is no CPU fallback anywhere in this file: without a CUDA device kmc_create fails with
// KMC_E_NO_GPU.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <mutex>
#include <new>
#include <thread>
#include <string>
#include <tuple>
#include <vector>

#include "kspecmc.h"

namespace M = kmc_model;
using M::State;

static constexpr int W = M::W;
static constexpr int ROW = W + 1;
static constexpr int MAX_WORLD = 8;
static constexpr uint64_t NO_PARENT = 0x0000FFFFFFFFFFFFull;
static constexpr uint64_t IDX_MASK = 0x000000FFFFFFFFFFull;
static constexpr bool EXACT64 = (M::STATE_BITS <= 63);
static_assert(M::NUM_ACTIONS <= 255, "the parent word holds the action id in 8 bits");

#define KMC_FAIL_TABLE_FULL 2
#define KMC_FAIL_STORE_FULL 3
#define KMC_FAIL_CAND_FULL 4
#define KMC_FAIL_PEER_TIMEOUT 5
#define KMC_FAIL_SET_TIMEOUT 6

// ----------------------------------------------------------------------------------------
// fingerprints
// ----------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint64_t fmix64(uint64_t x) {
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdull;
  x ^= x >> 33;
  x *= 0xc4ceb9fe1a85ec53ull;
  x ^= x >> 33;
  return x;
}

// Identity of a state in the set.
//   one-word models (<= 63 bits): the fingerprint is a bijection of the state, stored in 8-byte slots   -> exact
//   two-word models             : the key IS the packed state (16-byte slots, 128-bit CAS)              -> exact
//                                 (all-ones marks an empty slot; the lowering proves no valid state packs to it)
//   wider models                : a 128-bit fingerprint (two independent 64-bit chains) in 16-byte slots;
//                                 collision probability ~ n^2 / 2^129 (TLC's FP64 contract squared)
// The 64-bit fingerprint also picks the bucket and the owner rank and orders counterexamples.
// The option "exact_set" makes the hashed forms exact too: the key is then the packed state (see XSLOT_WORDS).
static constexpr bool KEY128 = (W >= 2);
static constexpr bool EXACT_SET = EXACT64 || (W == 2 && !M::ALL_ONES_POSSIBLE);
static constexpr int BUCKET_SLOTS = KEY128 ? 2 : 4;      // one 32 B sector per bucket
static constexpr int SLOT_BYTES = KEY128 ? 16 : 8;

struct alignas(16) Key128 {
  unsigned long long lo, hi;
};
__host__ __device__ __forceinline__ bool key_eq(const Key128& a, const Key128& b) { return a.lo == b.lo && a.hi == b.hi; }
__host__ __device__ __forceinline__ bool key_empty(const Key128& a) { return (a.lo & a.hi) == ~0ull; }

// KMC_TEST_FP_BITS (tests only, never in a default build): the hashed fingerprint keeps only its low bits and the hashed
// 128-bit key none beyond them, so that distinct states collide and a set keyed by them visibly loses states.
#ifdef KMC_TEST_FP_BITS
static constexpr uint64_t TEST_FP_MASK = (1ull << KMC_TEST_FP_BITS) - 1, TEST_KEY_HI_MASK = 0;
#else
static constexpr uint64_t TEST_FP_MASK = ~0ull, TEST_KEY_HI_MASK = ~0ull;
#endif

__host__ __device__ __forceinline__ uint64_t fingerprint(const State& s) {
  if (EXACT64) return fmix64(s.w[0] + 1);
  uint64_t h = fmix64(s.w[0] + 0x9E3779B97F4A7C15ull);
#pragma unroll
  for (int i = 1; i < W; ++i) h = fmix64(h ^ (s.w[i] + 0x9E3779B97F4A7C15ull * (uint64_t)(i + 1)));
  h &= TEST_FP_MASK;
  return h ? h : 1;
}
__host__ __device__ __forceinline__ uint64_t fmix64b(uint64_t x) {     // a second, unrelated finaliser (splitmix64's)
  x ^= x >> 30;
  x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27;
  x *= 0x94d049bb133111ebull;
  x ^= x >> 31;
  return x;
}
__host__ __device__ __forceinline__ Key128 key_of(const State& s, uint64_t fp) {
  Key128 k;
  if (W == 2 && !M::ALL_ONES_POSSIBLE) {
    k.lo = s.w[0];
    k.hi = s.w[W - 1];
  } else {
    uint64_t h = fmix64b(s.w[0] ^ 0xD6E8FEB86659FD93ull);
#pragma unroll
    for (int i = 1; i < W; ++i) h = fmix64b((h << 7 | h >> 57) ^ s.w[i]);
    k.lo = fp;
    k.hi = h & TEST_KEY_HI_MASK;
    if (key_empty(k)) k.hi ^= 1;
  }
  return k;
}

// With SYMMETRY the identity is that of the orbit representative (smallest packed image under the symmetry
// group, TLC's symmetry reduction); the state that is stored, expanded and shown in traces stays the one that
// was actually reached.  canonicalize() is a few thousand instructions (n!-1 permuted images); kept out of
// line so that it exists once per kernel instead of once per call site (nvcc time of a symmetric model: 16 min -> 2 min).
struct Ident {
  uint64_t fp;
  Key128 key;
};
__host__ __device__ __noinline__ void canonical_ident(const State& s, Ident& id) {
  State c;
  M::canonicalize(s, c);
  id.fp = fingerprint(c);
  id.key = key_of(c, id.fp);
}
__host__ __device__ __forceinline__ Ident state_ident(const State& s) {
  Ident id;
  if (M::HAS_SYMMETRY) {
    canonical_ident(s, id);
  } else {
    id.fp = fingerprint(s);
    id.key = key_of(s, id.fp);
  }
  return id;
}
__host__ __device__ __forceinline__ uint64_t state_fp(const State& s) { return state_ident(s).fp; }

// exact_set: the key is the packed state itself -- the orbit representative under SYMMETRY -- and fp is state_fp's.
__host__ __device__ __noinline__ void canonical_xident(const State& s, State& key, uint64_t& fp) {
  M::canonicalize(s, key);
  fp = fingerprint(key);
}
__host__ __device__ __forceinline__ void state_xident(const State& s, State& key, uint64_t& fp) {
  if (M::HAS_SYMMETRY) {
    canonical_xident(s, key, fp);
  } else {
    key = s;
    fp = fingerprint(s);
  }
}

__host__ __device__ __forceinline__ uint32_t owner_of(uint64_t fp, uint32_t world) {
  return (uint32_t)(((fp >> 32) * (uint64_t)world) >> 32);
}

// ----------------------------------------------------------------------------------------
// device-side counters
// ----------------------------------------------------------------------------------------
struct DevCounters {
  unsigned long long cand_count[MAX_WORLD];
  unsigned long long store_tail;
  unsigned long long generated;
  unsigned long long deadlocks;
  unsigned long long out_of_model;
  unsigned long long probes;
  unsigned long long fail;
  unsigned long long max_fanout_seen;
  unsigned long long viol_count;         // rows claimed in the violator ring
  // coverage (TLC -coverage), kept over all levels of a run:
  unsigned long long site_generated[M::NUM_SITES > 0 ? M::NUM_SITES : 1];   // successors per emit site (K1's A1 totals)
  unsigned long long action_distinct[M::NUM_ACTIONS];   // new states per action (K2, from the winners' parent words)
  // per-invariant report (kmc_invariant_reports), kept by record_invariants when inv_on is set ("continue"):
  unsigned long long inv_on;
  unsigned long long inv_pending;        // invariants not reported yet: only their violators take rows (host-written)
  unsigned long long inv_new;            // pending invariants violated since the last level end
  unsigned long long inv_rows;           // rows claimed in the per-invariant ring since the last level end
  unsigned long long inv_staged;         // discarded violators staged since the last level end
  unsigned long long inv_viol_seen;      // viol_count at the last level end (host-written)
  unsigned long long inv_count[64];      // violators per invariant over the run
  unsigned long long set_count;          // set_spill: keys a flush range copied out, or states a filter piece kept
  // device Init (k_init): the candidates decoded and the solutions among them (also counted in `generated`)
  unsigned long long init_candidates;
  unsigned long long init_generated;
};

// Violating states are rare and terminal, so they go to a small ring: W state words, the
// parent/action word, the fingerprint and the invariant index (~0 = deadlock).  The host picks
// the entry with the smallest fingerprint -> the reported counterexample is deterministic
// (as long as the first violating level has <= VIOL_RING violators).  Every writer fingerprints
// the violator by its set identity (state_fp: the orbit representative under SYMMETRY), never by
// the stored orbit member, which is whichever insert won: the pick is then a choice among orbits.
static constexpr int VIOL_RING = 1 << 16;     // rows; (W + 3) * 8 bytes each: 2.6 MB for a two-word model
static constexpr int VIOL_ROW = W + 3;
// Under "continue" two more rings of the same size and row format follow in the same allocation: the per-invariant ring
// (the last word of a row is the set of pending invariants the state violates) and the stage of constraint-discarded
// violators.  The host empties both at every level end.
static constexpr bool INV_REPORT = M::HAS_INVARIANT_MASK && M::NUM_INVARIANTS > 0;
__host__ __device__ __forceinline__ uint64_t* inv_ring_of(uint64_t* viol_ring) { return viol_ring + (size_t)VIOL_RING * VIOL_ROW; }
__host__ __device__ __forceinline__ uint64_t* stage_ring_of(uint64_t* viol_ring) { return viol_ring + (size_t)2 * VIOL_RING * VIOL_ROW; }

struct Params {
  void* table;              // 8-byte slots (one-word models) or 16-byte slots
  uint64_t bucket_mask;     // #buckets - 1
  uint64_t* store;
  uint64_t* parent;
  uint64_t max_states;      // capacity of the device-resident store (a ring when spilling)
  uint64_t store_mask;      // spill: max_states - 1 (power of two), device slot = global index & mask; else ~0
  uint64_t store_base;      // spill: global index of the oldest state still on the device (older ones are on the host)
  uint64_t* cand;
  uint64_t region_rows;
  DevCounters* ctr;
  uint64_t* viol_ring;
  uint32_t rank, world;
  uint32_t check_deadlock;
  // fused exchange (world > 1, after kmc_shard_open_peers): every rank's inbox, mapped into this
  // process through CUDA IPC.  An inbox is two buffers (double buffering); a buffer is an 8-word
  // header (rows sent by each source rank) followed by world regions of region_rows rows.
  uint64_t* peer_inbox[MAX_WORLD];
  uint64_t inbox_stride;    // words per inbox buffer
  uint32_t p2p;             // 1: expand stores rows straight into the owners' inboxes
  uint32_t inbox_buf;       // which of the two buffers this round uses
  // 1 (kmc_run, one rank): expand inserts its successors itself (insert_stage) instead of writing them to `cand` for
  // k_insert.  The kernel then reads the frontier with __ldg while it appends new states to the same store; that is
  // sound because every new index lies at or beyond the end of the level being expanded, and the
  // `idx - store_base < max_states` check of insert_row keeps a spilling ring from wrapping onto live states.
  uint32_t fused;
  uint32_t exact;           // 1: the option "exact_set" on a model whose key is hashed (never set when EXACT_SET)
};

static constexpr int INBOX_HEADER = 8;
// Sync page in front of every rank's inbox (same allocation, so peers map it with the inbox).  Peers PUSH into it
// (posted NVLink stores) and its owner polls it locally:
//   ready[src]   round number src has finished storing rows (and their counts) for, into this rank's inbox
//   done[dst]    round number dst has finished inserting from ITS inbox (so its buffer of that round may be reused)
//   board[r][8]  rank r's level summary {level id, new states, violations, store tail, generated, fail, deadlocks,
//                pending invariants violated at this level}
// All counters are monotonic over the life of the context (never reset), so no reset can race with a peer.
static constexpr int SYNC_WORDS = 256;
static constexpr int SYNC_READY = 0, SYNC_DONE = 8, SYNC_BOARD = 16, BOARD_WORDS = 8;

__device__ __forceinline__ unsigned lane_id() {
  unsigned r;
  asm volatile("mov.u32 %0, %%laneid;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void reds_add64(uint32_t a, unsigned long long v) {     // shared-memory add, no return value
  asm volatile("red.shared.add.u64 [%0], %1;" ::"r"(a), "l"(v) : "memory");
}

// The per-invariant report of the invariant violators (`member`) among a warp's states under "continue"
// (k_invariant_report, for the stored states of a level and the staged successors): their violated invariants counted
// with one atomic per warp and invariant, and a row in the per-invariant ring for each one that violates an invariant
// still pending.  Called by all 32 lanes of a warp at a converged point.
__device__ __noinline__ void record_invariants(DevCounters* ctr, uint64_t* viol_ring, const State& s, uint64_t meta, uint64_t fp,
                                               bool member) {
  if (!INV_REPORT || !ctr->inv_on) return;
  const unsigned active = 0xffffffffu, lane = lane_id();
  const int leader = 0;
  const uint64_t m = member ? M::violated_invariants(s) : 0;
  uint64_t all = (uint64_t)__reduce_or_sync(active, (unsigned)m) | (uint64_t)__reduce_or_sync(active, (unsigned)(m >> 32)) << 32;
  while (all) {
    const int i = __ffsll((long long)all) - 1;
    all &= all - 1;
    const unsigned who = __ballot_sync(active, (m >> i) & 1);
    if ((int)lane == leader) atomicAdd(&ctr->inv_count[i], (unsigned long long)__popc(who));
  }
  const uint64_t mine = m & ctr->inv_pending;         // (constant while a kernel runs: the host writes it between levels)
  const unsigned writers = __ballot_sync(active, mine != 0);
  if (!writers) return;
  const uint64_t fresh = (uint64_t)__reduce_or_sync(active, (unsigned)mine) |
                         (uint64_t)__reduce_or_sync(active, (unsigned)(mine >> 32)) << 32;
  unsigned long long base = 0;
  if ((int)lane == leader) {
    atomicOr(&ctr->inv_new, (unsigned long long)fresh);
    base = atomicAdd(&ctr->inv_rows, (unsigned long long)__popc(writers));
  }
  base = __shfl_sync(active, base, leader);
  if (!mine) return;
  const unsigned long long slot = base + __popc(writers & ((1u << lane) - 1));
  if (slot >= (unsigned long long)VIOL_RING) return;
  uint64_t* row = inv_ring_of(viol_ring) + slot * VIOL_ROW;
#pragma unroll
  for (int k = 0; k < W; ++k) row[k] = s.w[k];
  row[W] = meta;
  row[W + 1] = fp;
  row[W + 2] = mine;
}

// Out of line (rare, terminal), so it takes the two pointers it uses by value: a `const Params&` argument would make
// the caller keep a copy of the kernel parameters in local memory and reach them through generic loads.
__device__ __noinline__ void record_violation(DevCounters* ctr, uint64_t* viol_ring, const State& s, uint64_t meta, uint64_t fp,
                                              uint64_t inv) {
  unsigned long long slot = atomicAdd(&ctr->viol_count, 1ull);
  if (slot >= (unsigned long long)VIOL_RING) return;
  uint64_t* row = viol_ring + slot * VIOL_ROW;
#pragma unroll
  for (int k = 0; k < W; ++k) row[k] = s.w[k];
  row[W] = meta;
  row[W + 1] = fp;
  row[W + 2] = inv;
}

// A successor a CONSTRAINT discards is not stored, so under "continue" a violating one is staged (W words, parent word,
// fingerprint) for k_invariant_report.  Kept apart from record_invariants: evaluating every invariant here would
// raise the register use of this call, and with it the spills of the expand kernel that inserts successors itself.
__device__ __noinline__ void stage_violator(DevCounters* ctr, uint64_t* viol_ring, const State& s, uint64_t meta, uint64_t fp) {
  if (!INV_REPORT || !ctr->inv_on) return;
  const unsigned long long slot = atomicAdd(&ctr->inv_staged, 1ull);
  if (slot >= (unsigned long long)VIOL_RING) return;
  uint64_t* row = stage_ring_of(viol_ring) + slot * VIOL_ROW;
#pragma unroll
  for (int k = 0; k < W; ++k) row[k] = s.w[k];
  row[W] = meta;
  row[W + 1] = fp;
}

// ----------------------------------------------------------------------------------------
// K2 primitives: the fingerprint set
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ ulonglong2 ld_cg128(const void* p) {
  // L2-coherent 128-bit load, no L1 allocation: buckets are touched once per probe
  ulonglong2 v;
  asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p));
  return v;
}

__device__ __forceinline__ uint64_t bucket_of(uint64_t fp, uint64_t bucket_mask) { return (fp ^ (fp >> 31)) & bucket_mask; }

// One bucket = BUCKET_SLOTS slots, loaded with 128-bit loads: 8-byte slots -> 2 loads of 2 slots each (32 B);
// 16-byte slots -> one load per slot.
static constexpr int BUCKET_LOADS = KEY128 ? BUCKET_SLOTS : 2;
struct Bucket {
  ulonglong2 v[BUCKET_LOADS];
};
__device__ __forceinline__ const char* bucket_addr(const void* table, uint64_t b) {
  return static_cast<const char*>(table) + b * (uint64_t)(BUCKET_SLOTS * SLOT_BYTES);
}
__device__ __forceinline__ Bucket ld_bucket(const void* table, uint64_t b) {
  Bucket k;
  const char* base = bucket_addr(table, b);
#pragma unroll
  for (int i = 0; i < BUCKET_LOADS; ++i) k.v[i] = ld_cg128(base + 16 * i);
  return k;
}

// returns 1 = inserted (new), 0 = already present, -1 = table full.  `bk` = the first bucket, loaded by the
// caller ahead of time.  Correctness of the lock-free insert: slots never return to empty and every inserter
// of a key scans the same probe sequence without skipping an unverified slot, so a key occupies at most one
// slot; a stale read is harmless (the CAS decides).
__device__ __forceinline__ int set_insert_pre(void* table, uint64_t bucket_mask, const Ident& id, Bucket bk, unsigned& probes) {
  uint64_t b = bucket_of(id.fp, bucket_mask);
  for (int attempt = 0; attempt < 512; ++attempt) {
    if (attempt) bk = ld_bucket(table, b);
    ++probes;
    if constexpr (KEY128) {
      Key128* base = reinterpret_cast<Key128*>(const_cast<char*>(bucket_addr(table, b)));
#pragma unroll
      for (int k = 0; k < BUCKET_SLOTS; ++k)
        if (bk.v[k].x == id.key.lo && bk.v[k].y == id.key.hi) return 0;
#pragma unroll
      for (int k = 0; k < BUCKET_SLOTS; ++k) {
        if ((bk.v[k].x & bk.v[k].y) == ~0ull) {
          const Key128 empty{~0ull, ~0ull};
          Key128 old = atomicCAS(base + k, empty, id.key);          // ATOMG.E.CAS.128
          if (key_empty(old)) return 1;
          if (key_eq(old, id.key)) return 0;
          // another key took the slot: keep scanning (slots never empty again)
        }
      }
    } else {
      uint64_t* base = reinterpret_cast<uint64_t*>(const_cast<char*>(bucket_addr(table, b)));
      const uint64_t fp = id.fp;
      uint64_t v[4] = {bk.v[0].x, bk.v[0].y, bk.v[1].x, bk.v[1].y};
      if (v[0] == fp || v[1] == fp || v[2] == fp || v[3] == fp) return 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (v[k] == 0) {
          unsigned long long old = atomicCAS((unsigned long long*)(base + k), 0ull, (unsigned long long)fp);
          if (old == 0) return 1;
          if (old == fp) return 0;
        }
      }
    }
    b = (b + 1) & bucket_mask;
  }
  return -1;
}

__device__ __forceinline__ int set_insert(void* table, uint64_t bucket_mask, const Ident& id, unsigned& probes) {
  return set_insert_pre(table, bucket_mask, id, ld_bucket(table, bucket_of(id.fp, bucket_mask)), probes);
}

// returns the slot that holds the key (bucket * BUCKET_SLOTS + position), or -1 when it is absent
__device__ __forceinline__ long long set_contains(const void* table, uint64_t bucket_mask, const Ident& id) {
  uint64_t b = bucket_of(id.fp, bucket_mask);
  for (int attempt = 0; attempt < 512; ++attempt) {
    Bucket bk = ld_bucket(table, b);
    bool any_empty = false;
    const long long first = (long long)(b * BUCKET_SLOTS);
    if constexpr (KEY128) {
#pragma unroll
      for (int k = 0; k < BUCKET_SLOTS; ++k) {
        if (bk.v[k].x == id.key.lo && bk.v[k].y == id.key.hi) return first + k;
        any_empty |= (bk.v[k].x & bk.v[k].y) == ~0ull;
      }
    } else {
      const uint64_t fp = id.fp;
      const uint64_t v[4] = {bk.v[0].x, bk.v[0].y, bk.v[1].x, bk.v[1].y};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (v[k] == fp) return first + k;
        any_empty |= v[k] == 0;
      }
    }
    if (any_empty) return -1;
    b = (b + 1) & bucket_mask;
  }
  return -1;
}

// ---- exact_set: the key is the packed state (DESIGN.md section 4, "Identity of a state") ----------------------------
// A slot is a header word and the W words of the key, padded to 16 B (W = 1: two slots per 32 B bucket), 32 B (W = 2, 3)
// or 64 B (W = 4 .. 7: one bucket of two sectors).  Header: XEMPTY, then CLAIMED (tag = fp & ~3: the claimer is writing
// the words), then PUBLISHED (tag | 1).  Neither can be all-ones (bit 0 clear; bit 1 clear), so the table's empty marker
// is the all-ones fill of the 16-byte form.  A slot is claimed by one CAS on its header and never changes key.
// XS_ON is `true` only where the option can do anything: models whose key is exact already compile no exact_set code.
static constexpr bool XS_ON = !EXACT_SET;
static constexpr int XSLOT_WORDS = W == 1 ? 2 : (W <= 3 ? 4 : 8);
static constexpr int XBUCKET_SLOTS = W == 1 ? 2 : 1;
static constexpr int XSLOT_BYTES = XSLOT_WORDS * 8;
static constexpr int XPROBE_BUCKETS = 1024 / XBUCKET_SLOTS;     // the same 1024 slots as the 16-byte form's 512 buckets
static constexpr uint64_t XEMPTY = ~0ull;
static constexpr int XWAIT_ROUNDS = 1 << 20;                    // of >= 64 ns: a publish not seen in ~0.1 s fails the run

__device__ __forceinline__ uint64_t* xslot_addr(const void* table, uint64_t b, int k) {
  return const_cast<uint64_t*>(static_cast<const uint64_t*>(table)) + (b * XBUCKET_SLOTS + k) * XSLOT_WORDS;
}
// the first sector of bucket b: the header of each of its slots (v[k].x for W = 1, v[0].x otherwise)
__device__ __forceinline__ Bucket ld_xbucket(const void* table, uint64_t b) {
  Bucket k;
  const char* base = reinterpret_cast<const char*>(xslot_addr(table, b, 0));
#pragma unroll
  for (int i = 0; i < BUCKET_LOADS; ++i) k.v[i] = ld_cg128(base + 16 * i);
  return k;
}
__device__ __forceinline__ uint64_t xheader(const Bucket& bk, int k) { return W == 1 && k ? bk.v[1].x : bk.v[0].x; }
__device__ __forceinline__ uint64_t ld_acquire64(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release64(uint64_t* p, uint64_t v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t ld_cg64(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.global.cg.u64 %0, [%1];" : "=l"(v) : "l"(p));
  return v;
}

// A slot whose header carries the key's tag: 1 when it holds the key, 0 when another key, -2 when its claimer has not
// published within XWAIT_ROUNDS.  The words are read after an acquire load that saw the header published, so they are
// the claimer's words, never a half-written slot.
__device__ __noinline__ int xslot_match(const uint64_t* slot, const State& key) {
  uint64_t h = ld_acquire64(slot);
  for (int i = 0; !(h & 1); ++i) {
    if (i == XWAIT_ROUNDS) return -2;
    __nanosleep(64);
    h = ld_acquire64(slot);
  }
  bool eq = true;
#pragma unroll
  for (int w = 0; w < W; ++w) eq &= ld_cg64(slot + 1 + w) == key.w[w];
  return eq ? 1 : 0;
}

// returns 1 = inserted (new), 0 = already present, -1 = table full, -2 = a publish was never seen.  `bk` = the first
// bucket's headers, loaded by the caller ahead of time.  Every inserter of a key scans the same slots in the same order
// and passes a slot only when it is verified to hold another key (a different tag, or the published words differ), so a
// key occupies at most one slot; a stale header is harmless (the CAS decides, and a tag never changes).
__device__ __forceinline__ int xset_insert(void* table, uint64_t bucket_mask, uint64_t fp, const State& key, Bucket bk,
                                           unsigned& probes) {
  const uint64_t tag = fp & ~3ull;
  uint64_t b = bucket_of(fp, bucket_mask);
  for (int attempt = 0; attempt < XPROBE_BUCKETS; ++attempt) {
    ++probes;
#pragma unroll
    for (int k = 0; k < XBUCKET_SLOTS; ++k) {
      uint64_t* slot = xslot_addr(table, b, k);
      uint64_t h = attempt ? ld_cg64(slot) : xheader(bk, k);
      if (h == XEMPTY) {
        h = atomicCAS(reinterpret_cast<unsigned long long*>(slot), (unsigned long long)XEMPTY, (unsigned long long)tag);
        if (h == XEMPTY) {
#pragma unroll
          for (int w = 0; w < W; ++w) slot[1 + w] = key.w[w];
          st_release64(slot, tag | 1);        // the words are visible to whoever sees the header published
          return 1;
        }
      }
      if ((h & ~1ull) != tag) continue;       // another key
      const int m = xslot_match(slot, key);
      if (m) return m > 0 ? 0 : m;
    }
    b = (b + 1) & bucket_mask;
  }
  return -1;
}

// the slot that holds the key, or -1.  Only called while no insert runs (every claimed slot is published), and an
// empty slot ends the probe: an inserter never passes one.
__device__ __forceinline__ long long xset_contains(const void* table, uint64_t bucket_mask, uint64_t fp, const State& key) {
  const uint64_t tag = fp & ~3ull;
  uint64_t b = bucket_of(fp, bucket_mask);
  for (int attempt = 0; attempt < XPROBE_BUCKETS; ++attempt) {
#pragma unroll
    for (int k = 0; k < XBUCKET_SLOTS; ++k) {
      const uint64_t* slot = xslot_addr(table, b, k);
      const uint64_t h = ld_cg64(slot);
      if (h == XEMPTY) return -1;
      if ((h & ~1ull) == tag && xslot_match(slot, key) > 0) return (long long)(b * XBUCKET_SLOTS + k);
    }
    b = (b + 1) & bucket_mask;
  }
  return -1;
}

// Warp-collective insert of one candidate row per lane (invalid lanes pass valid = false):
// constraint check, identity, bucket probe + CAS, ballot/popc compaction of the winners into the
// state store, parent link.
// XS: the exact_set form, which carries the key (the packed state, canonical under SYMMETRY) instead of Ident::key.
template <bool XS = false>
struct Prefetched {
  Ident id;
  Bucket bk;
  bool inmodel;
};
template <>
struct Prefetched<true> {
  Ident id;
  Bucket bk;
  bool inmodel;
  State key;
};

// first half of an insert: identity + issue the bucket loads (no dependent use yet)
template <bool XS = false>
__device__ __forceinline__ Prefetched<XS> prefetch_row(const Params& p, const State& s, bool valid) {
  Prefetched<XS> f;
  f.id.fp = 0;
  f.id.key = Key128{0, 0};
#pragma unroll
  for (int i = 0; i < BUCKET_LOADS; ++i) f.bk.v[i] = make_ulonglong2(0, 0);
  f.inmodel = false;
  if constexpr (XS) {
    f.key = s;
    if (valid) {
      f.inmodel = (M::NUM_CONSTRAINTS == 0) || M::in_model(s);
      state_xident(s, f.key, f.id.fp);
      if (f.inmodel) f.bk = ld_xbucket(p.table, bucket_of(f.id.fp, p.bucket_mask));
    }
  } else if (valid) {
    f.inmodel = (M::NUM_CONSTRAINTS == 0) || M::in_model(s);
    f.id = state_ident(s);
    if (f.inmodel) f.bk = ld_bucket(p.table, bucket_of(f.id.fp, p.bucket_mask));
  }
  return f;
}

// CTA_ACTIONS: the new states per action go to this CTA's shared-memory counters at `act_smem` (u64 per action, the
// fused expand kernel flushes them once at its end) instead of one global atomic per action and warp.
template <bool CTA_ACTIONS = false, bool XS = false>
__device__ __forceinline__ void insert_row(const Params& p, const State& s, uint64_t meta, bool valid, const Prefetched<XS>& f,
                                            unsigned& probes, unsigned& oom, int& failed, uint32_t act_smem = 0) {
  bool is_new = false;
  if (valid) {
    if (f.inmodel) {
      int r;
      if constexpr (XS) {
        r = xset_insert(p.table, p.bucket_mask, f.id.fp, f.key, f.bk, probes);
        if (r < 0) failed = r == -1 ? KMC_FAIL_TABLE_FULL : KMC_FAIL_SET_TIMEOUT;
      } else {
        r = set_insert_pre(p.table, p.bucket_mask, f.id, f.bk, probes);
        if (r < 0) failed = KMC_FAIL_TABLE_FULL;
      }
      is_new = r > 0;
    } else {
      ++oom;
      // TLC also checks invariants on successors discarded by a CONSTRAINT; they are not stored,
      // so that (rare) case is handled here.  New in-model states are checked by k_invariants (K3).
      if (M::NUM_INVARIANTS > 0) {
        int inv = M::first_violated_invariant(s);
        if (inv >= 0) {
          record_violation(p.ctr, p.viol_ring, s, meta, f.id.fp, (uint64_t)inv);
          stage_violator(p.ctr, p.viol_ring, s, meta, f.id.fp);
        }
      }
    }
  }
  unsigned mask = __ballot_sync(0xffffffffu, is_new);
  if (mask) {
    unsigned lane = lane_id();
    int leader = __ffs(mask) - 1;
    unsigned long long base = 0;
    if ((int)lane == leader) base = atomicAdd(&p.ctr->store_tail, (unsigned long long)__popc(mask));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (is_new) {
      // coverage: distinct states per action = the action bits of the winners' parent words (initial states have
      // none); one atomic per action present among the warp's winners
      const unsigned act = ((meta & 0x0000FFFFFFFFFFFFull) == NO_PARENT) ? ~0u : (unsigned)(meta >> 56);
      const unsigned same = __match_any_sync(mask, act);
      if (act < (unsigned)M::NUM_ACTIONS && (int)lane == __ffs(same) - 1) {
        if (CTA_ACTIONS) reds_add64(act_smem + act * 8, (unsigned long long)__popc(same));
        else atomicAdd(&p.ctr->action_distinct[act], (unsigned long long)__popc(same));
      }
      uint64_t idx = base + __popc(mask & ((1u << lane) - 1));
      if (idx - p.store_base < p.max_states) {
        uint64_t* dst = p.store + (idx & p.store_mask) * W;
#pragma unroll
        for (int k = 0; k < W; ++k) dst[k] = s.w[k];
        p.parent[idx & p.store_mask] = meta;
      } else {
        failed = KMC_FAIL_STORE_FULL;
      }
    }
  }
}

// ----------------------------------------------------------------------------------------
// K1: expand
// ----------------------------------------------------------------------------------------
// Successor rows are staged per warp in shared memory and flushed in bulk: one global slot claim
// per flush (instead of one ~600-cycle atomic round trip per emit site), coalesced row stores,
// and -- multi-rank -- the owner computation (a fingerprint) done with all 32 lanes busy instead
// of inside the emit site.  The stage is addressed through 32-bit shared-window addresses and
// st.shared / atom.shared so that no generic-address store (ST + QSPC) is ever generated.
static constexpr int EXPAND_BLOCK = 1024;        // one CTA per SM
static constexpr int NWARPS = EXPAND_BLOCK / 32;
static constexpr int STAGE_ROWS = 64;            // rows per warp; a body pass adds <= 32, a flush empties it
static constexpr int STAGE_FLUSH = 32;           // flush once at least this many rows are staged
static constexpr int LIST_CAP = 12288;           // (state, site) pairs of one scatter round, 16-bit tile slots
static constexpr int MAX_GROUP_SITES = 64;

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void sts64(uint32_t a, uint64_t v) { asm volatile("st.shared.u64 [%0], %1;" ::"r"(a), "l"(v) : "memory"); }
__device__ __forceinline__ uint64_t lds64(uint32_t a) {
  uint64_t v;
  asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ unsigned atoms_add(uint32_t a, unsigned v) {
  unsigned old;
  asm volatile("atom.shared.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(a), "r"(v) : "memory");
  return old;
}

// one row per lane (valid lanes only) into the owner's region, slot claims aggregated per owner
__device__ __forceinline__ void claim_and_store(const Params& p, const State& s, uint64_t meta, bool valid, int& failed) {
  uint32_t dest = 0xFFu;
  if (valid) dest = owner_of(state_fp(s), p.world);
  unsigned peers = __match_any_sync(0xffffffffu, dest);
  unsigned lane = lane_id();
  int leader = __ffs(peers) - 1;
  unsigned long long base = 0;
  if (valid && (int)lane == leader) base = atomicAdd(&p.ctr->cand_count[dest], (unsigned long long)__popc(peers));
  base = __shfl_sync(0xffffffffu, base, leader);
  if (!valid) return;
  unsigned long long pos = base + __popc(peers & ((1u << lane) - 1));
  if (pos >= p.region_rows) {
    failed = KMC_FAIL_CAND_FULL;
    return;
  }
  // p2p: the row goes straight into region `rank` of the owner's inbox (a peer store over NVLink
  // when dest != rank); otherwise into the local per-owner candidate region for a later exchange
  uint64_t* row = p.p2p ? p.peer_inbox[dest] + (uint64_t)p.inbox_buf * p.inbox_stride + INBOX_HEADER +
                              ((uint64_t)p.rank * p.region_rows + pos) * ROW
                        : p.cand + ((uint64_t)dest * p.region_rows + pos) * ROW;
#pragma unroll
  for (int i = 0; i < W; ++i) row[i] = s.w[i];
  row[W] = meta;
}

// Per-CTA counters of the fused insert, u64 each in shared memory, flushed with one global atomic each at the end of
// k_expand: probes, out-of-model successors, successors generated (the candidate-region check) and new states per action.
static constexpr int CTA_PROBES = 0, CTA_OOM = 1, CTA_GEN = 2, CTA_ACTION = 3;
static constexpr int CTA_CTR_BYTES = (CTA_ACTION + M::NUM_ACTIONS) * 8;

// Fused expand + insert (p.fused): the warp inserts its staged rows itself, one row per lane and round, through the
// insert path of k_insert -- constraint and out-of-model invariant check, identity, probe + CAS, ballot compaction
// into the store, parent word.  Out of line, so that it exists once in k_expand instead of once per site group and
// its registers are not live across the bodies.  Called by all 32 lanes of a warp (n is warp-uniform).
// It gets the kernel parameters it reads by value, in registers: with a `const Params&` argument the caller kept a copy
// of Params in local memory and the insert reached every pointer through a generic load ahead of its first probe.
template <bool XS = false>
__device__ __noinline__ int insert_stage(void* table, uint64_t bucket_mask, uint64_t* store, uint64_t* parent,
                                         uint64_t max_states, uint64_t store_mask, uint64_t store_base, DevCounters* ctr,
                                         uint64_t* viol_ring, uint32_t wbuf, unsigned n, uint32_t cta) {
  Params p{};          // a value: only the fields above are read, and it is never addressed
  p.table = table;
  p.bucket_mask = bucket_mask;
  p.store = store;
  p.parent = parent;
  p.max_states = max_states;
  p.store_mask = store_mask;
  p.store_base = store_base;
  p.ctr = ctr;
  p.viol_ring = viol_ring;
  unsigned probes = 0, oom = 0;
  int failed = 0;
  const unsigned lane = lane_id();
  for (unsigned r0 = 0; r0 < n; r0 += 32) {
    const unsigned r = r0 + lane;
    const bool valid = r < n;
    const uint32_t row = wbuf + (valid ? r : 0) * (ROW * 8);
    State s;
#pragma unroll
    for (int k = 0; k < W; ++k) s.w[k] = lds64(row + k * 8);
    const uint64_t meta = lds64(row + W * 8);
    const Prefetched<XS> f = prefetch_row<XS>(p, s, valid);
    insert_row<true, XS>(p, s, meta, valid, f, probes, oom, failed, cta + CTA_ACTION * 8);
  }
  probes = __reduce_add_sync(0xffffffffu, probes);
  oom = __reduce_add_sync(0xffffffffu, oom);
  if (lane == 0) {
    if (probes) reds_add64(cta + CTA_PROBES * 8, probes);
    if (oom) reds_add64(cta + CTA_OOM * 8, oom);
  }
  return failed;
}

// insert_stage of a warp's n staged rows at `wbuf`, into the set form the context uses
__device__ __forceinline__ int insert_stage_of(const Params& p, uint32_t wbuf, unsigned n, uint32_t cta) {
  if constexpr (XS_ON) {
    if (p.exact)
      return insert_stage<XS_ON>(p.table, p.bucket_mask, p.store, p.parent, p.max_states, p.store_mask, p.store_base, p.ctr,
                                 p.viol_ring, wbuf, n, cta);
  }
  return insert_stage(p.table, p.bucket_mask, p.store, p.parent, p.max_states, p.store_mask, p.store_base, p.ctr,
                      p.viol_ring, wbuf, n, cta);
}

// called by all 32 lanes of a warp at a converged point
__device__ __forceinline__ void flush_stage(const Params& p, uint32_t wbuf, uint32_t wcnt, uint32_t cta, bool force, int& failed) {
  __syncwarp();
  unsigned n;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(n) : "r"(wcnt));
  if (n > (unsigned)STAGE_ROWS) n = STAGE_ROWS;
  if (n == 0 || (!force && n < (unsigned)STAGE_FLUSH)) return;
  unsigned lane = lane_id();
  if (p.fused) {
    const int f = insert_stage_of(p, wbuf, n, cta);
    if (f) failed = f;
  } else if (p.world == 1) {
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(&p.ctr->cand_count[0], (unsigned long long)n);
    base = __shfl_sync(0xffffffffu, base, 0);
    if (base + n > p.region_rows) {
      failed = KMC_FAIL_CAND_FULL;
    } else {
      uint64_t* dst = p.cand + base * ROW;
      for (unsigned k = lane; k < n * ROW; k += 32) dst[k] = lds64(wbuf + k * 8);      // coalesced
    }
  } else {
    for (unsigned r0 = 0; r0 < n; r0 += 32) {
      unsigned r = r0 + lane;
      bool valid = r < n;
      State s;
      const uint32_t row = wbuf + (valid ? r : 0) * (ROW * 8);
#pragma unroll
      for (int k = 0; k < W; ++k) s.w[k] = lds64(row + k * 8);
      claim_and_store(p, s, lds64(row + W * 8), valid, failed);
    }
  }
  __syncwarp();
  if (lane == 0) asm volatile("st.shared.u32 [%0], %1;" ::"r"(wcnt), "r"(0u) : "memory");
  __syncwarp();
}

// The sink handed to the lowered bodies.  It holds values only (no reference to the kernel parameters and no
// out-of-line member): anything that makes the object addressable sends it -- and every pointer in it --
// through local memory and turns the stage stores / counter atomics into generic-address operations.
struct CandSink {
  uint64_t parent_ref;
  uint32_t wbuf;       // this warp's staging rows (shared-window address)
  uint32_t wcnt;       // rows staged by this warp (shared-window address)
  int n;
  int failed;

  __device__ __forceinline__ void emit(const State& s, int action) {
    ++n;
    const uint64_t meta = parent_ref | ((uint64_t)action << 56);
    unsigned active = __activemask();
    unsigned lane = lane_id();
    int leader = __ffs(active) - 1;
    unsigned base = 0;
    if ((int)lane == leader) base = atoms_add(wcnt, (unsigned)__popc(active));
    base = __shfl_sync(active, base, leader);
    unsigned pos = base + __popc(active & ((1u << lane) - 1));
    if (pos < (unsigned)STAGE_ROWS) {
      const uint32_t row = wbuf + pos * (ROW * 8);
#pragma unroll
      for (int i = 0; i < W; ++i) sts64(row + i * 8, s.w[i]);
      sts64(row + W * 8, meta);
    } else {
      // cannot happen (a body pass adds <= 32 rows to a stage that is flushed at >= STAGE_FLUSH)
      failed = KMC_FAIL_CAND_FULL;
    }
  }
  __device__ __forceinline__ void fail(int code) { failed = code; }
};

__device__ __forceinline__ void load_state(State& s, const uint64_t* src) {
#pragma unroll
  for (int k = 0; k < W; ++k) s.w[k] = __ldg(src + k);
}

// ----------------------------------------------------------------------------------------
// K1, two-phase.  The round-1 kernel ran every thread through the whole lowered Next of its own
// states: ncu showed 12 of 32 lanes per issued instruction, because an action body is enabled for
// a few per cent of the states of a warp.  Here the lowering provides, per site group (<= 64 emit
// sites), site_mask(s) = the COMPLETE path condition of every site (cheap compares, evaluated by
// all lanes on their own states) and site_body<i>(s) = the straight-line successor construction.
// One 1024-thread CTA per SM works on a tile of EXPAND_BLOCK x SPT states held in shared memory:
//   A1  every thread evaluates the group's masks for its SPT states; per-site totals via ballot/popc
//       and one shared-memory atomic per warp and site                                  -- barrier --
//   A2  every warp derives the same segment offsets from the totals (segments padded to 32) and
//       scatters its enabled (site, tile slot) pairs into the sorted list                -- barrier --
//   B   the list is consumed 32 entries at a time; a chunk belongs to exactly one site, so the body
//       dispatch is warp-uniform and the body runs with (almost) all lanes on the same code.
//       B of group g overlaps A1 of group g+1 (double-buffered totals): two barriers per group.
// Successor counts per state (deadlock detection, "states generated") are popc(mask).  The A1 totals are also the
// coverage counts: each CTA adds them up per emit site in shared memory and flushes them with one global atomic per
// site at the end of the kernel.
// ----------------------------------------------------------------------------------------
static constexpr int STAGE_BYTES = NWARPS * STAGE_ROWS * ROW * 8;
static constexpr int FIXED_SMEM_BYTES = STAGE_BYTES + LIST_CAP * 2 + (4 * MAX_GROUP_SITES + NWARPS + 8) * 4;
static constexpr int SPT_FIT = (227 * 1024 - 1024 - FIXED_SMEM_BYTES) / (EXPAND_BLOCK * W * 8);
static constexpr int SPT = SPT_FIT > 4 ? 4 : SPT_FIT;
// The widest state is 7 words: at W = 8 the warps' stage rows (32 x 64 rows of 9 words, 144 KB) and a tile of one state
// per thread (1024 x 8 words, 64 KB) exceed the 226 KB of shared memory a CTA can have.  The lowering refuses wider
// models with a message (lower/model.py, MAX_WORDS); W = 5, 6, 7 get SPT = 2, 1, 1.
static_assert(SPT >= 1, "state too wide for the expand kernel's shared-memory tile");
static constexpr int TILE = EXPAND_BLOCK * SPT;
static_assert(TILE <= LIST_CAP, "a site's segment (<= TILE pairs) must fit one scatter round");
// the per-site coverage counters and the fused insert's counters live in the slack the tile leaves (SPT is sized
// without them)
static constexpr int SITE_GEN_BYTES = (M::NUM_SITES > 0 ? M::NUM_SITES : 1) * 8;
static constexpr size_t EXPAND_SMEM_BYTES = (size_t)TILE * W * 8 + FIXED_SMEM_BYTES + SITE_GEN_BYTES + CTA_CTR_BYTES;
static_assert(EXPAND_SMEM_BYTES <= 227 * 1024 - 1024, "the per-CTA counters do not fit next to the expand tile");

struct TileCtx {
  uint32_t tile;        // [TILE][W] states (shared-window addresses throughout)
  uint32_t list;        // [LIST_CAP] u16 tile slots, per-site segments
  uint32_t cnt;         // [2][MAX_GROUP_SITES] enabled pairs per site (double-buffered across groups)
  uint32_t cur;         // [MAX_GROUP_SITES] scatter cursors
  uint32_t seg;         // [MAX_GROUP_SITES] first chunk of each site's segment
  uint32_t site_gen;    // [NUM_SITES] u64: successors this CTA generated per emit site
  uint32_t cta;         // the fused insert's counters (CTA_PROBES ...)
  uint32_t wbuf, wcnt;
  uint64_t first, tile_base;
  unsigned nvalid;      // states in this tile
};

template <int LO, int HI>
struct SiteDispatch {
  static __device__ __forceinline__ void run(int i, const State& s, CandSink& sink) {
    if constexpr (HI - LO == 1) {
      // the opaque copy keeps the compiler from hoisting every body's unpacking above the dispatch
      State t = s;
#pragma unroll
      for (int k = 0; k < W; ++k) asm volatile("" : "+l"(t.w[k]));
      M::site_body(M::SiteTag<LO>{}, t, sink);
    } else {
      constexpr int MID = (LO + HI) / 2;
      if (i < MID) SiteDispatch<LO, MID>::run(i, s, sink);
      else SiteDispatch<MID, HI>::run(i, s, sink);
    }
  }
};

__device__ __forceinline__ unsigned lds32(uint32_t a) {
  unsigned v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ void sts32(uint32_t a, unsigned v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }

template <int G>
struct SiteGroupRunner {
  static __device__ __forceinline__ void run(const Params& p, const TileCtx& c, unsigned (&nsucc)[SPT], int& failed) {
    constexpr int BEGIN = M::SITE_GROUP_BEGIN[G];
    constexpr int END = M::SITE_GROUP_BEGIN[G + 1];
    constexpr int NS = END - BEGIN;
    static_assert(NS >= 1 && NS <= MAX_GROUP_SITES, "site group size");
    const unsigned lane = lane_id();
    const unsigned warp = threadIdx.x >> 5;
    const uint32_t cnt = c.cnt + (G & 1) * (MAX_GROUP_SITES * 4);
    // ---- A1: masks of this thread's states; every enabled (state, site) pair bumps the site's total.
    // (One shared-memory atomic per pair: ~3 per state -- fewer instructions than a ballot/popc census over all
    // sites and states, which the first version of this kernel used.)
    uint64_t masks[SPT];
#pragma unroll
    for (int j = 0; j < SPT; ++j) {
      const unsigned slot = (unsigned)j * EXPAND_BLOCK + threadIdx.x;
      masks[j] = 0;
      if (slot < c.nvalid) {
        State s;
#pragma unroll
        for (int k = 0; k < W; ++k) s.w[k] = lds64(c.tile + (slot * W + k) * 8);
        masks[j] = M::site_mask(M::SiteGroupTag<G>{}, s);
        nsucc[j] += (unsigned)__popcll(masks[j]);
      }
    }
    // a state enables ~0.6 sites of a group on average: three predicated steps (no loop control, no
    // reconvergence stack) cover nearly every mask; the loop behind them is the rare tail
#pragma unroll
    for (int j = 0; j < SPT; ++j) {
      uint64_t m = masks[j];
#pragma unroll
      for (int it = 0; it < 3; ++it) {
        if (m) {
          atoms_add(cnt + (__ffsll((long long)m) - 1) * 4, 1u);
          m &= m - 1;
        }
      }
      while (m) {
        atoms_add(cnt + (__ffsll((long long)m) - 1) * 4, 1u);
        m &= m - 1;
      }
    }
    __syncthreads();                                   // totals complete; B of the previous group finished
    // coverage: thread k adds this tile's total of site BEGIN + k (no other thread touches that counter)
    if (threadIdx.x < (unsigned)NS) {
      const uint32_t a = c.site_gen + (BEGIN + threadIdx.x) * 8;
      sts64(a, lds64(a) + lds32(cnt + threadIdx.x * 4));
    }
    // the other totals buffer (read last by B of group G-1) is cleared for A1 of group G+1
    if (threadIdx.x < MAX_GROUP_SITES) sts32(c.cnt + ((G + 1) & 1) * (MAX_GROUP_SITES * 4) + threadIdx.x * 4, 0u);
    // ---- every warp: the same padded segment layout, sites 2*lane and 2*lane+1 per lane
    const unsigned c0 = (2 * lane < (unsigned)NS) ? lds32(cnt + (2 * lane) * 4) : 0u;
    const unsigned c1 = (2 * lane + 1 < (unsigned)NS) ? lds32(cnt + (2 * lane + 1) * 4) : 0u;
    const unsigned ch0 = (c0 + 31) >> 5, ch1 = (c1 + 31) >> 5;       // chunks of 32 pairs
    unsigned incl = ch0 + ch1;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      unsigned t = __shfl_up_sync(0xffffffffu, incl, o);
      if ((int)lane >= o) incl += t;
    }
    const unsigned start0 = incl - ch0 - ch1, start1 = start0 + ch0;  // first chunk of each site
    const unsigned total_chunks = __shfl_sync(0xffffffffu, incl, 31);
    // segment starts where every thread of the CTA can look them up by site (all warps store the same values)
    sts32(c.seg + (2 * lane) * 4, start0);
    sts32(c.seg + (2 * lane + 1) * 4, start1);
    __syncwarp();
    // Scatter rounds.  The list holds LIST_CAP pairs; a round covers the chunks [r0, r_end) = the sites [k_lo, k_hi),
    // and a segment is never split across rounds (a segment has <= TILE/32 chunks, so every round makes
    // progress).  One round is the rule; more are needed only when a tile enables more than LIST_CAP pairs here.
    constexpr unsigned ROUND_CHUNKS = LIST_CAP / 32;
    unsigned r0 = 0;
#pragma unroll 1
    do {
      // end of this round: the start of the first segment that does not fit any more
      unsigned r_end = total_chunks;
      if (total_chunks > r0 + ROUND_CHUNKS) {
        unsigned cand0 = (ch0 && start0 >= r0 && start0 + ch0 > r0 + ROUND_CHUNKS) ? start0 : 0xFFFFFFFFu;
        unsigned cand1 = (ch1 && start1 >= r0 && start1 + ch1 > r0 + ROUND_CHUNKS) ? start1 : 0xFFFFFFFFu;
        unsigned nxt = min(cand0, cand1);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) nxt = min(nxt, __shfl_xor_sync(0xffffffffu, nxt, o));
        r_end = min(r_end, nxt);
      }
      // sites of this round = those whose (non-empty) segment starts in [r0, r_end): a contiguous index range
      const unsigned in0 = __ballot_sync(0xffffffffu, ch0 && start0 >= r0 && start0 < r_end);
      const unsigned in1 = __ballot_sync(0xffffffffu, ch1 && start1 >= r0 && start1 < r_end);
      int k_lo = 64, k_hi = 0;
      if (in0) { k_lo = min(k_lo, 2 * (__ffs(in0) - 1)); k_hi = max(k_hi, 2 * (31 - __clz(in0)) + 1); }
      if (in1) { k_lo = min(k_lo, 2 * (__ffs(in1) - 1) + 1); k_hi = max(k_hi, 2 * (31 - __clz(in1)) + 2); }
      if (r0) __syncthreads();                         // later rounds: the previous round's list is consumed
      // ---- A2: every thread scatters its own pairs: slot = cursor[site]++ inside the site's segment
      auto scatter_one = [&](uint64_t& m, int j) {
        const int k = __ffsll((long long)m) - 1;
        m &= m - 1;
        if (k >= k_lo && k < k_hi) {                   // (a later round takes the sites outside)
          const unsigned st = lds32(c.seg + k * 4);
          const unsigned pos = (st - r0) * 32 + atoms_add(c.cur + k * 4, 1u);
          asm volatile("st.shared.u16 [%0], %1;" ::"r"(c.list + pos * 2), "h"((unsigned short)((unsigned)j * EXPAND_BLOCK + threadIdx.x)) : "memory");
        }
      };
#pragma unroll
      for (int j = 0; j < SPT; ++j) {
        uint64_t m = masks[j];
#pragma unroll
        for (int it = 0; it < 3; ++it)
          if (m) scatter_one(m, j);
        while (m) scatter_one(m, j);
      }
      __syncthreads();                                 // list complete (also orders the clearing of the other totals buffer)
      if (threadIdx.x < MAX_GROUP_SITES) sts32(c.cur + threadIdx.x * 4, 0u);   // cursors ready for the next scatter
      // ---- B: bodies, one chunk (= 32 pairs of one site) per warp and step
#pragma unroll 1
      for (unsigned ch = r0 + warp; ch < r_end; ch += NWARPS) {
        // site of this chunk: the last site whose first chunk is <= ch (an empty site shares its successor's start)
        const int below = __popc(__ballot_sync(0xffffffffu, start0 <= ch && 2 * lane < (unsigned)NS)) +
                          __popc(__ballot_sync(0xffffffffu, start1 <= ch && 2 * lane + 1 < (unsigned)NS));
        const int k = below - 1;
        const unsigned st = __shfl_sync(0xffffffffu, (k & 1) ? start1 : start0, k >> 1);
        const unsigned ck = __shfl_sync(0xffffffffu, (k & 1) ? c1 : c0, k >> 1);
        const unsigned e = (ch - st) * 32 + lane;      // index inside the site's segment
        if (e < ck) {
          unsigned short slot16;
          asm volatile("ld.shared.u16 %0, [%1];" : "=h"(slot16) : "r"(c.list + ((st - r0) * 32 + e) * 2));
          const unsigned slot = slot16;
          State s;
#pragma unroll
          for (int q = 0; q < W; ++q) s.w[q] = lds64(c.tile + (slot * W + q) * 8);
          CandSink sink{(c.first + c.tile_base + slot) | ((uint64_t)p.rank << 40), c.wbuf, c.wcnt, 0, 0};
          SiteDispatch<BEGIN, END>::run(k + BEGIN, s, sink);
          failed |= sink.failed;
        }
        flush_stage(p, c.wbuf, c.wcnt, c.cta, false, failed);
      }
      r0 = r_end;
    } while (r0 < total_chunks);
    SiteGroupRunner<G + 1>::run(p, c, nsucc, failed);
  }
};
template <>
struct SiteGroupRunner<M::NUM_SITE_GROUPS> {
  static __device__ __forceinline__ void run(const Params&, const TileCtx&, unsigned (&)[SPT], int&) {}
};

__global__ void __launch_bounds__(EXPAND_BLOCK, 1) k_expand(Params p, uint64_t first, uint64_t count, unsigned tile_states) {
  // tile | stage | list | cnt[2][64] | cur[64] | seg[64] | wcnt[NWARPS] | - | site_gen | CTA counters
  extern __shared__ __align__(16) uint64_t smem[];
  const int warp = threadIdx.x >> 5;
  TileCtx c;
  c.tile = smem_addr(smem);
  const uint32_t stage = c.tile + TILE * W * 8;
  c.wbuf = stage + warp * (STAGE_ROWS * ROW * 8);
  c.list = stage + STAGE_BYTES;
  c.cnt = c.list + LIST_CAP * 2;
  c.cur = c.cnt + 2 * MAX_GROUP_SITES * 4;
  c.seg = c.cur + MAX_GROUP_SITES * 4;
  c.wcnt = c.seg + MAX_GROUP_SITES * 4 + warp * 4;
  c.site_gen = c.seg + MAX_GROUP_SITES * 4 + (NWARPS + 8) * 4;
  c.cta = c.site_gen + SITE_GEN_BYTES;
  c.first = first;
  if (lane_id() == 0) sts32(c.wcnt, 0u);
  for (unsigned i = threadIdx.x; i < (unsigned)M::NUM_SITES; i += EXPAND_BLOCK) sts64(c.site_gen + i * 8, 0ull);
  for (unsigned i = threadIdx.x; i < (unsigned)(CTA_CTR_BYTES / 8); i += EXPAND_BLOCK) sts64(c.cta + i * 8, 0ull);
  unsigned long long gen = 0, dead = 0;
  unsigned maxfan = 0;
  int failed = 0;
  // tile_states <= TILE: small levels use smaller tiles so that every SM still gets one
  for (uint64_t tile_base = (uint64_t)blockIdx.x * tile_states; tile_base < count; tile_base += (uint64_t)gridDim.x * tile_states) {
    c.tile_base = tile_base;
    c.nvalid = (unsigned)min((uint64_t)tile_states, count - tile_base);
    __syncthreads();                                   // every body of the previous tile has read its state
    if (threadIdx.x < 3 * MAX_GROUP_SITES) sts32(c.cnt + threadIdx.x * 4, 0u);      // cnt[2][64] and cur[64]
    {
      // frontier tile -> shared memory, coalesced (128-bit loads when the rows are 16-byte aligned)
      const uint64_t* src = p.store + ((first + tile_base) & p.store_mask) * W;      // (a chunk never crosses the ring's wrap)
      const unsigned nwords = c.nvalid * W;
      if (((W & 1) == 0)) {
        const ulonglong2* src2 = reinterpret_cast<const ulonglong2*>(src);
        for (unsigned i = threadIdx.x; i < nwords / 2; i += EXPAND_BLOCK) {
          ulonglong2 v = __ldg(src2 + i);
          asm volatile("st.shared.v2.u64 [%0], {%1, %2};" ::"r"(c.tile + i * 16), "l"(v.x), "l"(v.y) : "memory");
        }
      } else {
        for (unsigned i = threadIdx.x; i < nwords; i += EXPAND_BLOCK) sts64(c.tile + i * 8, __ldg(src + i));
      }
    }
    __syncthreads();
    unsigned nsucc[SPT];
#pragma unroll
    for (int j = 0; j < SPT; ++j) nsucc[j] = 0;
    SiteGroupRunner<0>::run(p, c, nsucc, failed);
    flush_stage(p, c.wbuf, c.wcnt, c.cta, true, failed);
#pragma unroll
    for (int j = 0; j < SPT; ++j) {
      const unsigned slot = (unsigned)j * EXPAND_BLOCK + threadIdx.x;
      if (slot < c.nvalid) {
        gen += nsucc[j];
        maxfan = max(maxfan, nsucc[j]);
        if (nsucc[j] == 0) {
          ++dead;
          if (p.check_deadlock) {
            State s;
            const uint64_t gi = (first + tile_base + slot) & p.store_mask;
            load_state(s, p.store + gi * W);
            record_violation(p.ctr, p.viol_ring, s, p.parent[gi], state_fp(s), ~0ull);
          }
        }
      }
    }
  }
  // warp reduce the statistics, one atomic per warp
  for (int o = 16; o > 0; o >>= 1) {
    gen += __shfl_xor_sync(0xffffffffu, gen, o);
    dead += __shfl_xor_sync(0xffffffffu, dead, o);
    maxfan = max(maxfan, __shfl_xor_sync(0xffffffffu, maxfan, o));
    failed = max(failed, __shfl_xor_sync(0xffffffffu, failed, o));
  }
  if (lane_id() == 0) {
    if (gen) atomicAdd(&p.ctr->generated, gen);
    if (dead) atomicAdd(&p.ctr->deadlocks, dead);
    if (maxfan) atomicMax(&p.ctr->max_fanout_seen, (unsigned long long)maxfan);
    if (failed) atomicCAS(&p.ctr->fail, 0ull, (unsigned long long)failed);
    if (p.fused && gen) reds_add64(c.cta + CTA_GEN * 8, gen);
  }
  // coverage and the fused insert's counters: one atomic per (CTA, counter)
  __syncthreads();
  for (unsigned i = threadIdx.x; i < (unsigned)M::NUM_SITES; i += EXPAND_BLOCK) {
    const unsigned long long v = lds64(c.site_gen + i * 8);
    if (v) atomicAdd(&p.ctr->site_generated[i], v);
  }
  if (p.fused) {
    for (unsigned i = threadIdx.x; i < (unsigned)M::NUM_ACTIONS; i += EXPAND_BLOCK) {
      const unsigned long long v = lds64(c.cta + (CTA_ACTION + i) * 8);
      if (v) atomicAdd(&p.ctr->action_distinct[i], v);
    }
    if (threadIdx.x == 0) {
      const unsigned long long probes = lds64(c.cta + CTA_PROBES * 8), oom = lds64(c.cta + CTA_OOM * 8);
      if (probes) atomicAdd(&p.ctr->probes, probes);
      if (oom) atomicAdd(&p.ctr->out_of_model, oom);
      // No candidate rows are written, but a chunk's successors are still bounded by the candidate region, so that
      // cand_bytes and fanout_bound mean the same with and without fusion: the CTA whose total crosses it fails the run.
      const unsigned long long g = lds64(c.cta + CTA_GEN * 8);
      if (g && atomicAdd(&p.ctr->cand_count[0], g) + g > p.region_rows)
        atomicCAS(&p.ctr->fail, 0ull, (unsigned long long)KMC_FAIL_CAND_FULL);
    }
  }
}

__device__ __forceinline__ void load_row(State& s, uint64_t& meta, const uint64_t* rows, uint64_t i, bool valid) {
  meta = 0;
  if (valid) {
    const uint64_t* row = rows + i * ROW;
#pragma unroll
    for (int k = 0; k < W; ++k) s.w[k] = __ldcs(row + k);
    meta = __ldcs(row + W);
  }
}

template <bool XS = false>
__device__ __forceinline__ void insert_rows(const Params& p, const uint64_t* rows, uint64_t n, unsigned& probes, unsigned& oom,
                                            int& failed) {
  const uint64_t n_round = (n + 31) & ~31ull;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += stride) {
    const bool v0 = i < n;
    State s0;
    uint64_t m0;
    load_row(s0, m0, rows, i, v0);
    const Prefetched<XS> f0 = prefetch_row<XS>(p, s0, v0);
    insert_row<false, XS>(p, s0, m0, v0, f0, probes, oom, failed);
  }
}

// One candidate row per thread per iteration.  (Two rows per thread -- two sectors in flight per
// lane -- was measured slower: 72 vs 63 ms on the 340 M-state model; the extra registers cost more
// occupancy than the added memory-level parallelism gains.)
__global__ void __launch_bounds__(256) k_insert(Params p, const uint64_t* rows, const unsigned long long* n_ptr,
                                                 uint64_t n_fixed) {
  uint64_t n = n_ptr ? (uint64_t)*n_ptr : n_fixed;
  unsigned probes = 0, oom = 0;
  int failed = 0;
  if (n_ptr && n > p.region_rows) {
    // the expand kernel's slot claims ran past the region (it reports KMC_FAIL_CAND_FULL itself; the
    // counter keeps counting): never read beyond the rows that were actually written
    n = p.region_rows;
    failed = KMC_FAIL_CAND_FULL;
  }
  if constexpr (XS_ON) {
    if (p.exact) insert_rows<XS_ON>(p, rows, n, probes, oom, failed);
    else insert_rows(p, rows, n, probes, oom, failed);
  } else {
    insert_rows(p, rows, n, probes, oom, failed);
  }
  for (int o = 16; o > 0; o >>= 1) {
    probes += __shfl_xor_sync(0xffffffffu, probes, o);
    oom += __shfl_xor_sync(0xffffffffu, oom, o);
    failed = max(failed, __shfl_xor_sync(0xffffffffu, failed, o));
  }
  if (lane_id() == 0) {
    if (probes) atomicAdd(&p.ctr->probes, (unsigned long long)probes);
    if (oom) atomicAdd(&p.ctr->out_of_model, (unsigned long long)oom);
    if (failed) atomicCAS(&p.ctr->fail, 0ull, (unsigned long long)failed);
  }
}

// ----------------------------------------------------------------------------------------
// K5: the transitions of a chunk of stored states (kmc_edges).  One thread per candidate row of a non-fused expand:
// rows a CONSTRAINT discards are dropped, and every other row becomes an edge -- the source's global store index and
// the set-identity fingerprints (state_fp) of source and successor, the source read back through the row's parent
// index.  The source states lie at srcs[(parent index & src_mask) * W] and their global index is parent index +
// src_offset (the device store in place, or a staging copy of spilled states).  A warp ballot compacts the edges.
// ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_edges(const uint64_t* rows, const unsigned long long* n_ptr, const uint64_t* srcs,
                                                uint64_t src_mask, uint64_t src_offset, uint64_t n_cap,
                                                kmc_edge_t* out, unsigned long long* out_n) {
  const uint64_t n = min((uint64_t)*n_ptr, n_cap);
  const uint64_t n_round = (n + 31) & ~31ull;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const unsigned lane = lane_id();
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += stride) {
    State s;
    uint64_t meta;
    load_row(s, meta, rows, i, i < n);
    const bool keep = i < n && ((M::NUM_CONSTRAINTS == 0) || M::in_model(s));
    kmc_edge_t e{};
    if (keep) {
      const uint64_t local = meta & IDX_MASK;
      State src;
      load_state(src, srcs + (local & src_mask) * W);
      e.src = local + src_offset;
      e.src_fp = state_fp(src);
      e.dst_fp = state_fp(s);
      e.action = (uint32_t)(meta >> 56);
    }
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    if (m == 0) continue;
    const int leader = __ffs(m) - 1;
    unsigned long long base = 0;
    if ((int)lane == leader) base = atomicAdd(out_n, (unsigned long long)__popc(m));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (keep) out[base + __popc(m & ((1u << lane) - 1))] = e;
  }
}

#ifdef KMC_HAS_DEVICE_INIT
// ----------------------------------------------------------------------------------------
// K0: device Init.  One candidate index of one branch per thread, grid-stride with 64-bit indices: the lowered
// init_candidate() decodes it, runs the branch's filters and packs a solution.  A warp ballot compacts the solutions
// into the warp's shared-memory stage (the rows of k_expand's stage, parent word NO_PARENT), which the warp inserts
// through insert_stage whenever it holds STAGE_FLUSH rows or more.  Solutions, candidates, probes and out-of-model
// initial states are counted per CTA in shared memory and flushed with one global atomic each.
// ----------------------------------------------------------------------------------------
static constexpr int INIT_BLOCK = 256;
static constexpr int INIT_WARPS = INIT_BLOCK / 32;
static constexpr int CTA_INIT_GEN = CTA_ACTION + M::NUM_ACTIONS, CTA_INIT_CAND = CTA_INIT_GEN + 1;

__global__ void __launch_bounds__(INIT_BLOCK) k_init(Params p, int branch, uint64_t first, uint64_t count) {
  __shared__ __align__(16) uint64_t stage[INIT_WARPS * STAGE_ROWS * ROW];
  __shared__ unsigned long long cta_ctr[CTA_INIT_CAND + 1];
  const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
  const uint32_t wbuf = smem_addr(stage) + warp * (STAGE_ROWS * ROW * 8);
  const uint32_t cta = smem_addr(cta_ctr);
  for (unsigned i = threadIdx.x; i < (unsigned)(CTA_INIT_CAND + 1); i += INIT_BLOCK) cta_ctr[i] = 0;
  __syncthreads();
  unsigned staged = 0;                     // rows in this warp's stage (warp-uniform)
  unsigned long long sols = 0, cands = 0;
  unsigned layout = 0;
  int failed = 0;
  const uint64_t stride = (uint64_t)gridDim.x * INIT_BLOCK;
  // the loop bound is warp-uniform, so that the ballot and the stage insert see all 32 lanes
  for (uint64_t base = (uint64_t)blockIdx.x * INIT_BLOCK + warp * 32; base < count; base += stride) {
    const uint64_t i = base + lane;
    const bool valid = i < count;
    State s;
    unsigned fail = 0;
    const bool ok = valid && M::init_candidate(branch, first + i, s, fail);
    if (fail) layout = fail;
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if (ok) {
      const uint32_t row = wbuf + (staged + __popc(m & ((1u << lane) - 1))) * (ROW * 8);
#pragma unroll
      for (int k = 0; k < W; ++k) sts64(row + k * 8, s.w[k]);
      sts64(row + W * 8, NO_PARENT);
    }
    staged += __popc(m);
    sols += __popc(m);
    cands += count - base < 32 ? count - base : 32;
    if (staged >= (unsigned)STAGE_FLUSH) {
      __syncwarp();
      const int f = insert_stage_of(p, wbuf, staged, cta);
      if (f) failed = f;
      staged = 0;
      __syncwarp();
    }
  }
  if (staged) {
    __syncwarp();
    const int f = insert_stage_of(p, wbuf, staged, cta);
    if (f) failed = f;
  }
  layout = __reduce_or_sync(0xffffffffu, layout);
  failed = __reduce_max_sync(0xffffffffu, failed);
  if (lane == 0) {
    if (sols) reds_add64(cta + CTA_INIT_GEN * 8, sols);
    if (cands) reds_add64(cta + CTA_INIT_CAND * 8, cands);
    // a solution that does not fit the layout is reported like a successor that does not: KMC_E_LAYOUT_OVERFLOW
    if (layout) atomicCAS(&p.ctr->fail, 0ull, (unsigned long long)KMC_FAIL_LAYOUT);
    else if (failed) atomicCAS(&p.ctr->fail, 0ull, (unsigned long long)failed);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned long long probes = cta_ctr[CTA_PROBES], oom = cta_ctr[CTA_OOM];
    const unsigned long long g = cta_ctr[CTA_INIT_GEN], c = cta_ctr[CTA_INIT_CAND];
    if (probes) atomicAdd(&p.ctr->probes, probes);
    if (oom) atomicAdd(&p.ctr->out_of_model, oom);
    if (g) {
      atomicAdd(&p.ctr->generated, g);
      atomicAdd(&p.ctr->init_generated, g);
    }
    if (c) atomicAdd(&p.ctr->init_candidates, c);
  }
}
#endif

__device__ __forceinline__ void st_release_sys(uint64_t* p, uint64_t v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t ld_acquire_sys(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint64_t* sync_page(const Params& p, uint32_t r) { return p.peer_inbox[r] - SYNC_WORDS; }

// Fused exchange, step 2: tell every owner how many rows this rank stored in its inbox region and (round > 0)
// raise this rank's ready flag there.  The expand kernel that stored the rows is complete (stream order); the
// system-scope fence + release store order its peer writes before the flag.
__global__ void k_publish_counts(Params p, uint64_t round) {
  unsigned d = threadIdx.x;
  if (d < p.world) {
    p.peer_inbox[d][(uint64_t)p.inbox_buf * p.inbox_stride + p.rank] = p.ctr->cand_count[d];
    if (round) {
      __threadfence_system();
      st_release_sys(sync_page(p, d) + SYNC_READY + p.rank, round);
    }
  }
}

// A device-side wait is bounded: a peer that never arrives (its process died, its context failed) turns into
// KMC_E_PEER_TIMEOUT on this rank after PEER_TIMEOUT_NS instead of a kernel that spins for ever and takes the
// GPU with it.  Once the flag is up, later waits of the run return at once (the run is lost anyway).
static constexpr unsigned long long PEER_TIMEOUT_NS = 30ull * 1000ull * 1000ull * 1000ull;
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void wait_flag(const uint64_t* flag, uint64_t value, DevCounters* ctr) {
  if (ld_acquire_sys(flag) >= value) return;
  if (*(volatile unsigned long long*)&ctr->fail == KMC_FAIL_PEER_TIMEOUT) return;
  const unsigned long long t0 = globaltimer_ns();
  unsigned ns = 32;
  while (ld_acquire_sys(flag) < value) {
    __nanosleep(ns);
    if (ns < 1024) ns <<= 1;
    if (globaltimer_ns() - t0 > PEER_TIMEOUT_NS) {
      atomicCAS(&ctr->fail, 0ull, (unsigned long long)KMC_FAIL_PEER_TIMEOUT);
      return;
    }
  }
}

// Device-side wait (one warp): lane i waits until flags[i] >= value.  The flags live in this rank's own memory
// (peers push), so the polling never crosses NVLink.
__global__ void k_wait_flags(const uint64_t* flags, unsigned n, uint64_t value, DevCounters* ctr) {
  unsigned i = threadIdx.x;
  if (i < n) wait_flag(flags + i, value, ctr);
}

// after the insert of a round: every source may now reuse this rank's inbox buffer of that round
__global__ void k_publish_done(Params p, uint64_t round) {
  unsigned s = threadIdx.x;
  if (s < p.world) {
    __threadfence_system();
    st_release_sys(sync_page(p, s) + SYNC_DONE + p.rank, round);
  }
}

// Level end: this rank's summary goes to every rank's board (peer stores), ...
__global__ void k_publish_level(Params p, uint64_t level_id, uint64_t prev_tail) {
  unsigned d = threadIdx.x;
  if (d < p.world) {
    uint64_t* e = sync_page(p, d) + SYNC_BOARD + p.rank * BOARD_WORDS;
    const unsigned long long tail = p.ctr->store_tail;
    e[1] = tail - prev_tail;
    e[2] = p.ctr->viol_count;
    e[3] = tail;
    e[4] = p.ctr->generated;
    e[5] = p.ctr->fail;
    e[6] = p.ctr->deadlocks;
    e[7] = p.ctr->inv_new;
    __threadfence_system();
    st_release_sys(e, level_id);
  }
}
// ... and once every rank's entry of this level has arrived the whole board is copied to pinned host memory:
// the host's single synchronisation per level is the stream sync after this kernel.
__global__ void k_gather_level(Params p, uint64_t level_id, uint64_t* host_out) {
  unsigned r = threadIdx.x;
  const uint64_t* board = sync_page(p, p.rank) + SYNC_BOARD;
  if (r < p.world) {
    wait_flag(board + r * BOARD_WORDS, level_id, p.ctr);
    for (int k = 0; k < BOARD_WORDS; ++k) host_out[r * BOARD_WORDS + k] = board[r * BOARD_WORDS + k];
    // a timed-out wait of this level (or of one of its rounds) reaches the host through this rank's own entry
    if (r == p.rank) {
      const unsigned long long f = *(volatile unsigned long long*)&p.ctr->fail;
      if (f == KMC_FAIL_PEER_TIMEOUT) host_out[r * BOARD_WORDS + 5] = f;
    }
  }
}

// Fused exchange, step 3 (after a cross-rank barrier): insert the rows of all source regions of
// this rank's inbox buffer.  Row counts come from the header the sources wrote -- the host never
// sees them.
__global__ void __launch_bounds__(256) k_insert_inbox(Params p) {
  const uint64_t* inbox = p.peer_inbox[p.rank] + (uint64_t)p.inbox_buf * p.inbox_stride;
  uint64_t starts[MAX_WORLD + 1];
  starts[0] = 0;
#pragma unroll
  for (int r = 0; r < MAX_WORLD; ++r) {
    uint64_t n = (r < (int)p.world) ? inbox[r] : 0;
    if (n > p.region_rows) n = p.region_rows;
    starts[r + 1] = starts[r] + n;
  }
  const uint64_t n = starts[MAX_WORLD];
  const uint64_t n_round = (n + 31) & ~31ull;
  unsigned probes = 0, oom = 0;
  int failed = 0;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += stride) {
    const bool v0 = i < n;
    State s0;
    uint64_t m0 = 0;
    if (v0) {
      int src = 0;
#pragma unroll
      for (int r = 1; r < MAX_WORLD; ++r) src += (i >= starts[r]) ? 1 : 0;
      const uint64_t* row = inbox + INBOX_HEADER + ((uint64_t)src * p.region_rows + (i - starts[src])) * ROW;
#pragma unroll
      for (int k = 0; k < W; ++k) s0.w[k] = __ldcs(row + k);
      m0 = __ldcs(row + W);
    }
    const Prefetched<> f0 = prefetch_row(p, s0, v0);
    insert_row(p, s0, m0, v0, f0, probes, oom, failed);
  }
  for (int o = 16; o > 0; o >>= 1) {
    probes += __shfl_xor_sync(0xffffffffu, probes, o);
    oom += __shfl_xor_sync(0xffffffffu, oom, o);
    failed = max(failed, __shfl_xor_sync(0xffffffffu, failed, o));
  }
  if (lane_id() == 0) {
    if (probes) atomicAdd(&p.ctr->probes, (unsigned long long)probes);
    if (oom) atomicAdd(&p.ctr->out_of_model, (unsigned long long)oom);
    if (failed) atomicCAS(&p.ctr->fail, 0ull, (unsigned long long)failed);
  }
}

// K3: invariants on the new states of a level.  They sit compacted in the store, so every lane
// has work (inside k_insert only the ~1/3 of lanes holding a new state would be active).
__global__ void __launch_bounds__(256) k_invariants(Params p, uint64_t first, const unsigned long long* end_ptr) {
  uint64_t end = (uint64_t)*end_ptr;
  if (end - p.store_base > p.max_states) end = p.store_base + p.max_states;
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = first + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < end; i += stride) {
    State s;
    const uint64_t* src = p.store + (i & p.store_mask) * W;
#pragma unroll
    for (int k = 0; k < W; ++k) s.w[k] = __ldcs(src + k);
    int inv = M::first_violated_invariant(s);
    if (inv >= 0) record_violation(p.ctr, p.viol_ring, s, p.parent[i & p.store_mask], state_fp(s), (uint64_t)inv);
  }
}

// K3 of a "continue" run, after k_invariants: the per-invariant report of the level's violators -- its new states and the
// discarded successors the inserts staged.  A level without violators (the violator count did not move since the last
// level end) returns at once, so k_invariants itself is unchanged; a level with some checks its new states a second
// time, in whole rounds of 32 (the last one padded) so that record_invariants is called by converged warps.
__global__ void __launch_bounds__(256) k_invariant_report(Params p, uint64_t first, const unsigned long long* end_ptr) {
  if (!INV_REPORT || !p.ctr->inv_on || p.ctr->viol_count == p.ctr->inv_viol_seen) return;
  uint64_t end = (uint64_t)*end_ptr;
  if (end - p.store_base > p.max_states) end = p.store_base + p.max_states;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t end_round = first + ((end - first + 31) & ~31ull);
  for (uint64_t i = first + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < end_round; i += stride) {
    State s;
    bool member = false;
    if (i < end) {
      const uint64_t* src = p.store + (i & p.store_mask) * W;
#pragma unroll
      for (int k = 0; k < W; ++k) s.w[k] = __ldcs(src + k);
      member = M::first_violated_invariant(s) >= 0;
    }
    if (__ballot_sync(0xffffffffu, member))
      record_invariants(p.ctr, p.viol_ring, s, member ? p.parent[i & p.store_mask] : 0, member ? state_fp(s) : 0, member);
  }
  const uint64_t staged = p.ctr->inv_staged < (uint64_t)VIOL_RING ? p.ctr->inv_staged : (uint64_t)VIOL_RING;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < ((staged + 31) & ~31ull); j += stride) {
    State s;
    uint64_t meta = 0, fp = 0;
    if (j < staged) {
      const uint64_t* row = stage_ring_of(p.viol_ring) + j * VIOL_ROW;
#pragma unroll
      for (int k = 0; k < W; ++k) s.w[k] = row[k];
      meta = row[W];
      fp = row[W + 1];
    }
    record_invariants(p.ctr, p.viol_ring, s, meta, fp, j < staged);
  }
}

// -recover: the set is not part of a checkpoint; it is rebuilt from the stored states (one insert each)
__global__ void __launch_bounds__(256) k_rebuild(Params p, const uint64_t* states, uint64_t n) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  int failed = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    State s;
#pragma unroll
    for (int k = 0; k < W; ++k) s.w[k] = states[i * W + k];
    unsigned probes = 0;
    if constexpr (XS_ON) {
      if (p.exact) {
        State key;
        uint64_t fp;
        state_xident(s, key, fp);
        const int r = xset_insert(p.table, p.bucket_mask, fp, key, ld_xbucket(p.table, bucket_of(fp, p.bucket_mask)), probes);
        if (r < 0) failed = r == -1 ? KMC_FAIL_TABLE_FULL : KMC_FAIL_SET_TIMEOUT;
        continue;
      }
    }
    if (set_insert(p.table, p.bucket_mask, state_ident(s), probes) < 0) failed = KMC_FAIL_TABLE_FULL;
  }
  if (failed) atomicCAS(&p.ctr->fail, 0ull, (unsigned long long)failed);
}

// The set alone (FPSet.put / contains): the caller's 64-bit fingerprints are the identities; with 16-byte
// slots the key is the fingerprint and its second mix.
__global__ void k_fpset_put(void* table, uint64_t bucket_mask, const uint64_t* fps, uint64_t n, uint8_t* seen,
                            DevCounters* ctr, int insert) {
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    Ident id;
    id.fp = fps[i] ? fps[i] : 1;
    id.key = Key128{id.fp, fmix64b(id.fp)};
    if (insert) {
      unsigned probes = 0;
      int r = set_insert(table, bucket_mask, id, probes);
      if (r < 0) atomicCAS(&ctr->fail, 0ull, (unsigned long long)KMC_FAIL_TABLE_FULL);
      if (r > 0) atomicAdd(&ctr->store_tail, 1ull);
      seen[i] = r == 0;
    } else {
      seen[i] = set_contains(table, bucket_mask, id) >= 0 ? 1 : 0;
    }
  }
}

// ----------------------------------------------------------------------------------------
// set_spill: the keys of the set move to host memory when the table fills (DESIGN.md section 3)
// ----------------------------------------------------------------------------------------
// An epoch is the time between two flushes.  k_set_flush copies the table's keys out (except those the last filter
// found in host memory already) and the host empties the table.  The filter (k_set_mark, then k_set_compact) removes
// from the states appended since the last filter those whose key is in host memory: they were found in an earlier epoch.
static constexpr int KEY_WORDS = SLOT_BYTES / 8;
static constexpr int XKEY_WORDS = W;          // exact_set: a key in host memory is the (canonical) packed state
static constexpr int SET_TILE = 256;          // states per tile of the filter's compaction

// The identity a stored key stands for: the key alone gives the fingerprint that picks its bucket.
__device__ __forceinline__ Ident key_ident(const uint64_t* k) {
  Ident id;
  if constexpr (!KEY128) {
    id.fp = k[0];
    id.key = Key128{0, 0};
  } else if constexpr (W == 2 && !M::ALL_ONES_POSSIBLE) {
    State s;                                   // the key is the packed (canonical) state itself
    s.w[0] = k[0];
    s.w[W - 1] = k[1];
    id.fp = fingerprint(s);
    id.key = Key128{k[0], k[1]};
  } else {
    id.fp = k[0];                              // the fingerprint is the key's low word
    id.key = Key128{k[0], k[1]};
  }
  return id;
}

__device__ __forceinline__ bool marked(const unsigned* marks, long long slot) {
  return slot >= 0 && ((marks[slot >> 5] >> (slot & 31)) & 1u);
}

// Slots [first, first + n) of the table: every key that is not marked goes to `out`, compacted with ballot/popc (the
// order does not matter), counted in ctr->set_count.  XS (exact_set): a key is the W state words behind a slot's
// header (XKEY_WORDS), and a slot is full when its header is not XEMPTY.
template <bool XS = false>
__global__ void __launch_bounds__(256) k_set_flush(const void* table, uint64_t first, uint64_t n, const unsigned* marks,
                                                    uint64_t* out, DevCounters* ctr) {
  constexpr int KW = XS ? XKEY_WORDS : KEY_WORDS;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const unsigned lane = lane_id();
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ((n + 31) & ~31ull); i += stride) {
    const uint64_t slot = first + i;
    uint64_t k[KW];
    bool take = false;
    if (i < n) {
      if constexpr (XS) {
        const uint64_t* src = static_cast<const uint64_t*>(table) + slot * XSLOT_WORDS;
#pragma unroll
        for (int w = 0; w < KW; ++w) k[w] = src[1 + w];
        take = src[0] != XEMPTY && !marked(marks, (long long)slot);
      } else {
        const uint64_t* src = static_cast<const uint64_t*>(table) + slot * KEY_WORDS;
#pragma unroll
        for (int w = 0; w < KEY_WORDS; ++w) k[w] = src[w];
        const bool full = KEY128 ? (k[0] & k[KEY_WORDS - 1]) != ~0ull : k[0] != 0;
        take = full && !marked(marks, (long long)slot);
      }
    }
    const unsigned who = __ballot_sync(0xffffffffu, take);
    if (!who) continue;
    unsigned long long base = 0;
    if ((int)lane == __ffs(who) - 1) base = atomicAdd(&ctr->set_count, (unsigned long long)__popc(who));
    base = __shfl_sync(0xffffffffu, base, __ffs(who) - 1);
    if (take) {
      uint64_t* dst = out + (base + __popc(who & ((1u << lane) - 1))) * KW;
#pragma unroll
      for (int w = 0; w < KW; ++w) dst[w] = k[w];
    }
  }
}

// n host keys (one chunk of the stream through HBM): each one found in the table marks its slot.
template <bool XS = false>
__global__ void __launch_bounds__(256) k_set_mark(const void* table, uint64_t bucket_mask, const uint64_t* keys, uint64_t n,
                                                   unsigned* marks) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    long long slot;
    if constexpr (XS) {
      State key;
#pragma unroll
      for (int w = 0; w < W; ++w) key.w[w] = keys[i * XKEY_WORDS + w];
      slot = xset_contains(table, bucket_mask, fingerprint(key), key);
    } else {
      slot = set_contains(table, bucket_mask, key_ident(keys + i * KEY_WORDS));
    }
    if (slot >= 0) atomicOr(marks + (slot >> 5), 1u << (slot & 31));
  }
}

// The filter's verdict on the states [first, first + n) of the store: a state is removed when the slot of its identity
// (state_ident: the orbit representative under SYMMETRY) is marked.  keep[j] = 1 for a survivor, tile_count[t] = the
// survivors of tile t, and the removed states leave the per-action distinct counts (their parent words' actions).
__global__ void __launch_bounds__(SET_TILE) k_set_compact(Params p, uint64_t first, uint64_t n, const unsigned* marks,
                                                           uint8_t* keep, unsigned long long* tile_count) {
  __shared__ unsigned long long removed[M::NUM_ACTIONS > 0 ? M::NUM_ACTIONS : 1];
  for (unsigned a = threadIdx.x; a < (unsigned)M::NUM_ACTIONS; a += SET_TILE) removed[a] = 0;
  __syncthreads();
  for (uint64_t t = blockIdx.x; t * SET_TILE < n; t += gridDim.x) {
    const uint64_t j = t * SET_TILE + threadIdx.x;
    bool kept = false;
    if (j < n) {
      const uint64_t g = (first + j) & p.store_mask;
      State s;
#pragma unroll
      for (int k = 0; k < W; ++k) s.w[k] = p.store[g * W + k];
      long long slot = -1;
      if constexpr (XS_ON) {
        if (p.exact) {
          State key;
          uint64_t fp;
          state_xident(s, key, fp);
          slot = xset_contains(p.table, p.bucket_mask, fp, key);
        } else {
          slot = set_contains(p.table, p.bucket_mask, state_ident(s));
        }
      } else {
        slot = set_contains(p.table, p.bucket_mask, state_ident(s));
      }
      kept = !marked(marks, slot);
      keep[j] = kept ? 1 : 0;
      if (!kept) {
        const uint64_t meta = p.parent[g];
        const unsigned act = ((meta & 0x0000FFFFFFFFFFFFull) == NO_PARENT) ? ~0u : (unsigned)(meta >> 56);
        if (act < (unsigned)M::NUM_ACTIONS) atomicAdd(&removed[act], 1ull);
      }
    }
    const int c = __syncthreads_count(kept);
    if (threadIdx.x == 0) tile_count[t] = (unsigned long long)c;
  }
  __syncthreads();
  for (unsigned a = threadIdx.x; a < (unsigned)M::NUM_ACTIONS; a += SET_TILE)
    if (removed[a]) atomicAdd(&p.ctr->action_distinct[a], 0ull - removed[a]);
}

// One CTA: tile_count[0, n) -> exclusive prefix sums in place; ctr->set_count = the total.
__global__ void __launch_bounds__(1024) k_set_scan(unsigned long long* tile_count, uint64_t n, DevCounters* ctr) {
  __shared__ unsigned long long warp_sum[32];
  __shared__ unsigned long long carry;
  const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (uint64_t base = 0; base < n; base += 1024) {
    const uint64_t i = base + threadIdx.x;
    const unsigned long long v = i < n ? tile_count[i] : 0;
    unsigned long long x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
      if ((int)lane >= o) x += y;
    }
    if (lane == 31) warp_sum[warp] = x;
    __syncthreads();
    if (warp == 0) {
      unsigned long long s = warp_sum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, s, o);
        if ((int)lane >= o) s += y;
      }
      warp_sum[lane] = s;
    }
    __syncthreads();
    if (i < n) tile_count[i] = carry + (warp ? warp_sum[warp - 1] : 0) + x - v;
    __syncthreads();
    if (threadIdx.x == 0) carry += warp_sum[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) ctr->set_count = carry;
}

// The survivors of [first, first + n), in their order, to out_states / out_parents at their tiles' offsets.
__global__ void __launch_bounds__(SET_TILE) k_set_scatter(Params p, uint64_t first, uint64_t n, const uint8_t* keep,
                                                           const unsigned long long* tile_off, uint64_t* out_states,
                                                           uint64_t* out_parents) {
  __shared__ unsigned warp_kept[SET_TILE / 32];
  const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
  for (uint64_t t = blockIdx.x; t * SET_TILE < n; t += gridDim.x) {
    const uint64_t j = t * SET_TILE + threadIdx.x;
    const bool kept = j < n && keep[j];
    const unsigned who = __ballot_sync(0xffffffffu, kept);
    if (lane == 0) warp_kept[warp] = __popc(who);
    __syncthreads();
    if (kept) {
      uint64_t o = tile_off[t] + __popc(who & ((1u << lane) - 1));
      for (unsigned w = 0; w < warp; ++w) o += warp_kept[w];
      const uint64_t g = (first + j) & p.store_mask;
#pragma unroll
      for (int k = 0; k < W; ++k) out_states[o * W + k] = p.store[g * W + k];
      out_parents[o] = p.parent[g];
    }
    __syncthreads();
  }
}

// ----------------------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------------------
struct LaunchRec {
  int kind;  // 0 expand, 1 insert, 2 other, 3 set_spill's flushes and filters, 4 device Init (k_init)
  cudaEvent_t a, b;
};

// A counterexample: the violator picked at `level` (its words, parent/action word `meta` and set-identity fingerprint)
// and its trace.  inv = -1 for a deadlock.  The run's violation is one (no `words`: none found yet); so is the report
// of each invariant under "continue" (kmc_invariant_reports), where `first_count` is the invariant's violators at
// `level`, its first violating level, and `words` is empty when every one of them fell beyond the per-invariant ring.
struct Counterexample {
  int32_t inv = -1;
  uint64_t level = 0, fp = 0, meta = 0, first_count = 0;
  std::vector<uint64_t> words;
  std::vector<std::vector<uint64_t>> trace;
  std::vector<uint32_t> actions;
};

struct Engine {
  int device = 0;
  int sms = 132;
  uint32_t rank = 0, world = 1;
  int table_log2 = 0;
  uint64_t max_states = 0;
  uint64_t cand_bytes = 0;
  bool cont = false;
  bool check_deadlock = M::CHECK_DEADLOCK;
  bool timing = true;
  uint64_t stop_after_states = 0;   // bounded run: stop at the first level end with >= this many states
  uint32_t fanout_bound = 0;        // successors per state assumed when sizing a frontier chunk (0: min(MAX_FANOUT, 32))
  // spill / checkpoint (single rank): the device store is a ring over the live window [store_base, tail); the
  // levels below the one being expanded move to host memory (TLC's DiskStateQueue / trace file on disk)
  bool spill = false;
  uint64_t store_base = 0;
  std::vector<uint64_t> host_store, host_parent;
  std::string checkpoint_dir, recover_dir;
  double checkpoint_minutes = 0;    // 0: a checkpoint after every level (when checkpoint_dir is set)
  std::chrono::steady_clock::time_point last_checkpoint;
  // set_spill (single rank): the keys of the set move to host memory whenever the table would pass set_limit(); the
  // filter's marks (a bit per table slot) and its staging and compaction space live at the end and the start of `cand`
  bool set_spill = false;
  // exact_set (single rank) on a model whose key is hashed: the set's key is the packed state (XSLOT_WORDS slots)
  bool exact = false;
  // the keys in host memory, key_words() words each as the table stores them: one block of exactly its size per flushed
  // slot range, so that the array grows without the copies (and the transient double size) of a growing vector
  std::vector<std::vector<uint64_t>> host_keys;
  uint64_t set_host_keys = 0;           // keys in host_keys
  uint64_t set_keys = 0;                // keys inserted into the table since the last flush
  uint64_t set_tail = 0;                // the store tail set_keys was last brought up to date with
  uint64_t set_from = 0;                // the first state the filter has not checked against host_keys
  uint64_t set_flushes = 0, set_filtered = 0, set_link_bytes = 0;
  uint64_t set_stage_keys = 0;          // keys per pinned staging buffer of the filter's key stream
  uint64_t* set_pinned[2] = {};
  cudaStream_t set_copy_stream = nullptr;
  cudaEvent_t set_copied[2] = {}, set_probed[2] = {};

  void* table = nullptr;
  uint64_t table_slots = 0;             // slots of slot_bytes() each
  uint64_t* store = nullptr;
  uint64_t* parent = nullptr;
  uint64_t* cand = nullptr;
  uint64_t region_rows = 0;
  uint64_t* recv = nullptr;
  uint64_t recv_rows = 0;
  uint64_t* inbox_alloc = nullptr;    // sync page + 2 inbox buffers, shared through CUDA IPC
  uint64_t* board_host = nullptr;     // pinned: the level board as gathered by k_gather_level
  uint64_t round = 0, level_id = 0;   // monotonic over the life of the context (see SYNC_WORDS)
  uint64_t prev_tail = 0;
  uint64_t* inbox = nullptr;          // fused exchange: 2 x (header + world regions)
  uint64_t inbox_stride = 0;
  uint64_t* peer_inbox[MAX_WORLD] = {};
  bool peers_open = false;
  bool peers_direct = false;          // peer pointers given directly (same process, cudaDeviceEnablePeerAccess)
  uint32_t inbox_buf = 0;
  uint64_t exchanged_rows = 0;
  DevCounters* ctr = nullptr;
  uint64_t* viol_ring = nullptr;
  cudaStream_t stream = nullptr;
  bool own_stream = true;       // false: the caller's stream (option "stream"), e.g. torch's current stream
  uint64_t chunk_states = 0;

  std::vector<cudaEvent_t> event_pool;
  size_t events_used = 0;
  std::vector<LaunchRec> launches;
  cudaEvent_t ev_begin = nullptr, ev_end = nullptr;

  // results
  mutable std::mutex mu;
  kmc_stats_t stats{};
  std::vector<uint64_t> widths;
  // coverage of the last run (host copies of the device counters, summed over the ranks of a "gpus" context);
  // incomplete after recovering from a checkpoint that predates the per-site counts
  std::vector<uint64_t> site_generated = std::vector<uint64_t>(M::NUM_SITES, 0);
  std::vector<uint64_t> action_distinct = std::vector<uint64_t>(M::NUM_ACTIONS, 0);
  bool coverage_complete = true;
  Counterexample viol;
  // per-invariant report of a "continue" run, in the order found; complete = 0 after a recover (it then covers only
  // the levels searched since)
  std::vector<Counterexample> inv_reports;
  uint64_t inv_pending = 0;
  std::vector<uint64_t> inv_count = std::vector<uint64_t>(64, 0);     // violators per invariant (the counters)
  bool inv_complete = true;
  bool ran = false;
  // the level cursor: the states [level_first, level_first + level_count) form BFS level `level`, the one expanded
  // next (level 0: nothing inserted yet)
  uint64_t level_first = 0, level_count = 0, level = 0;
  std::string last_error;

  uint64_t slot_bytes() const { return exact ? XSLOT_BYTES : SLOT_BYTES; }
  uint64_t bucket_mask() const { return table_slots / (exact ? XBUCKET_SLOTS : BUCKET_SLOTS) - 1; }
  uint64_t key_words() const { return exact ? XKEY_WORDS : KEY_WORDS; }      // a key in host memory (set_spill)
  // the table's empty fill: all-ones 16-byte keys and exact_set headers, zero 8-byte fingerprints
  int empty_byte() const { return KEY128 || exact ? 0xFF : 0; }

  Params params() const {
    Params p;
    p.table = table;
    p.bucket_mask = bucket_mask();
    p.store = store;
    p.parent = parent;
    p.max_states = max_states;
    p.store_mask = spill ? max_states - 1 : ~0ull;
    p.store_base = store_base;
    p.cand = cand;
    p.region_rows = region_rows;
    p.ctr = ctr;
    p.viol_ring = viol_ring;
    p.rank = rank;
    p.world = world;
    p.check_deadlock = check_deadlock ? 1 : 0;
    for (int r = 0; r < MAX_WORLD; ++r) p.peer_inbox[r] = peer_inbox[r];
    p.inbox_stride = inbox_stride;
    p.p2p = 0;
    p.inbox_buf = inbox_buf;
    p.fused = 0;
    p.exact = exact ? 1 : 0;
    return p;
  }
};

struct kmcm_ctx {
  Engine e;
  // option "gpus": N > 1 -- this context drives N GPUs of the process: one sub-context (rank) per device, peers
  // mapped directly (cudaDeviceEnablePeerAccess), one host thread per rank inside kmcm_run.  `e` then only
  // holds the aggregated results.
  std::vector<kmcm_ctx*> ranks;
};

#define CK(call)                                                                                         \
  do {                                                                                                   \
    cudaError_t _e = (call);                                                                             \
    if (_e != cudaSuccess) {                                                                             \
      E.last_error = std::string(#call) + ": " + cudaGetErrorString(_e);                                 \
      return (_e == cudaErrorMemoryAllocation) ? KMC_E_OOM : KMC_E_CUDA;                                 \
    }                                                                                                    \
  } while (0)

static bool json_find(const char* js, const char* key, const char** val) {
  if (!js) return false;
  std::string pat = std::string("\"") + key + "\"";
  const char* p = strstr(js, pat.c_str());
  if (!p) return false;
  p += pat.size();
  while (*p == ' ' || *p == '\t' || *p == '\n') ++p;
  if (*p != ':') return false;
  ++p;
  while (*p == ' ' || *p == '\t' || *p == '\n') ++p;
  *val = p;
  return true;
}
static bool json_num(const char* js, const char* key, double* out) {
  const char* v;
  if (!json_find(js, key, &v)) return false;
  char* end;
  double d = strtod(v, &end);
  if (end == v) return false;
  *out = d;
  return true;
}
static bool json_str(const char* js, const char* key, std::string* out) {
  const char* v;
  if (!json_find(js, key, &v) || *v != '"') return false;
  const char* e = strchr(v + 1, '"');
  if (!e) return false;
  out->assign(v + 1, e);
  return true;
}
static bool json_bool(const char* js, const char* key, bool* out) {
  const char* v;
  if (!json_find(js, key, &v)) return false;
  if (!strncmp(v, "true", 4)) { *out = true; return true; }
  if (!strncmp(v, "false", 5)) { *out = false; return true; }
  double d;
  if (json_num(js, key, &d)) { *out = d != 0; return true; }
  return false;
}

static cudaEvent_t get_event(Engine& E) {
  if (E.events_used == E.event_pool.size()) {
    cudaEvent_t ev;
    cudaEventCreate(&ev);
    E.event_pool.push_back(ev);
  }
  return E.event_pool[E.events_used++];
}

struct TimedLaunch {
  Engine& E;
  int kind;
  cudaEvent_t a = nullptr, b = nullptr;
  TimedLaunch(Engine& e, int k) : E(e), kind(k) {
    if (E.timing) {
      a = get_event(E);
      b = get_event(E);
      cudaEventRecord(a, E.stream);
    }
  }
  ~TimedLaunch() {
    if (E.timing) {
      cudaEventRecord(b, E.stream);
      E.launches.push_back({kind, a, b});
    }
  }
};

static int grid_for(const Engine& E, uint64_t n, int block, int per_sm) {
  uint64_t g = (n + block - 1) / block;
  uint64_t cap = (uint64_t)E.sms * per_sm;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

static int engine_alloc(Engine& E) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    E.last_error = "no CUDA device visible; this library has no CPU fallback";
    return KMC_E_NO_GPU;
  }
  if (E.device >= ndev) {
    E.last_error = "device index out of range";
    return KMC_E_BADARG;
  }
  CK(cudaSetDevice(E.device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, E.device));
  E.sms = prop.multiProcessorCount;
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  // Default sizing from the memory that is actually free: candidate buffers first, then set + store + parent
  // links share the rest (2.5 slots per state: load <= 0.4, rounded to a power of two).
  if (E.cand_bytes == 0) E.cand_bytes = std::min<uint64_t>(free_b / 8, (E.world > 1 ? 24ull : 12ull) << 30);
  const uint64_t cand_total = E.cand_bytes * (E.world > 1 ? 4 : 1);          // + recv + two inbox buffers
  const uint64_t budget = free_b > cand_total + (512ull << 20) ? (uint64_t)((free_b - cand_total) * 0.94) : 0;
  const uint64_t per_state = (uint64_t)W * 8 + 8;
  if (E.table_log2 == 0 && E.max_states == 0) {
    int lg = 34;
    while (lg > 16 && (E.slot_bytes() << lg) + (uint64_t)((1ull << lg) / 2.5) * per_state > budget) --lg;
    E.table_log2 = lg;
    E.max_states = (uint64_t)((1ull << lg) / 2.5);
  } else if (E.table_log2 == 0) {
    int lg = 16;
    while (lg < 34 && (1ull << lg) < (uint64_t)(2.5 * (double)E.max_states)) ++lg;
    E.table_log2 = lg;
  }
  if (E.spill && E.max_states) {
    uint64_t p2 = 1;
    while (p2 * 2 <= E.max_states) p2 *= 2;
    E.max_states = p2;                                  // the spilling store is a power-of-two ring
  }
  E.table_slots = 1ull << E.table_log2;
  if (E.max_states == 0) {
    const uint64_t table_bytes = E.table_slots * E.slot_bytes();
    const uint64_t room = budget > table_bytes ? (budget - table_bytes) / per_state : 0;
    E.max_states = std::max<uint64_t>(1024, std::min<uint64_t>(E.table_slots / 2, room));
    if (E.spill) {
      uint64_t p2 = 1;
      while (p2 * 2 <= E.max_states) p2 *= 2;
      E.max_states = p2;
    }
  }
  E.region_rows = E.cand_bytes / (ROW * 8) / E.world;
  if (E.region_rows < (uint64_t)M::MAX_FANOUT) E.region_rows = M::MAX_FANOUT;
  // A chunk of frontier states is sized for `fanout_bound` successors per state on average *per owner region*.
  // MAX_FANOUT (emit sites in expand) is a safe but very loose bound -- reachable states enable a small
  // fraction of the sites (max 15 successors seen on the Kafka models, MAX_FANOUT ~100); the default
  // assumes <= 32 and relies on the kernel's overflow check (KMC_E_CAND_FULL, nothing is lost silently).
  if (E.fanout_bound == 0) E.fanout_bound = std::min<uint32_t>((uint32_t)M::MAX_FANOUT, 32u);
  E.chunk_states = std::max<uint64_t>(1, E.region_rows / E.fanout_bound);
  if (E.own_stream) CK(cudaStreamCreateWithFlags(&E.stream, cudaStreamNonBlocking));
  CK(cudaMalloc(&E.table, E.table_slots * E.slot_bytes()));
  CK(cudaMalloc(&E.store, E.max_states * W * 8));
  CK(cudaMalloc(&E.parent, E.max_states * 8));
  CK(cudaMalloc(&E.cand, E.region_rows * E.world * ROW * 8));
  if (E.world > 1) {
    E.recv_rows = E.region_rows * E.world;
    CK(cudaMalloc(&E.recv, E.recv_rows * ROW * 8));
    E.inbox_stride = INBOX_HEADER + E.region_rows * E.world * ROW;
    CK(cudaMalloc(&E.inbox_alloc, (SYNC_WORDS + 2 * E.inbox_stride) * 8));
    CK(cudaMemset(E.inbox_alloc, 0, (SYNC_WORDS + 2 * E.inbox_stride) * 8));
    E.inbox = E.inbox_alloc + SYNC_WORDS;
    CK(cudaHostAlloc(&E.board_host, MAX_WORLD * BOARD_WORDS * 8, cudaHostAllocMapped));
    memset(E.board_host, 0, MAX_WORLD * BOARD_WORDS * 8);
  }
  // the expand kernel keeps its state tile, the successor stage and the pair list in > 48 KB of dynamic shared memory
  CK(cudaFuncSetAttribute(k_expand, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)EXPAND_SMEM_BYTES));
  CK(cudaMalloc(&E.ctr, sizeof(DevCounters)));
  CK(cudaMalloc(&E.viol_ring, (size_t)(INV_REPORT && E.cont ? 3 : 1) * VIOL_RING * VIOL_ROW * 8));   // (see inv_ring_of)
  CK(cudaEventCreate(&E.ev_begin));
  CK(cudaEventCreate(&E.ev_end));
  return KMC_OK;
}

// ---- set_spill: host side ----------------------------------------------------------------------------------------
// The table takes keys up to half its slots per epoch (the probe sequence stays short); then its keys move to host
// memory.  cand (unused by the single-rank fused path) holds the marks at its end and the filter's and the flush's
// working space before them.
static uint64_t set_limit(const Engine& E) { return E.table_slots / 2; }
static uint64_t set_mark_words(const Engine& E) { return (E.table_slots + 63) / 64; }
static uint64_t set_scratch_words(const Engine& E) { return E.region_rows * E.world * ROW - set_mark_words(E); }
static unsigned* set_marks(const Engine& E) { return reinterpret_cast<unsigned*>(E.cand + set_scratch_words(E)); }
// states per compaction piece: W + 1 words of survivors, a keep byte and a tile counter each
static uint64_t set_piece(const Engine& E) { return set_scratch_words(E) / (ROW + 1) / SET_TILE * SET_TILE; }

static int set_alloc(Engine& E) {
  const uint64_t limit = set_limit(E);
  if (limit < (uint64_t)M::MAX_FANOUT) {
    E.last_error = "set_spill: half the table's slots must hold one state's successors (raise table_log2)";
    return KMC_E_BADARG;
  }
  if (E.region_rows * E.world * ROW <= set_mark_words(E) || set_piece(E) == 0) {
    E.last_error = "set_spill: the candidate buffer cannot hold the filter's marks and working space (raise cand_bytes)";
    return KMC_E_BADARG;
  }
  E.set_stage_keys = std::min<uint64_t>(1 << 20, set_scratch_words(E) / (2 * E.key_words()));
  for (int b = 0; b < 2; ++b) {
    CK(cudaHostAlloc(&E.set_pinned[b], E.set_stage_keys * E.key_words() * 8, cudaHostAllocDefault));
    CK(cudaEventCreateWithFlags(&E.set_copied[b], cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&E.set_probed[b], cudaEventDisableTiming));
  }
  CK(cudaStreamCreateWithFlags(&E.set_copy_stream, cudaStreamNonBlocking));
  return KMC_OK;
}

static uint64_t ring_run(const Engine& E, uint64_t g, uint64_t end, uint64_t* slot);

// The store tail and the fail flag (one copy: the counters from store_tail to fail are contiguous).
static int read_tail(Engine& E, uint64_t* tail, uint64_t* fail) {
  constexpr size_t first = offsetof(DevCounters, store_tail), end = offsetof(DevCounters, fail) + 8;
  unsigned long long w[(end - first) / 8];
  CK(cudaMemcpyAsync(w, &E.ctr->store_tail, end - first, cudaMemcpyDeviceToHost, E.stream));
  CK(cudaStreamSynchronize(E.stream));
  *tail = w[0];
  *fail = w[(end - first) / 8 - 1];
  return KMC_OK;
}

// Every key of the table that the last filter did not find in host memory is appended to host_keys, in slot ranges that
// fit the scratch space; then the table and the marks are emptied and a new epoch begins.  Host memory running out is
// KMC_E_OOM.
static int set_flush(Engine& E) {
  TimedLaunch t(E, 3);
  const uint64_t KW = E.key_words();
  const uint64_t range = set_scratch_words(E) / KW;
  for (uint64_t s0 = 0; s0 < E.table_slots; s0 += range) {
    const uint64_t n = std::min(range, E.table_slots - s0);
    CK(cudaMemsetAsync(&E.ctr->set_count, 0, sizeof(unsigned long long), E.stream));
    if (E.exact) k_set_flush<XS_ON><<<grid_for(E, n, 256, 8), 256, 0, E.stream>>>(E.table, s0, n, set_marks(E), E.cand, E.ctr);
    else k_set_flush<<<grid_for(E, n, 256, 8), 256, 0, E.stream>>>(E.table, s0, n, set_marks(E), E.cand, E.ctr);
    CK(cudaGetLastError());
    unsigned long long k = 0;
    CK(cudaMemcpyAsync(&k, &E.ctr->set_count, sizeof(k), cudaMemcpyDeviceToHost, E.stream));
    CK(cudaStreamSynchronize(E.stream));
    if (k == 0) continue;
    try {
      E.host_keys.emplace_back(k * KW);
    } catch (const std::bad_alloc&) {
      E.last_error = "set_spill: host memory for the fingerprint set's keys is exhausted";
      return KMC_E_OOM;
    }
    CK(cudaMemcpy(E.host_keys.back().data(), E.cand, k * KW * 8, cudaMemcpyDeviceToHost));
    E.set_host_keys += k;
    E.set_link_bytes += k * KW * 8;
  }
  CK(cudaMemsetAsync(E.table, E.empty_byte(), E.table_slots * E.slot_bytes(), E.stream));
  CK(cudaMemsetAsync(set_marks(E), 0, set_mark_words(E) * 8, E.stream));
  E.set_keys = 0;
  E.set_from = E.set_tail;
  E.set_flushes++;
  return KMC_OK;
}

// Marks the slot of every table key that is in host memory: the host keys stream through two pinned buffers into two
// staging areas of the scratch space, the copy of one chunk (on its own stream) overlapping the probes of the previous.
static int set_mark(Engine& E) {
  const uint64_t S = E.set_stage_keys, KW = E.key_words();
  uint64_t* stage[2] = {E.cand, E.cand + S * KW};
  const uint64_t bucket_mask = E.bucket_mask();
  // the staging areas are free once the work already on the engine stream (which may use the scratch space) is done
  for (int b = 0; b < 2; ++b) CK(cudaEventRecord(E.set_probed[b], E.stream));
  uint64_t k = 0;
  for (const std::vector<uint64_t>& block : E.host_keys) {
    const uint64_t nkeys = block.size() / KW;
    for (uint64_t i = 0; i < nkeys; i += S, ++k) {
      const int b = (int)(k & 1);
      const uint64_t n = std::min(S, nkeys - i);
      CK(cudaEventSynchronize(E.set_probed[b]));          // the probes of chunk k - 2 are done with buffer b
      memcpy(E.set_pinned[b], block.data() + i * KW, n * KW * 8);
      CK(cudaStreamWaitEvent(E.set_copy_stream, E.set_probed[b], 0));
      CK(cudaMemcpyAsync(stage[b], E.set_pinned[b], n * KW * 8, cudaMemcpyHostToDevice, E.set_copy_stream));
      CK(cudaEventRecord(E.set_copied[b], E.set_copy_stream));
      CK(cudaStreamWaitEvent(E.stream, E.set_copied[b], 0));
      if (E.exact) k_set_mark<XS_ON><<<grid_for(E, n, 256, 8), 256, 0, E.stream>>>(E.table, bucket_mask, stage[b], n, set_marks(E));
      else k_set_mark<<<grid_for(E, n, 256, 8), 256, 0, E.stream>>>(E.table, bucket_mask, stage[b], n, set_marks(E));
      CK(cudaGetLastError());
      CK(cudaEventRecord(E.set_probed[b], E.stream));
    }
  }
  E.set_link_bytes += E.set_host_keys * KW * 8;
  return KMC_OK;
}

// The filter: the states appended since the last one whose key is in host memory were found in an earlier epoch.  They
// are removed, and the survivors are compacted in place, in their order, piece by piece (a piece's survivors go to the
// scratch space, then back to the store behind the previous pieces' survivors): nothing points at the level being
// built until it is expanded.  store_tail, set_filtered and the per-action distinct counts follow.
// After a failure the filter does nothing and end_level reports the error: once the store is full, the inserts still
// count store_tail up but write no rows, so [set_from, tail) would reach past the store (or, in a ring, onto the
// frontier being expanded).
static int set_filter(Engine& E) {
  if (E.set_host_keys == 0) return KMC_OK;            // nothing flushed yet: every appended state is new
  uint64_t tail, fail;
  int rc = read_tail(E, &tail, &fail);
  if (rc || fail) return rc;
  E.set_keys += tail - E.set_tail;
  E.set_tail = tail;
  if (tail == E.set_from) return KMC_OK;
  TimedLaunch t(E, 3);
  if ((rc = set_mark(E))) return rc;
  const uint64_t P = set_piece(E);
  uint64_t* out_states = E.cand;
  uint64_t* out_parents = out_states + P * W;
  uint8_t* keep = reinterpret_cast<uint8_t*>(out_parents + P);
  unsigned long long* tiles = reinterpret_cast<unsigned long long*>(keep + P);
  const Params p = E.params();
  uint64_t cursor = E.set_from;
  for (uint64_t g = E.set_from; g < tail; g += P) {
    const uint64_t n = std::min(P, tail - g);
    const int grid = grid_for(E, n, SET_TILE, 8);
    k_set_compact<<<grid, SET_TILE, 0, E.stream>>>(p, g, n, set_marks(E), keep, tiles);
    k_set_scan<<<1, 1024, 0, E.stream>>>(tiles, (n + SET_TILE - 1) / SET_TILE, E.ctr);
    k_set_scatter<<<grid, SET_TILE, 0, E.stream>>>(p, g, n, keep, tiles, out_states, out_parents);
    CK(cudaGetLastError());
    unsigned long long kept = 0;
    CK(cudaMemcpyAsync(&kept, &E.ctr->set_count, sizeof(kept), cudaMemcpyDeviceToHost, E.stream));
    CK(cudaStreamSynchronize(E.stream));
    for (uint64_t c = cursor, slot, m; c < cursor + kept; c += m) {
      m = ring_run(E, c, cursor + kept, &slot);
      CK(cudaMemcpyAsync(E.store + slot * W, out_states + (c - cursor) * W, m * W * 8, cudaMemcpyDeviceToDevice, E.stream));
      CK(cudaMemcpyAsync(E.parent + slot, out_parents + (c - cursor), m * 8, cudaMemcpyDeviceToDevice, E.stream));
    }
    cursor += kept;
  }
  const unsigned long long new_tail = cursor;
  CK(cudaMemcpyAsync(&E.ctr->store_tail, &new_tail, sizeof(new_tail), cudaMemcpyHostToDevice, E.stream));
  CK(cudaStreamSynchronize(E.stream));
  E.set_filtered += tail - cursor;
  E.set_from = E.set_tail = cursor;
  return KMC_OK;
}

// At a chunk boundary (one counter read): the table's keys of this epoch are brought up to date; when the room left
// below set_limit() would cut the chunk below a quarter of the limit's worth of states, the epoch ends (filter, then
// flush).  The chunk then gets at most room / MAX_FANOUT states -- MAX_FANOUT is a true bound on a state's successors,
// unlike fanout_bound, an assumed average -- so its successors, and so its inserts, fit the room whatever the states;
// Params::region_rows (the KMC_E_CAND_FULL check of the expand kernel) is capped to the room as well.  After a failure
// the chunk is left as it is: the run ends at the level end with that error.  `per_item`: inserts one item of the chunk
// can make (a state's successors; 1 for a candidate of the device Init).
static int set_room(Engine& E, uint64_t* count, uint64_t* bound, uint64_t per_item = (uint64_t)M::MAX_FANOUT) {
  uint64_t tail, fail;
  int rc = read_tail(E, &tail, &fail);
  if (rc || fail) return rc;
  E.set_keys += tail - E.set_tail;
  E.set_tail = tail;
  const uint64_t limit = set_limit(E), F = per_item;
  auto room = [&] { return E.set_keys < limit ? limit - E.set_keys : 0; };
  if (room() / F < std::min<uint64_t>(*count, std::max<uint64_t>(1, limit / F / 4))) {
    if ((rc = set_filter(E)) || (rc = set_flush(E))) return rc;
  }
  *count = std::min(*count, room() / F);
  *bound = std::min(E.region_rows, room());
  return KMC_OK;
}

static uint64_t all_invariants() { return M::NUM_INVARIANTS >= 64 ? ~0ull : (1ull << M::NUM_INVARIANTS) - 1; }

// The per-invariant report starts afresh (every invariant pending) and, under "continue", the recorder is switched on.
static int inv_begin(Engine& E, bool complete) {
  const bool on = INV_REPORT && E.cont;
  E.inv_reports.clear();
  E.inv_pending = on ? all_invariants() : 0;
  E.inv_complete = complete;
  const unsigned long long w[6] = {on ? 1ull : 0ull, E.inv_pending, 0, 0, 0, 0};   // inv_on .. inv_viol_seen
  CK(cudaMemcpyAsync(&E.ctr->inv_on, w, sizeof(w), cudaMemcpyHostToDevice, E.stream));
  return KMC_OK;
}

static int engine_reset(Engine& E) {
  CK(cudaSetDevice(E.device));
  CK(cudaMemsetAsync(E.table, E.empty_byte(), E.table_slots * E.slot_bytes(), E.stream));
  DevCounters h;
  memset(&h, 0, sizeof(h));
  CK(cudaMemcpyAsync(E.ctr, &h, sizeof(h), cudaMemcpyHostToDevice, E.stream));
  CK(cudaStreamSynchronize(E.stream));
  E.events_used = 0;
  E.launches.clear();
  E.widths.clear();
  E.viol = Counterexample();
  E.level_first = E.level_count = E.level = 0;
  E.store_base = 0;
  E.host_store.clear();
  E.host_parent.clear();
  E.host_keys.clear();
  E.set_host_keys = 0;
  E.set_keys = E.set_tail = E.set_from = E.set_flushes = E.set_filtered = E.set_link_bytes = 0;
  if (E.set_spill) CK(cudaMemsetAsync(set_marks(E), 0, set_mark_words(E) * 8, E.stream));
  {
    std::lock_guard<std::mutex> g(E.mu);
    std::fill(E.site_generated.begin(), E.site_generated.end(), 0);
    std::fill(E.action_distinct.begin(), E.action_distinct.end(), 0);
    std::fill(E.inv_count.begin(), E.inv_count.end(), 0);
    E.coverage_complete = true;
  }
  return inv_begin(E, true);
}

// The stats and coverage that come from the device counters (the caller holds E.mu).  kmc_run clamps distinct to
// the store (`clamp`): without spill, a run that overflowed the store counted states it could not keep.
static void publish(Engine& E, const DevCounters& h, bool clamp) {
  kmc_stats_t& st = E.stats;
  st.distinct = clamp && !E.spill ? std::min<uint64_t>(h.store_tail, E.max_states) : h.store_tail;
  st.generated = h.generated;
  st.deadlocks = h.deadlocks;
  st.out_of_model = h.out_of_model;
  st.probes = h.probes;
  st.table_slots = E.table_slots;
  st.slot_bytes = E.slot_bytes();
  st.max_states = E.max_states;
  st.set_flushes = E.set_flushes;
  st.set_host_keys = E.set_host_keys;
  st.set_filtered = E.set_filtered;
  st.set_link_bytes = E.set_link_bytes;
#ifdef KMC_HAS_DEVICE_INIT
  st.init_generated = h.init_generated;
#else
  st.init_generated = E.rank == 0 ? M::NUM_INIT : 0;
#endif
  st.init_candidates = h.init_candidates;
  E.site_generated.assign(h.site_generated, h.site_generated + M::NUM_SITES);
  E.action_distinct.assign(h.action_distinct, h.action_distinct + M::NUM_ACTIONS);
  E.inv_count.assign(h.inv_count, h.inv_count + 64);
}

static int read_counters(Engine& E, DevCounters* h) {
  CK(cudaMemcpyAsync(h, E.ctr, sizeof(DevCounters), cudaMemcpyDeviceToHost, E.stream));
  CK(cudaStreamSynchronize(E.stream));
  return KMC_OK;
}

static int fail_to_error(unsigned long long f) {
  switch (f) {
    case 0: return KMC_OK;
    case KMC_FAIL_LAYOUT: return KMC_E_LAYOUT_OVERFLOW;
    case KMC_FAIL_TABLE_FULL: return KMC_E_TABLE_FULL;
    case KMC_FAIL_STORE_FULL: return KMC_E_STORE_FULL;
    case KMC_FAIL_CAND_FULL: return KMC_E_CAND_FULL;
    case KMC_FAIL_PEER_TIMEOUT: return KMC_E_PEER_TIMEOUT;
    case KMC_FAIL_SET_TIMEOUT: return KMC_E_SET_TIMEOUT;
    default: return KMC_E_CUDA;
  }
}

// writes the init states as candidate rows (one region per owner) -- host side, tiny
static int seed_init(Engine& E) {
  std::vector<uint64_t> rows[MAX_WORLD];
  unsigned long long counts[MAX_WORLD] = {0};
  for (int i = 0; i < M::NUM_INIT; ++i) {
    State s;
    memcpy(s.w, M::INIT_STATES[i], sizeof(s.w));
    uint32_t d = E.world > 1 ? owner_of(state_fp(s), E.world) : 0;
    // every rank seeds the same init states but only rank 0 contributes them, so that the
    // generated count and the exchange see each init state exactly once
    if (E.rank != 0) continue;
    for (int k = 0; k < W; ++k) rows[d].push_back(s.w[k]);
    rows[d].push_back(NO_PARENT);
    counts[d]++;
  }
  for (uint32_t d = 0; d < E.world; ++d) {
    if (counts[d] == 0) continue;
    if (counts[d] > E.region_rows) return KMC_E_OOM;
    CK(cudaMemcpyAsync(E.cand + (uint64_t)d * E.region_rows * ROW, rows[d].data(), rows[d].size() * 8,
                       cudaMemcpyHostToDevice, E.stream));
  }
  CK(cudaMemcpyAsync(E.ctr, counts, sizeof(counts), cudaMemcpyHostToDevice, E.stream));
  unsigned long long gen = E.rank == 0 ? M::NUM_INIT : 0;
  CK(cudaMemcpyAsync(&E.ctr->generated, &gen, sizeof(gen), cudaMemcpyHostToDevice, E.stream));
  CK(cudaStreamSynchronize(E.stream));
  return KMC_OK;
}

#ifdef KMC_HAS_DEVICE_INIT
// Level 1 from the device form of Init: each branch's candidate space in chunks of at most region_rows candidates.  A
// candidate yields at most one initial state, so a chunk's inserts are bounded like a frontier chunk's successors:
// by the store (KMC_E_STORE_FULL) and, under set_spill, by the room left before the next flush, which may then fall
// in the middle of level 1.
static int seed_device_init(Engine& E) {
  const Params p = E.params();
  for (int b = 0; b < M::INIT_BRANCHES; ++b) {
    for (uint64_t off = 0, cnt; off < M::INIT_SPACE[b]; off += cnt) {
      cnt = std::min<uint64_t>(std::max<uint64_t>(1, E.region_rows), M::INIT_SPACE[b] - off);
      uint64_t tail, fail, bound = 0;
      int rc = read_tail(E, &tail, &fail);
      if (rc) return rc;
      if (fail) return KMC_OK;                     // the level end reports it
      if (E.set_spill && (rc = set_room(E, &cnt, &bound, 1))) return rc;
      if (cnt == 0) return KMC_OK;                 // (set_room failed: the level end reports it)
      {
        TimedLaunch t(E, 4);
        k_init<<<grid_for(E, cnt, INIT_BLOCK, 8), INIT_BLOCK, 0, E.stream>>>(p, b, off, cnt);
      }
      CK(cudaGetLastError());
    }
  }
  return KMC_OK;
}
#endif

static int launch_insert(Engine& E, const uint64_t* rows, const unsigned long long* n_dev, uint64_t n_fixed,
                         uint64_t n_bound) {
  Params p = E.params();
  {
    TimedLaunch t(E, 1);
    k_insert<<<grid_for(E, n_bound, 256, 8), 256, 0, E.stream>>>(p, rows, n_dev, n_fixed);
  }
  CK(cudaGetLastError());
  return KMC_OK;
}

static int launch_invariants(Engine& E, uint64_t first, uint64_t count_bound) {
  if (M::NUM_INVARIANTS == 0) return KMC_OK;
  Params p = E.params();
  TimedLaunch t(E, 2);
  const int grid = grid_for(E, std::max<uint64_t>(count_bound, 1), 256, 8);
  k_invariants<<<grid, 256, 0, E.stream>>>(p, first, &E.ctr->store_tail);
  if (INV_REPORT && E.cont) k_invariant_report<<<grid, 256, 0, E.stream>>>(p, first, &E.ctr->store_tail);
  CK(cudaGetLastError());
  return KMC_OK;
}

// fused (kmc_run, one rank): the kernel inserts the successors itself; otherwise they go to the candidate buffer
// (or the owners' inboxes) for k_insert / k_insert_inbox.  cand_bound (set_spill): a smaller bound on the chunk's successors.
// the expand kernel's grid for `count` states; small levels get smaller tiles so that every SM still gets one (a tile
// is a multiple of 32 states)
static int expand_grid(const Engine& E, uint64_t count, unsigned* tile_states) {
  const uint64_t ctas = (uint64_t)E.sms;
  uint64_t per_cta = (count + ctas - 1) / ctas;
  *tile_states = (unsigned)std::min<uint64_t>((uint64_t)TILE, std::max<uint64_t>(32, (per_cta + 31) & ~31ull));
  uint64_t tiles = (count + *tile_states - 1) / *tile_states;
  return (int)std::min<uint64_t>(tiles, ctas);
}

static int launch_expand(Engine& E, uint64_t first, uint64_t count, bool p2p = false, bool fused = false, uint64_t cand_bound = 0) {
  Params p = E.params();
  p.p2p = p2p ? 1 : 0;
  p.fused = fused ? 1 : 0;
  if (cand_bound) p.region_rows = cand_bound;
  if (count == 0) return KMC_OK;
  TimedLaunch t(E, 0);
  unsigned tile_states;
  const int grid = expand_grid(E, count, &tile_states);
  k_expand<<<grid, EXPAND_BLOCK, EXPAND_SMEM_BYTES, E.stream>>>(p, first, count, tile_states);
  CK(cudaGetLastError());
  return KMC_OK;
}

static int reset_cand(Engine& E) {
  CK(cudaMemsetAsync(E.ctr->cand_count, 0, sizeof(unsigned long long) * MAX_WORLD, E.stream));
  return KMC_OK;
}

// The store by GLOBAL index: below store_base it is the host spill, from there on the device store, a ring when
// spilling.  Returns the device slot of index g and how many indices from g on, up to `end`, precede the ring's wrap.
static uint64_t ring_run(const Engine& E, uint64_t g, uint64_t end, uint64_t* slot) {
  *slot = E.spill ? (g & (E.max_states - 1)) : g;
  return E.spill ? std::min<uint64_t>(end - g, E.max_states - *slot) : end - g;
}

// Store range [first, first + count) -> host buffers; either may be null.  The device part is copied synchronously,
// after the stream synchronisation of the counter read that made the range known.
static int read_range(Engine& E, uint64_t first, uint64_t count, uint64_t* states, uint64_t* parents) {
  const uint64_t end = first + count, host_end = std::min(end, std::max(first, E.store_base));
  if (host_end > first) {
    if (states) memcpy(states, E.host_store.data() + first * W, (host_end - first) * W * 8);
    if (parents) memcpy(parents, E.host_parent.data() + first, (host_end - first) * 8);
  }
  for (uint64_t g = host_end, slot, n; g < end; g += n) {
    n = ring_run(E, g, end, &slot);
    if (states) CK(cudaMemcpy(states + (g - first) * W, E.store + slot * W, n * W * 8, cudaMemcpyDeviceToHost));
    if (parents) CK(cudaMemcpy(parents + (g - first), E.parent + slot, n * 8, cudaMemcpyDeviceToHost));
  }
  return KMC_OK;
}

// host buffers -> store range [first, first + count) (recover); the device part is copied on the engine stream
static int write_range(Engine& E, uint64_t first, uint64_t count, const uint64_t* states, const uint64_t* parents) {
  const uint64_t end = first + count, host_end = std::min(end, std::max(first, E.store_base));
  if (host_end > first) {
    memcpy(E.host_store.data() + first * W, states, (host_end - first) * W * 8);
    memcpy(E.host_parent.data() + first, parents, (host_end - first) * 8);
  }
  for (uint64_t g = host_end, slot, n; g < end; g += n) {
    n = ring_run(E, g, end, &slot);
    CK(cudaMemcpyAsync(E.store + slot * W, states + (g - first) * W, n * W * 8, cudaMemcpyHostToDevice, E.stream));
    CK(cudaMemcpyAsync(E.parent + slot, parents + (g - first), n * 8, cudaMemcpyHostToDevice, E.stream));
  }
  return KMC_OK;
}

// Spill: everything below the level that is expanded next moves to host memory and its ring slots become free.
static int spill_below(Engine& E, uint64_t level_first) {
  if (!E.spill || level_first <= E.store_base) return KMC_OK;
  const uint64_t base = E.store_base;
  E.host_store.resize(level_first * W);
  E.host_parent.resize(level_first);
  int rc = read_range(E, base, level_first - base, E.host_store.data() + base * W, E.host_parent.data() + base);
  if (rc) return rc;
  E.store_base = level_first;
  return KMC_OK;
}

// ---- kmc_edges: the transitions out of stored states -------------------------------------------------------------
// The states [first, first + count) are expanded again, chunk by chunk, by the non-fused expand kernel into the
// candidate buffer, and k_edges turns its rows into edges.  Nothing of the run changes: both kernels count into scratch
// counters, deadlocks are not recorded (check_deadlock = 0) and nothing is inserted.  The candidate buffer (under
// set_spill only its scratch part: the filter's marks lie behind it) is cut into the candidate rows, the edge rows and
// a staging area for spilled states.  A chunk holds at most as many states as their MAX_FANOUT successors each fill, so
// neither kind of row can overflow.  Spilled states (below store_base) are read through read_range and copied to the
// staging area; the others are expanded in place, a chunk never crossing the ring's wrap.
static constexpr int EDGE_WORDS = sizeof(kmc_edge_t) / 8;
static_assert(sizeof(kmc_edge_t) == 32, "kmc_edge_t is four 64-bit words");

struct EdgeScratch {
  DevCounters ctr;
  unsigned long long edges;
};

static int edges_chunks(Engine& E, EdgeScratch* d, uint64_t first, uint64_t count, kmc_edge_t* out, size_t cap,
                        size_t* n) {
  const uint64_t F = std::max<uint64_t>(1, (uint64_t)M::MAX_FANOUT);
  const uint64_t words = E.set_spill ? set_scratch_words(E) : E.region_rows * ROW;
  const uint64_t chunk = words > 1 ? (words - 1) / (F * (ROW + EDGE_WORDS) + W) : 0;      // (- 1: the staging alignment)
  if (chunk == 0) {
    E.last_error = "kmc_edges: the candidate buffer cannot hold one state's successors and their edges (raise cand_bytes)";
    return KMC_E_BADARG;
  }
  uint64_t* rows = E.cand;
  kmc_edge_t* edges = reinterpret_cast<kmc_edge_t*>(E.cand + chunk * F * ROW);
  uint64_t* staging = E.cand + ((chunk * F * (ROW + EDGE_WORDS) + 1) & ~1ull);          // 16-byte aligned tile loads
  Params p = E.params();
  p.ctr = &d->ctr;
  p.check_deadlock = 0;
  p.region_rows = chunk * F;
  std::vector<uint64_t> host;
  size_t total = 0;
  for (uint64_t g = first, end = first + count, slot, cnt; g < end; g += cnt) {
    Params q = p;
    uint64_t start = g, offset = 0;
    if (g < E.store_base) {
      cnt = std::min({chunk, E.store_base - g, end - g});
      host.resize(cnt * W);
      if (int rc = read_range(E, g, cnt, host.data(), nullptr)) return rc;
      CK(cudaMemcpyAsync(staging, host.data(), cnt * W * 8, cudaMemcpyHostToDevice, E.stream));
      q.store = staging;
      q.store_mask = ~0ull;
      start = 0;
      offset = g;
    } else {
      cnt = std::min(chunk, ring_run(E, g, end, &slot));
    }
    CK(cudaMemsetAsync(d, 0, sizeof(EdgeScratch), E.stream));
    unsigned tile_states;
    const int grid = expand_grid(E, cnt, &tile_states);
    k_expand<<<grid, EXPAND_BLOCK, EXPAND_SMEM_BYTES, E.stream>>>(q, start, cnt, tile_states);
    k_edges<<<grid_for(E, cnt * F, 256, 8), 256, 0, E.stream>>>(rows, &d->ctr.cand_count[0], q.store, q.store_mask, offset,
                                                                p.region_rows, edges, &d->edges);
    CK(cudaGetLastError());
    unsigned long long fail = 0, k = 0;
    CK(cudaMemcpyAsync(&fail, &d->ctr.fail, 8, cudaMemcpyDeviceToHost, E.stream));
    CK(cudaMemcpyAsync(&k, &d->edges, 8, cudaMemcpyDeviceToHost, E.stream));
    CK(cudaStreamSynchronize(E.stream));
    // a successor that does not fit the layout (the unexpanded last level of a stopped run can hold one): an error
    if (fail) return fail_to_error(fail);
    if (total < cap) CK(cudaMemcpy(out + total, edges, std::min<uint64_t>(k, cap - total) * sizeof(kmc_edge_t),
                                   cudaMemcpyDeviceToHost));
    total += k;
  }
  *n = total;
  return KMC_OK;
}

static int engine_edges(Engine& E, uint64_t first, uint64_t count, kmc_edge_t* out, size_t cap, size_t* n) {
  EdgeScratch* d = nullptr;
  CK(cudaMalloc(&d, sizeof(EdgeScratch)));
  const int rc = edges_chunks(E, d, first, count, out, cap, n);
  cudaFree(d);
  return rc;
}

// ---- checkpoint / recover (TLC -checkpoint / -recover): written at a level boundary -------------------------------
// <dir>/checkpoint.meta  text: key value per line;  <dir>/checkpoint.bin  states [0, tail) then parent words [0, tail).
// The fingerprint set is not stored: it is rebuilt from the states on recover (and may then have another size).
static int write_checkpoint(Engine& E, const DevCounters& h) {
  const std::string meta = E.checkpoint_dir + "/checkpoint.meta", bin = E.checkpoint_dir + "/checkpoint.bin";
  const std::string tmp = bin + ".tmp";
  FILE* f = fopen(tmp.c_str(), "wb");
  if (!f) {
    E.last_error = "cannot write " + tmp;
    return KMC_E_BADARG;
  }
  // the states, then the parent words, through a bounded buffer: with spill most of the store is in host memory
  const uint64_t tail = h.store_tail, piece = 1 << 20;
  std::vector<uint64_t> buf;
  bool ok = true;
  for (int parents = 0; parents < 2 && ok; ++parents)
    for (uint64_t g = 0; g < tail && ok; g += piece) {
      const uint64_t n = std::min(piece, tail - g);
      buf.resize(parents ? n : n * W);
      int rc = read_range(E, g, n, parents ? nullptr : buf.data(), parents ? buf.data() : nullptr);
      if (rc) { fclose(f); return rc; }
      ok = fwrite(buf.data(), 8, buf.size(), f) == buf.size();
    }
  ok = (fclose(f) == 0) && ok;
  if (!ok || rename(tmp.c_str(), bin.c_str()) != 0) {
    E.last_error = "short write on " + tmp;
    return KMC_E_BADARG;
  }
  f = fopen((meta + ".tmp").c_str(), "w");
  if (!f) return KMC_E_BADARG;
  fprintf(f, "model %s\ndigest %s\nwords %d\ntail %llu\nlevel_first %llu\nlevel_end %llu\nlevel %llu\ngenerated %llu\n"
             "deadlocks %llu\nout_of_model %llu\nprobes %llu\nsite_generated",
          KMC_MODEL_NAME, KMC_MODEL_DIGEST, W, (unsigned long long)tail, (unsigned long long)E.level_first,
          (unsigned long long)(E.level_first + E.level_count), (unsigned long long)E.level, (unsigned long long)h.generated,
          (unsigned long long)h.deadlocks, (unsigned long long)h.out_of_model, (unsigned long long)h.probes);
  // (before widths: a reader stops at widths.  Distinct per action is not written: it is the histogram of the
  // parent words, which recover reads anyway)
  for (int i = 0; i < M::NUM_SITES; ++i) fprintf(f, " %llu", (unsigned long long)h.site_generated[i]);
#ifdef KMC_HAS_DEVICE_INIT
  fprintf(f, "\ninit_generated %llu\ninit_candidates %llu", h.init_generated, h.init_candidates);
#endif
  fprintf(f, "\nwidths");
  for (uint64_t w : E.widths) fprintf(f, " %llu", (unsigned long long)w);
  fprintf(f, "\n");
  fclose(f);
  if (rename((meta + ".tmp").c_str(), meta.c_str()) != 0) return KMC_E_BADARG;
  E.last_checkpoint = std::chrono::steady_clock::now();
  return KMC_OK;
}

// Sets the level cursor to the level the checkpoint expands next, and *h to the counters it restored.
static int read_checkpoint(Engine& E, DevCounters* h) {
  const std::string meta = E.recover_dir + "/checkpoint.meta", bin = E.recover_dir + "/checkpoint.bin";
  FILE* f = fopen(meta.c_str(), "r");
  if (!f) {
    E.last_error = "cannot read " + meta;
    return KMC_E_BADARG;
  }
  char key[64], val[256];
  unsigned long long tail = 0, words = 0, level_first = 0, level_end = 0, level = 1;
  std::string digest;
  bool have_sites = false;
  memset(h, 0, sizeof(*h));
  E.widths.clear();
  while (fscanf(f, "%63s", key) == 1) {
    if (!strcmp(key, "widths")) {
      unsigned long long w;
      while (fscanf(f, "%llu", &w) == 1) E.widths.push_back(w);
      break;
    }
    if (!strcmp(key, "site_generated")) {
      int i = 0;
      for (; i < M::NUM_SITES && fscanf(f, "%llu", &h->site_generated[i]) == 1; ++i) {}
      have_sites = i == M::NUM_SITES;
      continue;
    }
    if (fscanf(f, "%255s", val) != 1) break;
    const unsigned long long v = strtoull(val, nullptr, 10);
    if (!strcmp(key, "digest")) digest = val;
    else if (!strcmp(key, "words")) words = v;
    else if (!strcmp(key, "tail")) tail = v;
    else if (!strcmp(key, "level_first")) level_first = v;
    else if (!strcmp(key, "level_end")) level_end = v;
    else if (!strcmp(key, "level")) level = v;
    else if (!strcmp(key, "generated")) h->generated = v;
    else if (!strcmp(key, "deadlocks")) h->deadlocks = v;
    else if (!strcmp(key, "out_of_model")) h->out_of_model = v;
    else if (!strcmp(key, "probes")) h->probes = v;
    else if (!strcmp(key, "init_generated")) h->init_generated = v;
    else if (!strcmp(key, "init_candidates")) h->init_candidates = v;
  }
  fclose(f);
  if (digest != KMC_MODEL_DIGEST || words != (unsigned long long)W) {
    E.last_error = "checkpoint belongs to another model (digest mismatch)";
    return KMC_E_MODEL;
  }
  h->store_tail = tail;
  // states below the level to expand go to the host (spill) or, without spill, everything to the device
  const uint64_t keep_from = E.spill ? level_first : 0;
  if (tail - keep_from > E.max_states) {
    E.last_error = "checkpoint does not fit the state store (raise max_states or use spill)";
    return KMC_E_STORE_FULL;
  }
  f = fopen(bin.c_str(), "rb");
  if (!f) {
    E.last_error = "cannot read " + bin;
    return KMC_E_BADARG;
  }
  std::vector<uint64_t> st((size_t)tail * W), pa((size_t)tail);
  bool ok = fread(st.data(), 8, st.size(), f) == st.size() && fread(pa.data(), 8, pa.size(), f) == pa.size();
  fclose(f);
  if (!ok) {
    E.last_error = "short read on " + bin;
    return KMC_E_BADARG;
  }
  // distinct per action: the action bits of the stored parent words (initial states have none)
  for (uint64_t g = 0; g < tail; ++g) {
    if ((pa[g] & 0x0000FFFFFFFFFFFFull) == NO_PARENT) continue;
    const uint64_t a = pa[g] >> 56;
    if (a < (uint64_t)M::NUM_ACTIONS) h->action_distinct[a]++;
  }
  if (!have_sites) memset(h->site_generated, 0, sizeof(h->site_generated));
  E.coverage_complete = have_sites;      // a checkpoint written before the per-site counts existed: generated is partial
  E.store_base = keep_from;
  E.host_store.resize((size_t)keep_from * W);
  E.host_parent.resize((size_t)keep_from);
  int rc = write_range(E, 0, tail, st.data(), pa.data());
  if (rc) return rc;
  // the counters in one copy, before the rebuild: k_rebuild sets `fail` when the set overflows
  CK(cudaMemcpyAsync(E.ctr, h, sizeof(*h), cudaMemcpyHostToDevice, E.stream));
  // rebuild the set: every stored state is inserted once, in batches through the candidate buffer.  With set_spill
  // the batches stay clear of the marks, and the table is flushed whenever a batch would pass set_limit() (the states
  // are distinct: no filter is needed)
  Params p = E.params();
  uint64_t batch = E.region_rows * ROW / W;
  if (E.set_spill) batch = std::min(set_scratch_words(E) / W, set_limit(E));
  for (uint64_t g = 0; g < tail; g += batch) {
    const uint64_t n = std::min<uint64_t>(batch, tail - g);
    if (E.set_spill && E.set_keys + n > set_limit(E))
      if (int rc = set_flush(E)) return rc;
    CK(cudaMemcpyAsync(E.cand, st.data() + g * W, n * W * 8, cudaMemcpyHostToDevice, E.stream));
    k_rebuild<<<grid_for(E, n, 256, 8), 256, 0, E.stream>>>(p, E.cand, n);
    CK(cudaStreamSynchronize(E.stream));
    E.set_keys += n;
  }
  E.set_tail = E.set_from = tail;
  DevCounters now;
  if ((rc = read_counters(E, &now))) return rc;
  if ((rc = fail_to_error(now.fail))) return rc;
  E.level_first = level_first;
  E.level_count = level_end - level_first;
  E.level = level;
  return KMC_OK;
}

// The order of violators, the same for every pick: a deadlock first (it belongs to the level being expanded, before the
// invariant violations of the next level), then the smaller set-identity fingerprint, then the smaller parent word.
static std::tuple<bool, uint64_t, uint64_t> violator_key(bool deadlock, uint64_t fp, uint64_t meta) {
  return {!deadlock, fp, meta};
}
// Whether x is the better pick: x has a violator and y none, or x's comes first.
static bool better(const Counterexample& x, const Counterexample& y) {
  return !x.words.empty() &&
         (y.words.empty() || violator_key(x.inv < 0, x.fp, x.meta) < violator_key(y.inv < 0, y.fp, y.meta));
}

// The first of n ring rows in violator order.  inv < 0: every row of the violator ring, whose last word is the invariant
// or ~0 for a deadlock.  inv >= 0: the rows of the per-invariant ring whose last word, a set of invariants, holds `inv`;
// that ring has no deadlocks.  Null when no row qualifies.
static const uint64_t* pick(const uint64_t* rows, uint64_t n, int inv) {
  auto key = [inv](const uint64_t* r) { return violator_key(inv < 0 && r[W + 2] == ~0ull, r[W + 1], r[W]); };
  const uint64_t* best = nullptr;
  for (const uint64_t* r = rows; r < rows + n * VIOL_ROW; r += VIOL_ROW)
    if ((inv < 0 || (r[W + 2] >> inv) & 1) && (!best || key(r) < key(best))) best = r;
  return best;
}

static void take_row(Counterexample& x, const uint64_t* row) {
  x.words.assign(row, row + W);
  x.meta = row[W];
  x.fp = row[W + 1];
}

// The trace of x back to an initial state along the parent links, each parent read on its own rank (through that
// rank's host spill): `ranks` is {&E} for one rank, or every rank of a "gpus" context.  A parent on a rank not in
// `ranks` ends the walk (the multi-process driver's ranks each hold only their own part).  Errors go to E.
static int walk_trace(Engine& E, const std::vector<Engine*>& ranks, Counterexample& x) {
  std::vector<std::vector<uint64_t>> rev{x.words};
  std::vector<uint32_t> rev_act{(uint32_t)(x.meta >> 56)};
  uint64_t meta = x.meta, guard = 0;
  while ((meta & 0x0000FFFFFFFFFFFFull) != NO_PARENT && guard++ < 100000) {
    const uint64_t idx = meta & IDX_MASK;
    const uint32_t prank = (uint32_t)((meta >> 40) & 0xFF);
    Engine* P = nullptr;
    for (Engine* r : ranks)
      if (r->rank == prank) P = r;
    if (!P || (idx >= P->store_base && idx - P->store_base >= P->max_states)) break;
    std::vector<uint64_t> st(W);
    CK(cudaSetDevice(P->device));
    if (int rc = read_range(*P, idx, 1, st.data(), &meta)) {
      E.last_error = P->last_error;
      return rc;
    }
    rev.push_back(st);
    rev_act.push_back((uint32_t)(meta >> 56));
  }
  x.trace.assign(rev.rbegin(), rev.rend());
  x.actions.assign(rev_act.rbegin(), rev_act.rend());
  return KMC_OK;
}

// The run's violation from the violator ring at the end of level `level` (the level being expanded, 0 for the init
// insert): the pick, its level and its trace on this rank.
static int build_trace(Engine& E, const DevCounters& h, uint64_t level) {
  uint64_t n = std::min<uint64_t>(h.viol_count, VIOL_RING);
  if (n == 0) return KMC_OK;
  std::vector<uint64_t> ring(n * VIOL_ROW);
  CK(cudaMemcpy(ring.data(), E.viol_ring, ring.size() * 8, cudaMemcpyDeviceToHost));
  const uint64_t* best = pick(ring.data(), n, -1);
  Counterexample x;
  x.inv = best[W + 2] == ~0ull ? -1 : (int32_t)best[W + 2];
  x.level = x.inv < 0 ? level : level + 1;
  take_row(x, best);
  if (int rc = walk_trace(E, {&E}, x)) return rc;
  E.viol = std::move(x);
  return KMC_OK;
}

// Level end of a "continue" run: every pending invariant that a state of level `level` violates (`fresh`: the inv_new
// words of the ranks, ORed) is reported -- its violators at that level (before it, it had none) and its pick from the
// per-invariant ring.  `walk`: walk the pick's trace now (one rank; multi_run walks across the ranks).  Then those
// invariants stop being pending and the rings empty.  A level with more discarded violators than the stage holds
// makes the report incomplete.
static int collect_invariants(Engine& E, const DevCounters& h, uint64_t level, uint64_t fresh, bool walk) {
  fresh &= E.inv_pending;
  if (h.inv_staged > (uint64_t)VIOL_RING) E.inv_complete = false;
  const uint64_t n = fresh ? std::min<uint64_t>(h.inv_rows, VIOL_RING) : 0;
  std::vector<uint64_t> ring(n * VIOL_ROW);
  if (n) CK(cudaMemcpy(ring.data(), inv_ring_of(E.viol_ring), ring.size() * 8, cudaMemcpyDeviceToHost));
  for (uint64_t b = fresh; b; b &= b - 1) {
    Counterexample x;
    x.inv = __builtin_ctzll(b);
    x.level = level;
    x.first_count = h.inv_count[x.inv];
    if (const uint64_t* best = pick(ring.data(), n, x.inv)) {
      take_row(x, best);
      if (walk)
        if (int rc = walk_trace(E, {&E}, x)) return rc;
    }
    E.inv_reports.push_back(std::move(x));
  }
  E.inv_pending &= ~fresh;
  const unsigned long long w[5] = {E.inv_pending, 0, 0, 0, h.viol_count};   // inv_pending .. inv_viol_seen
  CK(cudaMemcpyAsync(&E.ctr->inv_pending, w, sizeof(w), cudaMemcpyHostToDevice, E.stream));
  return KMC_OK;
}

static void accumulate_timing(Engine& E, kmc_stats_t& st) {
  st.gpu_ms_expand = st.gpu_ms_insert = st.gpu_ms_invariant = st.gpu_ms_set_spill = st.gpu_ms_init = 0;
  st.launches_expand = st.launches_insert = st.launches_other = 0;
  for (const LaunchRec& r : E.launches) {
    float ms = 0;
    cudaEventElapsedTime(&ms, r.a, r.b);
    if (r.kind == 0) { st.gpu_ms_expand += ms; st.launches_expand++; }
    else if (r.kind == 1) { st.gpu_ms_insert += ms; st.launches_insert++; }
    else if (r.kind == 3) st.gpu_ms_set_spill += ms;
    else if (r.kind == 4) st.gpu_ms_init += ms;
    else { st.gpu_ms_invariant += ms; st.launches_other++; }
  }
}

// End of a level: invariants on the states it added (`inv_bound` bounds their grid), one counter read, the cursor
// moves on to those states, stats and coverage are published, and the first violation builds the trace.
// kmc_run (`shard` false) reports distinct clamped to the store and the queue, lists the widths of the levels it
// expands itself and does not trace a failed level; the shard calls list every non-empty level they find.
static int end_level(Engine& E, uint64_t inv_bound, bool shard, DevCounters& h) {
  const uint64_t end = E.level_first + E.level_count;
  int rc = launch_invariants(E, end, inv_bound);
  if (rc || (rc = read_counters(E, &h))) return rc;
  const uint64_t level = E.level++;
  E.level_first = end;
  E.level_count = h.store_tail - end;
  {
    std::lock_guard<std::mutex> g(E.mu);
    publish(E, h, !shard);
    if (shard && E.level_count) E.widths.push_back(E.level_count);
    E.stats.depth = E.widths.size();
    if (shard) E.stats.levels = E.stats.depth;
    else E.stats.queue = E.level_count;
  }
  if (h.viol_count && E.viol.words.empty() && (shard || !h.fail)) build_trace(E, h, level);
  if (INV_REPORT && E.cont && (shard || !h.fail)) return collect_invariants(E, h, level + 1, h.inv_new, true);
  return KMC_OK;
}

static int engine_run(Engine& E) {
  auto t0 = std::chrono::steady_clock::now();
  int rc = engine_reset(E);
  if (rc) return rc;
  if (E.world != 1) {
    E.last_error = "kmc_run drives one rank; use the kmc_shard_* calls for world > 1";
    return KMC_E_BADARG;
  }
  CK(cudaEventRecord(E.ev_begin, E.stream));
  DevCounters h;
  bool stopped = false;
  int err = 0;
  E.last_checkpoint = std::chrono::steady_clock::now();
  if (!E.recover_dir.empty()) {
    // -recover: continue from the level boundary a checkpoint was written at
    if ((rc = read_checkpoint(E, &h))) return rc;
    if ((rc = inv_begin(E, false))) return rc;
  } else {
#ifdef KMC_HAS_DEVICE_INIT
    if ((rc = seed_device_init(E))) return rc;
    if (E.set_spill && (rc = set_filter(E))) return rc;         // before k_invariants sees the level
    if ((rc = end_level(E, M::INIT_CANDIDATES, false, h))) return rc;
#else
    if ((rc = seed_init(E))) return rc;
    if ((rc = launch_insert(E, E.cand, &E.ctr->cand_count[0], 0, M::NUM_INIT))) return rc;
    if ((rc = end_level(E, M::NUM_INIT, false, h))) return rc;
#endif
    err = fail_to_error(h.fail);
    if (!err && h.viol_count && !E.cont) stopped = true;
  }
  while (!err && !stopped && E.level_count) {
    E.widths.push_back(E.level_count);
    if ((rc = spill_below(E, E.level_first))) return rc;         // (no-op unless spilling)
    const uint64_t level_end = E.level_first + E.level_count;
    for (uint64_t off = E.level_first, slot, cnt; off < level_end; off += cnt) {
      cnt = std::min<uint64_t>(E.chunk_states, ring_run(E, off, level_end, &slot));   // a chunk never crosses the wrap
      uint64_t bound = 0;
      if (E.set_spill && (rc = set_room(E, &cnt, &bound))) return rc;
      // one launch per chunk: the expand kernel inserts its successors itself (Params::fused); the candidate
      // counter only bounds the chunk's successors
      if ((rc = reset_cand(E))) return rc;
      if ((rc = launch_expand(E, off, cnt, false, true, bound))) return rc;
    }
    if (E.set_spill && (rc = set_filter(E))) return rc;         // before k_invariants sees the level
    if ((rc = end_level(E, E.level_count * 2, false, h))) return rc;
    err = fail_to_error(h.fail);
    if (!err && h.viol_count && !E.cont) {
      stopped = true;
      break;
    }
    if (!err && !E.checkpoint_dir.empty() && E.level_count) {
      const double mins = std::chrono::duration<double>(std::chrono::steady_clock::now() - E.last_checkpoint).count() / 60.0;
      if (mins >= E.checkpoint_minutes) {
        if ((rc = spill_below(E, E.level_first))) return rc;
        if ((rc = write_checkpoint(E, h))) return rc;
      }
    }
    if (E.stop_after_states && h.store_tail >= E.stop_after_states && E.level_count) {
      stopped = true;          // bounded throughput run: the queue is reported, no error
      break;
    }
  }
  CK(cudaEventRecord(E.ev_end, E.stream));
  CK(cudaStreamSynchronize(E.stream));
  float total_ms = 0;
  cudaEventElapsedTime(&total_ms, E.ev_begin, E.ev_end);
  auto t1 = std::chrono::steady_clock::now();
  {
    std::lock_guard<std::mutex> g(E.mu);
    publish(E, h, true);
    kmc_stats_t& st = E.stats;
    st.queue = stopped ? E.level_count : 0;
    st.depth = st.levels = E.widths.size();
    st.gpu_ms_total = total_ms;
    st.wall_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
    st.complete = (!err && !stopped) ? 1 : 0;
    if (E.timing) accumulate_timing(E, st);
    E.ran = true;
  }
  return err;
}

// ----------------------------------------------------------------------------------------
// exported per-model ABI (the dispatcher libkspecmc.so forwards kmc_* to these)
// ----------------------------------------------------------------------------------------
static int multi_create(kmcm_ctx* c, const char* options_json, int gpus);
static int multi_run(kmcm_ctx* c);

// A model whose Init is enumerated on the GPU (k_init) seeds level 1 on one GPU only: the sharded building blocks and
// the "gpus" / world > 1 contexts refuse it with this text.
static constexpr const char* DEVICE_INIT_ONE_GPU =
    "this model's Init is enumerated on the GPU (device Init), which runs on one GPU: no \"gpus\" > 1, no world > 1, "
    "no kmc_shard_* calls";
// An exact_set context keys its set by the packed state, which the exchange of fingerprint-sharded rows and the
// fingerprint-only kmc_fpset_* calls do not carry.
static constexpr const char* EXACT_SET_ONE_GPU =
    "exact_set runs on one GPU: no \"gpus\" > 1, no world > 1, no kmc_shard_* calls";
static constexpr const char* EXACT_SET_NO_FPSET =
    "exact_set keys the set by the packed state: a 64-bit fingerprint is not a key of it (no kmc_fpset_* calls)";
static bool shard_refused(Engine& e) {
  if (e.exact) {
    e.last_error = EXACT_SET_ONE_GPU;
    return true;
  }
#ifdef KMC_HAS_DEVICE_INIT
  e.last_error = DEVICE_INIT_ONE_GPU;
  return true;
#else
  (void)e;
  return false;
#endif
}

#define E (c->e)
extern "C" {

int kmcm_create(const char* options_json, kmcm_ctx** out) {
  if (!out) return KMC_E_BADARG;
  kmcm_ctx* c = new kmcm_ctx();
  double d;
  bool b;
  if (json_num(options_json, "device", &d)) E.device = (int)d;
  if (json_num(options_json, "table_log2", &d)) E.table_log2 = (int)d;
  if (json_num(options_json, "max_states", &d)) E.max_states = (uint64_t)d;
  if (json_num(options_json, "cand_bytes", &d)) E.cand_bytes = (uint64_t)d;
  if (json_num(options_json, "rank", &d)) E.rank = (uint32_t)d;
  if (json_num(options_json, "world", &d)) E.world = (uint32_t)d;
  if (json_bool(options_json, "continue", &b)) E.cont = b;
  if (json_bool(options_json, "check_deadlock", &b)) E.check_deadlock = b;
  if (json_bool(options_json, "timing", &b)) E.timing = b;
  if (json_num(options_json, "stop_after_states", &d)) E.stop_after_states = (uint64_t)d;
  if (json_bool(options_json, "spill", &b)) E.spill = b;
  if (json_bool(options_json, "set_spill", &b)) E.set_spill = b;
  if (json_bool(options_json, "exact_set", &b)) E.exact = b && !EXACT_SET;      // (an exact key already: nothing to do)
  json_str(options_json, "checkpoint_dir", &E.checkpoint_dir);
  json_str(options_json, "recover", &E.recover_dir);
  if (json_num(options_json, "checkpoint_minutes", &d)) E.checkpoint_minutes = d;
  if (json_num(options_json, "fanout_bound", &d)) E.fanout_bound = (uint32_t)d;
  if (json_num(options_json, "stream", &d) && d != 0) {
    // a cudaStream_t handle of the calling process (e.g. torch.cuda.current_stream().cuda_stream): engine
    // kernels are then ordered with the caller's own work (NCCL exchange) without host synchronisation
    E.stream = reinterpret_cast<cudaStream_t>((uintptr_t)d);
    E.own_stream = false;
  }
  if (E.world < 1 || E.world > MAX_WORLD || E.rank >= E.world || (E.table_log2 && (E.table_log2 < 4 || E.table_log2 > 34))) {
    delete c;
    return KMC_E_BADARG;
  }
  const bool gpus = json_num(options_json, "gpus", &d) && d > 1;
#ifdef KMC_HAS_DEVICE_INIT
  if (gpus || E.world > 1) {
    E.last_error = DEVICE_INIT_ONE_GPU;
    *out = c;
    return KMC_E_BADARG;
  }
#endif
  if (E.exact && (gpus || E.world > 1)) {
    E.last_error = EXACT_SET_ONE_GPU;
    *out = c;
    return KMC_E_BADARG;
  }
  if (E.set_spill && (gpus || E.world > 1)) {
    // each rank's set would need the keys of the others' host memory too
    E.last_error = "set_spill runs on one GPU (no \"gpus\" > 1, no world > 1)";
    *out = c;
    return KMC_E_BADARG;
  }
  if (gpus) {
    *out = c;
    return multi_create(c, options_json, (int)d);
  }
  int rc = engine_alloc(E);
  *out = c;   // returned even on failure so that the caller can read the error text
  if (rc == KMC_OK && E.set_spill) rc = set_alloc(E);
  if (rc == KMC_OK) rc = engine_reset(E);
  return rc;
}

void kmcm_destroy(kmcm_ctx* c) {
  if (!c) return;
  if (!c->ranks.empty()) {
    for (kmcm_ctx* r : c->ranks) kmcm_destroy(r);
    delete c;
    return;
  }
  cudaSetDevice(E.device);
  cudaFree(E.table);
  cudaFree(E.store);
  cudaFree(E.parent);
  cudaFree(E.cand);
  cudaFree(E.recv);
  if (E.peers_open)
    for (uint32_t r = 0; r < E.world; ++r)
      if (r != E.rank && E.peer_inbox[r] && !E.peers_direct) cudaIpcCloseMemHandle(E.peer_inbox[r] - SYNC_WORDS);
  cudaFree(E.inbox_alloc);
  if (E.board_host) cudaFreeHost(E.board_host);
  cudaFree(E.ctr);
  cudaFree(E.viol_ring);
  for (int b = 0; b < 2; ++b) {
    if (E.set_pinned[b]) cudaFreeHost(E.set_pinned[b]);
    if (E.set_copied[b]) cudaEventDestroy(E.set_copied[b]);
    if (E.set_probed[b]) cudaEventDestroy(E.set_probed[b]);
  }
  if (E.set_copy_stream) cudaStreamDestroy(E.set_copy_stream);
  for (cudaEvent_t ev : E.event_pool) cudaEventDestroy(ev);
  if (E.ev_begin) cudaEventDestroy(E.ev_begin);
  if (E.ev_end) cudaEventDestroy(E.ev_end);
  if (E.stream && E.own_stream) cudaStreamDestroy(E.stream);
  delete c;
}

int kmcm_model_info(const kmcm_ctx* c, kmc_model_info_t* out) {
  if (!out) return KMC_E_BADARG;
  memset(out, 0, sizeof(*out));
  out->words = W;
  out->state_bits = M::STATE_BITS;
  out->num_actions = M::NUM_ACTIONS;
  out->num_invariants = M::NUM_INVARIANTS;
  out->num_init = M::NUM_INIT;
#ifdef KMC_HAS_DEVICE_INIT
  out->init_candidates = M::INIT_CANDIDATES;
#endif
  out->max_fanout = M::MAX_FANOUT;
  out->check_deadlock = M::CHECK_DEADLOCK;
  out->exact = (EXACT_SET || (c && E.exact)) ? 1 : 0;
  strncpy(out->name, KMC_MODEL_NAME, sizeof(out->name) - 1);
  strncpy(out->digest, KMC_MODEL_DIGEST, sizeof(out->digest) - 1);
  return KMC_OK;
}

int kmcm_run(kmcm_ctx* c) {
  if (!c) return KMC_E_BADARG;
  if (!c->ranks.empty()) return multi_run(c);
  return engine_run(E);
}

int kmcm_stats(const kmcm_ctx* c, kmc_stats_t* out) {
  if (!c || !out) return KMC_E_BADARG;
  std::lock_guard<std::mutex> g(E.mu);
  *out = E.stats;
  return KMC_OK;
}

int kmcm_level_widths(const kmcm_ctx* c, uint64_t* out, size_t cap, size_t* n) {
  if (!c || !n) return KMC_E_BADARG;
  std::lock_guard<std::mutex> g(E.mu);
  *n = E.widths.size();
  for (size_t i = 0; i < E.widths.size() && i < cap; ++i) out[i] = E.widths[i];
  return KMC_OK;
}

// generated per action = the per-site counts summed by the site's action
static std::vector<uint64_t> action_generated(const Engine& e) {
  std::vector<uint64_t> a(M::NUM_ACTIONS, 0);
  for (int i = 0; i < M::NUM_SITES; ++i)
    if (M::SITE_ACTION[i] >= 0 && M::SITE_ACTION[i] < M::NUM_ACTIONS) a[M::SITE_ACTION[i]] += e.site_generated[i];
  return a;
}

int kmcm_action_counts(const kmcm_ctx* c, uint64_t* out, size_t cap, size_t* n) {
  if (!c || !n || (!out && cap)) return KMC_E_BADARG;
  std::lock_guard<std::mutex> g(E.mu);
  const std::vector<uint64_t> a = action_generated(E);
  *n = a.size();
  for (size_t i = 0; i < a.size() && i < cap; ++i) out[i] = a[i];
  return KMC_OK;
}

int kmcm_coverage(const kmcm_ctx* c, uint64_t* action_gen, uint64_t* action_dist, size_t action_cap, uint64_t* site_gen,
                  size_t site_cap, size_t* n_actions, size_t* n_sites, int32_t* complete) {
  if (!c || !n_actions || !n_sites || !complete) return KMC_E_BADARG;
  if ((action_cap && (!action_gen || !action_dist)) || (site_cap && !site_gen)) return KMC_E_BADARG;
  std::lock_guard<std::mutex> g(E.mu);
  const std::vector<uint64_t> a = action_generated(E);
  *n_actions = a.size();
  *n_sites = E.site_generated.size();
  *complete = E.coverage_complete ? 1 : 0;
  for (size_t i = 0; i < a.size() && i < action_cap; ++i) {
    action_gen[i] = a[i];
    action_dist[i] = E.action_distinct[i];
  }
  for (size_t i = 0; i < E.site_generated.size() && i < site_cap; ++i) site_gen[i] = E.site_generated[i];
  return KMC_OK;
}

int kmcm_violation(const kmcm_ctx* c, kmc_violation_t* out) {
  if (!c || !out) return KMC_E_BADARG;
  if (!E.ran && E.level == 0) return KMC_E_STATE;
  const Counterexample& x = E.viol;
  memset(out, 0, sizeof(*out));
  out->kind = x.words.empty() ? KMC_RESULT_OK : x.inv < 0 ? KMC_RESULT_DEADLOCK : KMC_RESULT_INVARIANT;
  out->invariant = x.inv;
  out->level = x.level;
  out->trace_len = x.trace.size();
  out->fingerprint = x.fp;
  return KMC_OK;
}

static int trace_state(const Counterexample& x, uint32_t i, uint64_t* buf, size_t cap_words, uint32_t* action_id) {
  if (i >= x.trace.size() || cap_words < (size_t)W) return KMC_E_BADARG;
  memcpy(buf, x.trace[i].data(), W * 8);
  if (action_id) *action_id = x.actions[i];
  return KMC_OK;
}

int kmcm_trace_state(const kmcm_ctx* c, uint32_t i, uint64_t* buf, size_t cap_words, uint32_t* action_id) {
  if (!c || !buf) return KMC_E_BADARG;
  return trace_state(E.viol, i, buf, cap_words, action_id);
}

// the offending state of this rank (before any cross-rank trace walk): packed words + parent/action word
int kmcm_violation_record(const kmcm_ctx* c, uint64_t* words, size_t cap_words, uint64_t* parent_meta) {
  if (!c || !words || !parent_meta || cap_words < (size_t)W) return KMC_E_BADARG;
  if (E.viol.words.empty()) return KMC_E_STATE;
  memcpy(words, E.viol.words.data(), W * 8);
  *parent_meta = E.viol.meta;
  return KMC_OK;
}

// the reports of a "continue" run, ordered by (level, invariant); the multi-process driver's ranks (world > 1 without
// "gpus") each see only their own violators and report nothing
static bool inv_reports_readable(const kmcm_ctx* c, int* rc) {
  *rc = !M::HAS_INVARIANT_MASK ? KMC_E_BADARG : (c->ranks.empty() && E.world > 1) || (!E.ran && E.level == 0) ? KMC_E_STATE : KMC_OK;
  return *rc == KMC_OK;
}
static std::vector<const Counterexample*> inv_reports_sorted(const Engine& e) {
  std::vector<const Counterexample*> v;
  for (const Counterexample& r : e.inv_reports) v.push_back(&r);
  std::sort(v.begin(), v.end(), [](const Counterexample* a, const Counterexample* b) {
    return a->level != b->level ? a->level < b->level : a->inv < b->inv;
  });
  return v;
}

int kmcm_invariant_reports(const kmcm_ctx* c, kmc_invariant_report_t* out, size_t cap, size_t* n, int32_t* complete) {
  if (!c || !n || !complete || (!out && cap)) return KMC_E_BADARG;
  int rc;
  if (!inv_reports_readable(c, &rc)) return rc;
  std::lock_guard<std::mutex> g(E.mu);
  const std::vector<const Counterexample*> v = inv_reports_sorted(E);
  *n = v.size();
  *complete = E.inv_complete ? 1 : 0;
  for (size_t k = 0; k < v.size() && k < cap; ++k) {
    kmc_invariant_report_t& o = out[k];
    memset(&o, 0, sizeof(o));
    o.invariant = v[k]->inv;
    o.level = v[k]->level;
    o.violators_first_level = v[k]->first_count;
    o.violators = E.inv_count[v[k]->inv];
    o.trace_len = v[k]->trace.size();
    o.fingerprint = v[k]->fp;
  }
  return KMC_OK;
}

int kmcm_invariant_trace_state(const kmcm_ctx* c, int32_t invariant, uint32_t i, uint64_t* buf, size_t cap_words,
                               uint32_t* action_id) {
  if (!c || !buf || cap_words < (size_t)W) return KMC_E_BADARG;
  int rc;
  if (!inv_reports_readable(c, &rc)) return rc;
  std::lock_guard<std::mutex> g(E.mu);
  for (const Counterexample& r : E.inv_reports)
    if (r.inv == invariant) return trace_state(r, i, buf, cap_words, action_id);
  return KMC_E_BADARG;
}

// states and / or parent words [first, first + count) by global index
static int copy_store(const kmcm_ctx* c_, uint64_t first, uint64_t count, uint64_t* states, uint64_t* parents) {
  kmcm_ctx* c = const_cast<kmcm_ctx*>(c_);
  if (!c || !(states || parents)) return KMC_E_BADARG;
  if (!c->ranks.empty()) return KMC_E_STATE;      // per-rank stores: address a rank's own context
  CK(cudaSetDevice(E.device));
  if (!E.spill && first + count > E.max_states) return KMC_E_BADARG;
  return read_range(E, first, count, states, parents);
}
int kmcm_copy_parents(const kmcm_ctx* c, uint64_t first, uint64_t count, uint64_t* buf) {
  return copy_store(c, first, count, nullptr, buf);
}
int kmcm_copy_states(const kmcm_ctx* c, uint64_t first, uint64_t count, uint64_t* buf) {
  return copy_store(c, first, count, buf, nullptr);
}

// kmc_edges and kmc_fingerprints read the store a kmc_run left on one GPU
static int stored_range(kmcm_ctx* c, uint64_t first, uint64_t count) {
  if (!c->ranks.empty() || E.world > 1) {
    E.last_error = "kmc_edges / kmc_fingerprints read the store of a one-GPU kmc_run: no \"gpus\" > 1, no world > 1";
    return KMC_E_BADARG;
  }
  if (!E.ran) return KMC_E_STATE;
  if (first + count < first || first + count > E.stats.distinct) {
    E.last_error = "kmc_edges / kmc_fingerprints: the range reaches past the stored states";
    return KMC_E_BADARG;
  }
  CK(cudaSetDevice(E.device));
  return KMC_OK;
}

int kmcm_edges(kmcm_ctx* c, uint64_t first, uint64_t count, kmc_edge_t* out, size_t cap, size_t* n) {
  if (!c || !n || (cap && !out)) return KMC_E_BADARG;
  if (int rc = stored_range(c, first, count)) return rc;
  return engine_edges(E, first, count, out, cap, n);
}

// host side: state_fp is a host function too, and a fingerprint per stored state is what a graph writer needs once
int kmcm_fingerprints(kmcm_ctx* c, uint64_t first, uint64_t count, uint64_t* out) {
  if (!c || (count && !out)) return KMC_E_BADARG;
  if (int rc = stored_range(c, first, count)) return rc;
  std::vector<uint64_t> buf;
  for (uint64_t g = first, end = first + count, m; g < end; g += m) {
    m = std::min<uint64_t>(end - g, 1 << 20);
    buf.resize(m * W);
    if (int rc = read_range(E, g, m, buf.data(), nullptr)) return rc;
    for (uint64_t i = 0; i < m; ++i) {
      State s;
      memcpy(s.w, buf.data() + i * W, sizeof(s.w));
      out[g - first + i] = state_fp(s);
    }
  }
  return KMC_OK;
}

const char* kmcm_strerror(const kmcm_ctx* c, int code) {
  switch (code) {
    case KMC_OK: return "ok";
    case KMC_E_BADARG: return (c && !E.last_error.empty()) ? E.last_error.c_str() : "bad argument";
    case KMC_E_CUDA: return (c && !E.last_error.empty()) ? E.last_error.c_str() : "CUDA error";
    case KMC_E_OOM: return "out of device memory";
    case KMC_E_TABLE_FULL: return "fingerprint set is full (raise table_log2)";
    case KMC_E_STORE_FULL: return "state store is full (raise max_states)";
    case KMC_E_LAYOUT_OVERFLOW: return "a successor value does not fit the packed state layout";
    case KMC_E_MODEL: return "cannot load the lowered model library";
    case KMC_E_STATE: return "call sequence error";
    case KMC_E_NO_GPU: return "no CUDA device visible; this library has no CPU fallback";
    case KMC_E_CAND_FULL: return "candidate buffer overflow (raise cand_bytes or fanout_bound)";
    case KMC_E_PEER_TIMEOUT: return "a peer rank did not arrive at a device-side synchronisation point within 30 s";
    case KMC_E_SET_TIMEOUT: return "exact_set: a claimed slot of the set was not published in time";
    default: return "unknown error";
  }
}

// ---- fingerprint set alone ---------------------------------------------------------------
// (not with set_spill: the keys in host memory are not consulted, so put() could call a known fingerprint new)
static int fpset_call(kmcm_ctx* c, const uint64_t* fps, size_t n, uint8_t* out, int insert) {
  if (c && E.exact) E.last_error = EXACT_SET_NO_FPSET;
  if (!c || E.set_spill || E.exact || (!fps && n) || (!out && n)) return KMC_E_BADARG;
  if (n == 0) return KMC_OK;
  CK(cudaSetDevice(E.device));
  uint64_t* d_fps = nullptr;
  uint8_t* d_out = nullptr;
  CK(cudaMalloc(&d_fps, n * 8));
  CK(cudaMalloc(&d_out, n));
  CK(cudaMemcpyAsync(d_fps, fps, n * 8, cudaMemcpyHostToDevice, E.stream));
  k_fpset_put<<<grid_for(E, n, 256, 8), 256, 0, E.stream>>>(E.table, E.table_slots / BUCKET_SLOTS - 1, d_fps, n, d_out, E.ctr, insert);
  CK(cudaMemcpyAsync(out, d_out, n, cudaMemcpyDeviceToHost, E.stream));
  CK(cudaStreamSynchronize(E.stream));
  cudaFree(d_fps);
  cudaFree(d_out);
  unsigned long long f = 0;
  CK(cudaMemcpy(&f, &E.ctr->fail, 8, cudaMemcpyDeviceToHost));
  return fail_to_error(f);
}
int kmcm_fpset_put(kmcm_ctx* c, const uint64_t* fps, size_t n, uint8_t* out_seen) { return fpset_call(c, fps, n, out_seen, 1); }
int kmcm_fpset_contains(kmcm_ctx* c, const uint64_t* fps, size_t n, uint8_t* out) { return fpset_call(c, fps, n, out, 0); }
int kmcm_fpset_size(const kmcm_ctx* c_, uint64_t* out) {
  kmcm_ctx* c = const_cast<kmcm_ctx*>(c_);
  if (c && E.exact) E.last_error = EXACT_SET_NO_FPSET;
  if (!c || E.set_spill || E.exact || !out) return KMC_E_BADARG;
  unsigned long long t = 0;
  CK(cudaSetDevice(E.device));
  CK(cudaMemcpy(&t, &E.ctr->store_tail, 8, cudaMemcpyDeviceToHost));
  *out = t;
  return KMC_OK;
}

// ---- sharded (multi-rank) building blocks -------------------------------------------------
// None of them runs on a set_spill context: they insert without the filter that keeps the store free of states whose
// keys are in host memory.
int kmcm_shard_begin(kmcm_ctx* c) {
  if (c && (E.set_spill || shard_refused(E))) return KMC_E_BADARG;
  if (!c) return KMC_E_BADARG;
  int rc = engine_reset(E);
  if (rc) return rc;
  E.inbox_buf = 0;
  E.ran = false;
  CK(cudaEventRecord(E.ev_begin, E.stream));
  return KMC_OK;
}

int kmcm_shard_buffers(kmcm_ctx* c, kmc_shard_buffers_t* out) {
  if (c && (E.set_spill || shard_refused(E))) return KMC_E_BADARG;
  if (!c || !out) return KMC_E_BADARG;
  out->cand = E.cand;
  out->region_rows = E.region_rows;
  out->cand_counts = (uint64_t*)E.ctr->cand_count;
  out->recv = E.world > 1 ? E.recv : E.cand;
  out->recv_rows_cap = E.world > 1 ? E.recv_rows : E.region_rows;
  out->row_words = ROW;
  return KMC_OK;
}

int kmcm_shard_seed_init(kmcm_ctx* c) {
  if (c && (E.set_spill || shard_refused(E))) return KMC_E_BADARG;
  if (!c) return KMC_E_BADARG;
  return seed_init(E);
}

int kmcm_shard_expand(kmcm_ctx* c, uint64_t first, uint64_t count) {
  if (c && (E.set_spill || shard_refused(E))) return KMC_E_BADARG;
  if (!c) return KMC_E_BADARG;
  if (count > E.chunk_states) {
    E.last_error = "expand chunk larger than chunk_states";
    return KMC_E_BADARG;
  }
  if (count == 0) return KMC_OK;
  return launch_expand(E, first, count);
}

int kmcm_shard_counts(kmcm_ctx* c, uint64_t* host_counts) {
  if (c && (E.set_spill || shard_refused(E))) return KMC_E_BADARG;
  if (!c || !host_counts) return KMC_E_BADARG;
  unsigned long long tmp[MAX_WORLD];
  CK(cudaMemcpyAsync(tmp, E.ctr->cand_count, sizeof(tmp), cudaMemcpyDeviceToHost, E.stream));
  CK(cudaStreamSynchronize(E.stream));
  for (uint32_t d = 0; d < E.world; ++d) host_counts[d] = tmp[d];
  return KMC_OK;
}

int kmcm_shard_reset_cand(kmcm_ctx* c) {
  if (c && (E.set_spill || shard_refused(E))) return KMC_E_BADARG;
  if (!c) return KMC_E_BADARG;
  return reset_cand(E);
}

int kmcm_shard_insert(kmcm_ctx* c, const uint64_t* rows_dev, uint64_t rows, uint64_t* new_tail) {
  if (c && (E.set_spill || shard_refused(E))) return KMC_E_BADARG;
  if (!c) return KMC_E_BADARG;
  if (rows) {
    int rc = launch_insert(E, rows_dev, nullptr, rows, rows);
    if (rc) return rc;
  }
  if (new_tail) {
    DevCounters h;
    int rc = read_counters(E, &h);
    if (rc) return rc;
    *new_tail = h.store_tail;
    return fail_to_error(h.fail);
  }
  return KMC_OK;
}

int kmcm_shard_level_done(kmcm_ctx* c, uint64_t* level_first, uint64_t* level_count) {
  if (c && (E.set_spill || shard_refused(E))) return KMC_E_BADARG;
  if (!c) return KMC_E_BADARG;
  DevCounters h;
  int rc = end_level(E, std::max<uint64_t>(E.level_count * 2, 1024), true, h);
  if (rc) return rc;
  if (level_first) *level_first = E.level_first;
  if (level_count) *level_count = E.level_count;
  return fail_to_error(h.fail);
}

// ---- fused exchange over peer memory ---------------------------------------------------------
int kmcm_shard_ipc_handle(kmcm_ctx* c, void* out64) {
  if (c && (E.set_spill || shard_refused(E))) return KMC_E_BADARG;
  if (!c || !out64 || !E.inbox) return KMC_E_BADARG;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaIpcMemHandle_t h;
  CK(cudaSetDevice(E.device));
  CK(cudaIpcGetMemHandle(&h, E.inbox_alloc));
  memcpy(out64, &h, 64);
  return KMC_OK;
}

int kmcm_shard_open_peers(kmcm_ctx* c, const void* handles, uint32_t world) {
  if (c && (E.set_spill || shard_refused(E))) return KMC_E_BADARG;
  if (!c || !handles || world != E.world || !E.inbox) return KMC_E_BADARG;
  CK(cudaSetDevice(E.device));
  for (uint32_t r = 0; r < world; ++r) {
    if (r == E.rank) {
      E.peer_inbox[r] = E.inbox;
      continue;
    }
    cudaIpcMemHandle_t h;
    memcpy(&h, (const char*)handles + 64 * r, 64);
    void* ptr = nullptr;
    CK(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
    E.peer_inbox[r] = (uint64_t*)ptr + SYNC_WORDS;
  }
  E.peers_open = true;
  return KMC_OK;
}

// expand a frontier chunk, storing every successor row directly into its owner's inbox, then
// publish the per-owner row counts into the owners' inbox headers (both on the engine stream)
int kmcm_shard_expand_p2p(kmcm_ctx* c, uint64_t first, uint64_t count) {
  if (c && (E.set_spill || shard_refused(E))) return KMC_E_BADARG;
  if (!c || !E.peers_open) return KMC_E_STATE;
  if (count > E.chunk_states) return KMC_E_BADARG;
  int rc = reset_cand(E);
  if (rc) return rc;
  if ((rc = launch_expand(E, first, count, true))) return rc;
  Params p = E.params();
  p.p2p = 1;
  {
    TimedLaunch t(E, 2);
    k_publish_counts<<<1, 32, 0, E.stream>>>(p, 0);
  }
  CK(cudaGetLastError());
  return KMC_OK;
}

// seed: the initial states go through the same inbox path (rank 0 contributes them)
static int seed_p2p(kmcm_ctx* c, bool publish) {
  if (c && (E.set_spill || shard_refused(E))) return KMC_E_BADARG;
  if (!c || !E.peers_open) return KMC_E_STATE;
  CK(cudaSetDevice(E.device));
  unsigned long long counts[MAX_WORLD] = {0};
  if (E.rank == 0) {
    for (int i = 0; i < M::NUM_INIT; ++i) {
      State s;
      memcpy(s.w, M::INIT_STATES[i], sizeof(s.w));
      uint32_t d = owner_of(state_fp(s), E.world);
      uint64_t row[ROW];
      for (int k = 0; k < W; ++k) row[k] = s.w[k];
      row[W] = NO_PARENT;
      uint64_t* dst = E.peer_inbox[d] + (uint64_t)E.inbox_buf * E.inbox_stride + INBOX_HEADER +
                      ((uint64_t)E.rank * E.region_rows + counts[d]) * ROW;
      CK(cudaMemcpyAsync(dst, row, sizeof(row), cudaMemcpyHostToDevice, E.stream));
      CK(cudaStreamSynchronize(E.stream));
      counts[d]++;
    }
    unsigned long long gen = M::NUM_INIT;
    CK(cudaMemcpyAsync(&E.ctr->generated, &gen, sizeof(gen), cudaMemcpyHostToDevice, E.stream));
  }
  CK(cudaMemcpyAsync(E.ctr, counts, sizeof(counts), cudaMemcpyHostToDevice, E.stream));
  if (publish) {
    Params p = E.params();
    p.p2p = 1;
    k_publish_counts<<<1, 32, 0, E.stream>>>(p, 0);
    CK(cudaGetLastError());
  }
  CK(cudaStreamSynchronize(E.stream));
  return KMC_OK;
}
int kmcm_shard_seed_p2p(kmcm_ctx* c) { return seed_p2p(c, true); }

// insert everything the peers stored into the current inbox buffer, then switch buffers.
// The caller must have put a cross-rank barrier on the stream between expand_p2p and this call.
int kmcm_shard_insert_p2p(kmcm_ctx* c) {
  if (c && (E.set_spill || shard_refused(E))) return KMC_E_BADARG;
  if (!c || !E.peers_open) return KMC_E_STATE;
  Params p = E.params();
  {
    TimedLaunch t(E, 1);
    k_insert_inbox<<<E.sms * 8, 256, 0, E.stream>>>(p);
  }
  CK(cudaGetLastError());
  E.inbox_buf ^= 1;
  return KMC_OK;
}

// One expand -> exchange -> insert round with device-side cross-rank synchronisation (no NCCL, no host wait):
//   wait until every destination has consumed the buffer this round reuses (done >= round - 2)
//   expand (or, seed != 0, store the initial states) straight into the owners' inboxes; publish counts + ready
//   wait until every source is ready for this round; insert from the own inbox; publish done
// Every rank must call it the same number of times (count = 0 on ranks without work).
int kmcm_shard_round_p2p(kmcm_ctx* c, uint64_t first, uint64_t count, int seed) {
  if (c && (E.set_spill || shard_refused(E))) return KMC_E_BADARG;
  if (!c || !E.peers_open) return KMC_E_STATE;
  if (count > E.chunk_states) return KMC_E_BADARG;
  CK(cudaSetDevice(E.device));
  const uint64_t round = ++E.round;
  E.inbox_buf = (uint32_t)(round & 1);
  int rc;
  if (round > 2) k_wait_flags<<<1, 32, 0, E.stream>>>(E.inbox_alloc + SYNC_DONE, E.world, round - 2, E.ctr);
  if (seed) {
    if ((rc = seed_p2p(c, false))) return rc;
  } else {
    if ((rc = reset_cand(E))) return rc;
    if ((rc = launch_expand(E, first, count, true))) return rc;
  }
  Params p = E.params();
  p.p2p = 1;
  k_publish_counts<<<1, 32, 0, E.stream>>>(p, round);
  k_wait_flags<<<1, 32, 0, E.stream>>>(E.inbox_alloc + SYNC_READY, E.world, round, E.ctr);
  {
    TimedLaunch t(E, 1);
    k_insert_inbox<<<E.sms * 8, 256, 0, E.stream>>>(p);
  }
  k_publish_done<<<1, 32, 0, E.stream>>>(p, round);
  CK(cudaGetLastError());
  return KMC_OK;
}

// Level end on all ranks at once: invariants on this rank's new states, publish the summary to every board, wait
// for all summaries, copy the board to pinned host memory, ONE stream synchronisation.  board_out receives
// world x 8 words: {level id, new states, violations, store tail, generated, fail, deadlocks, -} per rank.
int kmcm_shard_level_sync(kmcm_ctx* c, uint64_t* board_out) {
  if (c && (E.set_spill || shard_refused(E))) return KMC_E_BADARG;
  if (!c || !E.peers_open || !board_out) return KMC_E_STATE;
  CK(cudaSetDevice(E.device));
  int rc = launch_invariants(E, E.level_first + E.level_count, std::max<uint64_t>(E.level_count * 2, 1024));
  if (rc) return rc;
  const uint64_t level_id = ++E.level_id;
  Params p = E.params();
  k_publish_level<<<1, 32, 0, E.stream>>>(p, level_id, E.level_first + E.level_count);
  uint64_t* dev_view = nullptr;
  CK(cudaHostGetDevicePointer((void**)&dev_view, E.board_host, 0));
  k_gather_level<<<1, 32, 0, E.stream>>>(p, level_id, dev_view);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(E.stream));
  memcpy(board_out, E.board_host, (size_t)E.world * BOARD_WORDS * 8);
  const uint64_t* mine = E.board_host + (size_t)E.rank * BOARD_WORDS;
  const uint64_t prev_end = E.level_first + E.level_count;
  E.level_first = prev_end;
  E.level_count = mine[1];
  E.level++;
  {
    std::lock_guard<std::mutex> g(E.mu);
    E.stats.distinct = mine[3];
    E.stats.generated = mine[4];
    E.stats.deadlocks = mine[6];
    E.stats.table_slots = E.table_slots;
    E.stats.slot_bytes = E.slot_bytes();
    E.stats.max_states = E.max_states;
    if (E.level_count) E.widths.push_back(E.level_count);
    E.stats.levels = E.stats.depth = E.widths.size();
  }
  if (mine[2] && E.viol.words.empty()) {
    DevCounters h;
    if ((rc = read_counters(E, &h))) return rc;
    build_trace(E, h, E.level - 1);
  }
  // the invariants first violated at this level on any rank stop being pending on every rank
  uint64_t fresh = 0;
  for (uint32_t r = 0; r < E.world; ++r) fresh |= E.board_host[(size_t)r * BOARD_WORDS + 7];
  if (INV_REPORT && E.cont) {
    DevCounters h;
    if ((rc = read_counters(E, &h)) || (rc = collect_invariants(E, h, E.level, fresh, false))) return rc;
  }
  return fail_to_error(mine[5]);
}

// same-process peers (one context per GPU in one process): direct pointers instead of CUDA IPC handles.
// inboxes[r] = the value kmcm_shard_inbox_ptr returned for rank r's context.
int kmcm_shard_inbox_ptr(kmcm_ctx* c, void** out) {
  if (c && (E.set_spill || shard_refused(E))) return KMC_E_BADARG;
  if (!c || !out || !E.inbox_alloc) return KMC_E_BADARG;
  *out = E.inbox_alloc;
  return KMC_OK;
}
int kmcm_shard_open_peers_direct(kmcm_ctx* c, void* const* inboxes, const int* devices, uint32_t world) {
  if (c && (E.set_spill || shard_refused(E))) return KMC_E_BADARG;
  if (!c || !inboxes || !devices || world != E.world || !E.inbox_alloc) return KMC_E_BADARG;
  CK(cudaSetDevice(E.device));
  for (uint32_t r = 0; r < world; ++r) {
    if (r != E.rank) {
      cudaError_t e = cudaDeviceEnablePeerAccess(devices[r], 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) {
        E.last_error = std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e);
        return KMC_E_CUDA;
      }
      cudaGetLastError();
    }
    E.peer_inbox[r] = (uint64_t*)inboxes[r] + SYNC_WORDS;
  }
  E.peers_open = true;
  E.peers_direct = true;
  return KMC_OK;
}

int kmcm_shard_sync(kmcm_ctx* c) {
  if (c && (E.set_spill || shard_refused(E))) return KMC_E_BADARG;
  if (!c) return KMC_E_BADARG;
  CK(cudaEventRecord(E.ev_end, E.stream));
  DevCounters h;
  int rc = read_counters(E, &h);              // synchronises the stream
  if (rc) return rc;
  float total_ms = 0;
  cudaEventElapsedTime(&total_ms, E.ev_begin, E.ev_end);
  std::lock_guard<std::mutex> g(E.mu);
  publish(E, h, false);
  E.stats.gpu_ms_total = total_ms;
  if (E.timing) accumulate_timing(E, E.stats);
  return KMC_OK;
}

}  // extern "C"
#undef E

// ----------------------------------------------------------------------------------------
// N GPUs behind one context (kmc_create option "gpus": N): tlc2 -workers N, or any C / JNI caller.
// The ranks are ordinary sub-contexts driven through the same kmcm_shard_* entry points the multi-process
// driver uses; they see each other's inboxes through direct peer pointers.  Every rank thread reads the same
// level board, so all of them take the same decisions without any host-side barrier.
// ----------------------------------------------------------------------------------------
static int multi_create(kmcm_ctx* c, const char* options_json, int gpus) {
  Engine& A = c->e;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    A.last_error = "no CUDA device visible; this library has no CPU fallback";
    return KMC_E_NO_GPU;
  }
  if (gpus > ndev || gpus > MAX_WORLD) {
    A.last_error = "option gpus exceeds the visible devices";
    return KMC_E_BADARG;
  }
  std::string base = options_json ? options_json : "{}";
  size_t close = base.rfind('}');
  if (close == std::string::npos) return KMC_E_BADARG;
  const int dev0 = A.device;
  for (int r = 0; r < gpus; ++r) {
    // the sub-context's own keys go first: json_find takes the first occurrence of a key
    std::string opt = "{\"device\": " + std::to_string(dev0 + r) + ", \"rank\": " + std::to_string(r) + ", \"world\": " +
                      std::to_string(gpus) + ", \"gpus\": 0, " + base.substr(base.find('{') + 1);
    kmcm_ctx* sub = nullptr;
    int rc = kmcm_create(opt.c_str(), &sub);
    if (sub) c->ranks.push_back(sub);
    if (rc) {
      A.last_error = sub ? sub->e.last_error : "cannot create a rank context";
      return rc;
    }
  }
  void* inboxes[MAX_WORLD] = {};
  int devices[MAX_WORLD] = {};
  for (int r = 0; r < gpus; ++r) {
    kmcm_shard_inbox_ptr(c->ranks[r], &inboxes[r]);
    devices[r] = dev0 + r;
  }
  for (int r = 0; r < gpus; ++r) {
    int rc = kmcm_shard_open_peers_direct(c->ranks[r], inboxes, devices, (uint32_t)gpus);
    if (rc) {
      A.last_error = c->ranks[r]->e.last_error;
      return rc;
    }
  }
  A.world = (uint32_t)gpus;
  return KMC_OK;
}

struct RankOutcome {
  int rc = KMC_OK;
  std::vector<uint64_t> levels;
  bool stopped = false;
  uint64_t board[MAX_WORLD * BOARD_WORDS] = {};
};

static void rank_loop(kmcm_ctx* sub, bool cont, uint64_t stop_after, RankOutcome* out) {
  Engine& R = sub->e;
  const uint32_t world = R.world, rank = R.rank;
  uint64_t* board = out->board;
  auto fail = [&](int rc) { out->rc = rc; };
  int rc;
  if ((rc = kmcm_shard_begin(sub))) return fail(rc);
  if ((rc = kmcm_shard_round_p2p(sub, 0, 0, 1))) return fail(rc);
  rc = kmcm_shard_level_sync(sub, board);
  uint64_t first = 0;
  for (;;) {
    // a failure flag of ANY rank ends the run on every rank (they all read the same board)
    int err = rc;
    uint64_t total = 0, viol = 0, max_new = 0, distinct = 0;
    for (uint32_t r = 0; r < world; ++r) {
      const uint64_t* b = board + r * BOARD_WORDS;
      total += b[1];
      viol += b[2];
      distinct += b[3];
      max_new = std::max(max_new, b[1]);
      if (!err && b[5]) err = fail_to_error(b[5]);
    }
    if (err) return fail(err);
    if (viol && !cont) { out->stopped = true; break; }
    if (total == 0) break;
    out->levels.push_back(total);
    if (stop_after && distinct >= stop_after) { out->stopped = true; break; }
    const uint64_t count = board[rank * BOARD_WORDS + 1];
    const uint64_t n_chunks = (max_new + R.chunk_states - 1) / R.chunk_states;
    for (uint64_t ci = 0; ci < n_chunks; ++ci) {
      const uint64_t off = ci * R.chunk_states;
      const uint64_t n = off < count ? std::min<uint64_t>(R.chunk_states, count - off) : 0;
      if ((rc = kmcm_shard_round_p2p(sub, first + off, n, 0))) return fail(rc);
    }
    first += count;
    rc = kmcm_shard_level_sync(sub, board);
  }
  if ((rc = kmcm_shard_sync(sub))) return fail(rc);
}

static int multi_run(kmcm_ctx* c) {
  Engine& A = c->e;
  const size_t n = c->ranks.size();
  auto t0 = std::chrono::steady_clock::now();
  std::vector<RankOutcome> out(n);
  std::vector<std::thread> th;
  for (size_t r = 0; r < n; ++r) th.emplace_back(rank_loop, c->ranks[r], A.cont, A.stop_after_states, &out[r]);
  for (auto& t : th) t.join();
  auto t1 = std::chrono::steady_clock::now();
  int rc = KMC_OK;
  for (size_t r = 0; r < n; ++r)
    if (out[r].rc && !rc) {
      rc = out[r].rc;
      A.last_error = c->ranks[r]->e.last_error;
    }
  std::lock_guard<std::mutex> g(A.mu);
  kmc_stats_t& st = A.stats;
  memset(&st, 0, sizeof(st));
  A.widths = out[0].levels;
  for (size_t r = 0; r < n; ++r) {
    const kmc_stats_t& s = c->ranks[r]->e.stats;
    st.distinct += s.distinct;
    st.generated += s.generated;
    st.deadlocks += s.deadlocks;
    st.out_of_model += s.out_of_model;
    st.probes += s.probes;
    st.table_slots += s.table_slots;
    st.max_states += s.max_states;
    st.launches_expand += s.launches_expand;
    st.launches_insert += s.launches_insert;
    st.launches_other += s.launches_other;
    st.gpu_ms_total = std::max(st.gpu_ms_total, s.gpu_ms_total);
    st.gpu_ms_expand = std::max(st.gpu_ms_expand, s.gpu_ms_expand);
    st.gpu_ms_insert = std::max(st.gpu_ms_insert, s.gpu_ms_insert);
    st.gpu_ms_invariant = std::max(st.gpu_ms_invariant, s.gpu_ms_invariant);
    st.slot_bytes = s.slot_bytes;
  }
  st.depth = st.levels = A.widths.size();
  st.complete = (!rc && !out[0].stopped) ? 1 : 0;
  std::fill(A.site_generated.begin(), A.site_generated.end(), 0);
  std::fill(A.action_distinct.begin(), A.action_distinct.end(), 0);
  for (size_t r = 0; r < n; ++r) {
    const Engine& R = c->ranks[r]->e;
    std::lock_guard<std::mutex> gr(R.mu);
    for (size_t i = 0; i < A.site_generated.size(); ++i) A.site_generated[i] += R.site_generated[i];
    for (size_t i = 0; i < A.action_distinct.size(); ++i) A.action_distinct[i] += R.action_distinct[i];
  }
  if (out[0].stopped && !rc) {
    // the states of the last level were inserted but not expanded: they are the queue
    for (size_t r = 0; r < n; ++r) st.queue += out[0].board[r * BOARD_WORDS + 1];
  }
  st.wall_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
  // The ranks' picks merged in violator order (reports: the earliest level first; the ranks' violators of an invariant
  // at that level summed), then walked from store to store.  Every rank reports the same invariants at the same
  // levels (they share the board).  No tie between ranks needs breaking: a violator's row is written on the rank that
  // owns its fingerprint (owner_of(state_fp(s))), or on the rank that expands it, which for a deadlock is its owner
  // too, so no two ranks hold candidates with the same fingerprint.
  Counterexample viol;
  A.inv_reports.clear();
  A.inv_complete = true;
  std::fill(A.inv_count.begin(), A.inv_count.end(), 0);
  std::vector<Engine*> ranks;
  for (size_t r = 0; r < n; ++r) {
    Engine& R = c->ranks[r]->e;
    ranks.push_back(&R);
    if (better(R.viol, viol)) viol = R.viol;
    A.inv_complete = A.inv_complete && R.inv_complete;
    for (size_t i = 0; i < A.inv_count.size(); ++i) A.inv_count[i] += R.inv_count[i];
    for (const Counterexample& x : R.inv_reports) {
      auto y = std::find_if(A.inv_reports.begin(), A.inv_reports.end(), [&](const Counterexample& a) { return a.inv == x.inv; });
      if (y == A.inv_reports.end()) {
        A.inv_reports.push_back(x);
      } else if (x.level < y->level) {
        *y = x;
      } else if (x.level == y->level) {
        const uint64_t count = y->first_count + x.first_count;
        if (better(x, *y)) *y = x;
        y->first_count = count;
      }
    }
  }
  A.viol = rc ? Counterexample() : std::move(viol);
  if (!rc && !A.viol.words.empty()) rc = walk_trace(A, ranks, A.viol);
  for (Counterexample& x : A.inv_reports)
    if (!rc && !x.words.empty()) rc = walk_trace(A, ranks, x);
  A.ran = true;
  return rc;
}

