/* kspecmc.h -- C ABI of the H100-native explicit-state model checker (libkspecmc.so).
 *
 * This is the drop-in boundary for the BFS frontier-expansion path of a TLC run
 * (SURVEY.md section 8b).  The reference (hachikuji/kafka-specification) has no FFI of its
 * own: it is input for TLC, so each entry point cites the TLC seam it replaces.  TLC is not
 * in the reference tree (third-party tla2tools.jar, no pinned version); class and method
 * names below are TLC's published ones and the spec-side anchors are the reference files
 * whose Init/Next/invariants the lowered model evaluates (e.g. Kip320.tla:150-159,
 * KafkaReplication.tla:101-120,320-345).
 *
 *   kmc_create          tlc2.TLC.handleParameters + tlc2.tool.ModelChecker.<init>
 *                       (loads the lowered model = Tool/SpecProcessor output; allocates the
 *                        FPSet, the StateQueue and the trace store in HBM)
 *   kmc_run             tlc2.tool.ModelChecker.doInit + runTLC: N x tlc2.tool.Worker.run --
 *                       the hot loop: StateQueue.sDequeue -> Tool.getNextStates ->
 *                       TLCState.fingerPrint -> FPSet.put -> Tool.isValid -> sEnqueue
 *                       Level 1 comes from the lowered model's table of initial states or, for a
 *                       model lowered with the device form of Init (model.json init.device), from
 *                       k_init, which decodes every candidate assignment of Init's generators on the
 *                       GPU and keeps those that satisfy the rest of Init (one GPU only: "gpus" > 1,
 *                       world > 1 and the kmc_shard_* calls give KMC_E_BADARG)
 *   kmc_stats           ModelChecker.reportSuccess / printSummary ("N states generated,
 *                       M distinct states found, Q states left on queue", depth); init_generated
 *                       and init_candidates count TLC's doInit ("N distinct states generated")
 *   kmc_violation       ModelChecker.doNext's invariant/deadlock failure report
 *   kmc_invariant_*     the same per invariant under -continue (first level, violators, counterexample)
 *   kmc_coverage        ModelChecker's coverage report (TLC -coverage: "distinct:generated" per action, at the
 *                       action level of TLC >= 1.7), from counters the kernels keep on every run
 *   kmc_trace_*         tlc2.tool.TLCTrace.getTrace / printTrace (error trace by parent links)
 *   kmc_fpset_*         tlc2.tool.fp.FPSet.put / contains / size (the set alone, for callers
 *                       that keep TLC's own Worker loop)
 *   kmc_shard_*         tlc2.tool.distributed.fp (fingerprint-sharded FPSet servers): the
 *                       per-level building blocks a multi-rank driver exchanges between
 *
 * Conventions: plain C, no C++ types, no exceptions across the boundary.  Every function
 * returns 0 (KMC_OK) or a negative KMC_E_* code; kmc_strerror gives the text.  Caller
 * allocates all output structs.  One kmc_ctx drives one GPU; kmc_run is not re-entrant;
 * kmc_stats may be called from another thread while kmc_run is in flight.
 */
#ifndef KSPECMC_H
#define KSPECMC_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct kmc_ctx kmc_ctx;

enum {
  KMC_OK = 0,
  KMC_E_BADARG = -1,
  KMC_E_CUDA = -2,
  KMC_E_OOM = -3,
  KMC_E_TABLE_FULL = -4,      /* fingerprint set saturated (raise table_log2)            */
  KMC_E_STORE_FULL = -5,      /* more distinct states than max_states                    */
  KMC_E_LAYOUT_OVERFLOW = -6, /* a successor value does not fit the packed state layout  */
  KMC_E_MODEL = -7,           /* cannot load / mismatching lowered model library         */
  KMC_E_STATE = -8,           /* call sequence error (e.g. trace before run)             */
  KMC_E_NO_GPU = -9,          /* no CUDA device: there is deliberately no CPU fallback   */
  KMC_E_CAND_FULL = -10,      /* candidate buffer overflow (raise cand_bytes / fanout_bound) */
  KMC_E_PEER_TIMEOUT = -11,   /* multi-GPU: a peer rank never reached a device-side synchronisation point */
  KMC_E_SET_TIMEOUT = -12     /* "exact_set": a claimed slot of the set was not published within its bounded wait */
};

/* result kinds (kmc_violation_t.kind); a driver maps them to TLC's exit codes 0/12/11 */
enum { KMC_RESULT_OK = 0, KMC_RESULT_INVARIANT = 1, KMC_RESULT_DEADLOCK = 2 };

typedef struct {
  uint64_t distinct;        /* states in the fingerprint set (this rank)                  */
  uint64_t generated;       /* init states + every successor produced, duplicates included */
  uint64_t queue;           /* states left on the queue (0 after a complete run)          */
  uint64_t depth;           /* BFS levels, Init = level 1                                 */
  uint64_t deadlocks;       /* states without any successor                               */
  uint64_t out_of_model;    /* successors discarded by a CONSTRAINT                       */
  uint64_t probes;          /* hash-set buckets (32 B sectors) touched                    */
  uint64_t levels;          /* number of valid entries for kmc_level_widths               */
  double gpu_ms_total;      /* CUDA-event time of the whole level loop of the last run    */
  double gpu_ms_expand;     /* sum over expand-kernel launches                            */
  double gpu_ms_insert;     /* sum over insert-kernel (hash probe) launches               */
  uint64_t launches_expand;
  uint64_t launches_insert;
  uint64_t launches_other;
  double wall_ms;           /* host wall clock of the last kmc_run                        */
  uint64_t table_slots;     /* fingerprint-set capacity in slots (slot_bytes each)        */
  uint64_t max_states;      /* state-store capacity                                       */
  uint64_t complete;        /* 1 if the search ran to an empty queue                      */
  double gpu_ms_invariant;  /* sum over invariant-kernel launches (counted in launches_other) */
  uint64_t slot_bytes;      /* 8: 64-bit fingerprints (one-word states); 16: 128-bit keys (the state itself when it fits);
                               "exact_set" on a hashed model: 16 (one word), 32 (two or three words), 64 (four to seven) */
  uint64_t set_flushes;     /* "set_spill": times the table's keys moved to host memory                */
  uint64_t set_host_keys;   /* "set_spill": keys in host memory (each distinct state's key at most once) */
  uint64_t set_filtered;    /* "set_spill": appended states removed because their key was in host memory */
  double gpu_ms_set_spill;  /* "set_spill": CUDA-event time of the flushes and filters (part of gpu_ms_total) */
  uint64_t set_link_bytes;  /* "set_spill": key bytes the flushes (device to host) and filters (host to device) moved */
  uint64_t init_generated;  /* Init solutions, duplicates included (part of `generated`): NUM_INIT for a table model */
  uint64_t init_candidates; /* device Init: candidate assignments k_init decoded; 0 for a table model */
  double gpu_ms_init;       /* device Init: CUDA-event time of the k_init launches (part of gpu_ms_total) */
} kmc_stats_t;

typedef struct {
  int32_t kind;             /* KMC_RESULT_*                                               */
  int32_t invariant;        /* index into the cfg's INVARIANT list, -1 for deadlock       */
  uint64_t level;           /* BFS level of the offending state (Init = 1)                */
  uint64_t trace_len;       /* number of states in the error trace                        */
  uint64_t fingerprint;     /* 64-bit fingerprint of the offending state; under SYMMETRY that of
                               its orbit (the canonical form), whichever member was reached  */
} kmc_violation_t;

/* One violated invariant of a "continue" run (kmc_invariant_reports). */
typedef struct {
  int32_t invariant;              /* index into the cfg's INVARIANT list                              */
  uint64_t level;                 /* first BFS level with a checked state that violates it (Init = 1) */
  uint64_t violators_first_level; /* checked states of that level that violate it                     */
  uint64_t violators;             /* ... over the whole run                                           */
  uint64_t trace_len;             /* states in its counterexample (= level)                           */
  uint64_t fingerprint;           /* set-identity fingerprint of the counterexample's last state      */
} kmc_invariant_report_t;

typedef struct {
  int32_t words;            /* 64-bit words per packed state                              */
  int32_t state_bits;
  int32_t num_actions;
  int32_t num_invariants;
  int32_t num_init;
  int32_t max_fanout;       /* static bound on successors per state                       */
  int32_t check_deadlock;
  int32_t exact;            /* 1: the set key is a bijection of the state (<= 63 bits, or two words stored as a 128-bit key),
                               or the context was created with "exact_set" (the key is then the packed state) */
  char name[128];
  char digest[32];
  uint64_t init_candidates;  /* device Init: candidate assignments over all branches (num_init is then 0); 0 for a table */
} kmc_model_info_t;

/* model_lib: path of a lowered-model library (libkmc_<model>.so, built ahead of time by
 * `python -m kafka_specification_b200.build`).  options_json: flat JSON object, all keys
 * optional: "device":0, "table_log2":27, "max_states":N, "cand_bytes":N, "rank":0, "world":1,
 * "continue":false, "check_deadlock":true|false (override), "timing":true,
 * "stop_after_states":N (bounded run: stop at the first level end holding >= N states),
 * "stream":H (cudaStream_t handle of the caller to launch on instead of a private stream),
 * "fanout_bound":K (successors per state assumed when sizing frontier chunks; default min(MAX_FANOUT, 32)),
 * "gpus":N (N > 1: this ONE context drives N GPUs of the process -- fingerprint-sharded, one host thread per GPU
 *   inside kmc_run, peers mapped with cudaDeviceEnablePeerAccess; kmc_stats / kmc_violation / kmc_trace_* then
 *   report the whole job),
 * "spill":false (the state store is a ring over the live BFS window, max_states slots rounded down to a power of
 *   two; older levels move to host memory -- TLC's DiskStateQueue),
 * "checkpoint_dir":"d", "checkpoint_minutes":M (TLC -checkpoint: states + parent links + counters written at a level
 *   boundary at most every M minutes, 0 = every level; the per-site coverage counts are part of it),
 *   "recover":"d" (TLC -recover: continue from that checkpoint; the set is rebuilt from the stored states),
 * "set_spill":false (one GPU only: when the fingerprint set's table would pass half its slots, its keys move to a host
 *   memory array and the table starts empty, instead of the run ending in KMC_E_TABLE_FULL.  States appended since then
 *   whose key is in host memory are removed before each move and at each level end, so the results are those of a run
 *   with a table large enough.  With "spill" host memory bounds the run; about slot_bytes + 8 * words + 8 bytes per
 *   state, and KMC_E_OOM when it runs out.  A set_spill context refuses "gpus" > 1, world > 1, the kmc_shard_* calls and kmc_fpset_*: KMC_E_BADARG).
 * "exact_set":false (an extension, one GPU only: the fingerprint set's key is the packed state itself -- under SYMMETRY
 *   its orbit's canonical form -- so that no two distinct states can share a key and "no violation" is exact on every
 *   model, not only on those whose key is a bijection already (kmc_model_info.exact = 1 without the option; there the
 *   option is accepted and changes nothing).  A slot is a header word and the state's words: slot_bytes 16 at one word,
 *   32 at two or three, 64 at four to seven, so the same table_log2 takes 1x, 2x or 4x the memory of the 16-byte form
 *   and the default sizing gives a table of fewer slots.  The 64-bit fingerprint still picks the bucket, orders the
 *   counterexamples and names -dump dot nodes.  It combines with "spill", "set_spill" (the keys in host memory are the
 *   states' words) and "recover".  An exact_set context refuses "gpus" > 1, world > 1, the kmc_shard_* calls and
 *   kmc_fpset_* (a 64-bit fingerprint is not a key of this set): KMC_E_BADARG with a message.
 * Unknown keys are ignored.  */
int kmc_create(const char* model_lib, const char* options_json, kmc_ctx** out);
void kmc_destroy(kmc_ctx* ctx);
int kmc_model_info(const kmc_ctx* ctx, kmc_model_info_t* out);

int kmc_run(kmc_ctx* ctx);                                   /* blocking full BFS         */
int kmc_stats(const kmc_ctx* ctx, kmc_stats_t* out);
int kmc_level_widths(const kmc_ctx* ctx, uint64_t* out, size_t cap, size_t* n);
/* successors generated per action of the last run (index = action id of the parent words); *n = number of actions */
int kmc_action_counts(const kmc_ctx* ctx, uint64_t* out, size_t cap, size_t* n);
/* Coverage of the last run (TLC -coverage), kept by the kernels on every run at no measurable cost:
 *   action_generated[a]  successors produced by action a (duplicates and successors a CONSTRAINT discards included)
 *   action_distinct[a]   new states whose parent word carries action a (initial states are not counted)
 *   site_generated[i]    successors produced by emit site i of the lowered Next (model.json "sites" maps i to its action)
 * Up to action_cap / site_cap entries are written; *n_actions / *n_sites receive the full counts.  Generated per action
 * is deterministic, and so is generated per site without SYMMETRY (with it, the orbit member that is stored and
 * expanded is the one whose insert won, and members spread their successors differently over per-replica sites).
 * Distinct per action depends on which generator of a new state won the insert (as in TLC with more than one
 * worker), and sum(distinct) + initial states = distinct states.  *complete = 0 after recovering from a
 * checkpoint written without per-site counts: the generated counts then cover only the levels run since.  With
 * "gpus": N the counts are summed over the GPUs; a multi-process (kmc_shard_*) driver reads them per rank. */
int kmc_coverage(const kmc_ctx* ctx, uint64_t* action_generated, uint64_t* action_distinct, size_t action_cap,
                 uint64_t* site_generated, size_t site_cap, size_t* n_actions, size_t* n_sites, int32_t* complete);
int kmc_violation(const kmc_ctx* ctx, kmc_violation_t* out);
/* i-th state of the error trace (0 = an initial state); buf receives `words` uint64_t.    */
int kmc_trace_state(const kmc_ctx* ctx, uint32_t i, uint64_t* buf, size_t cap_words, uint32_t* action_id);
/* Every violated invariant of the last run with "continue": true, ordered by (level, invariant); invariants never
 * violated are absent, and deadlocks stay in kmc_violation.  "Checked" states are the stored states and the successors
 * a CONSTRAINT discards (each time one is generated).  Each report's counterexample is, among the violators of its
 * first level, the one kmc_violation's rule picks (smallest fingerprint, then smallest parent word); so when
 * kmc_violation reports an invariant, it is that invariant's entry here (as long as the level's violators fit the
 * 2^16-row ring: beyond that neither pick is deterministic).  Up to cap entries are written, *n receives the full
 * count.  *complete = 0 after -recover: the report then covers only the levels searched since.  KMC_E_BADARG on a
 * model with more than 64 invariants; KMC_E_STATE on one rank of a multi-process (kmc_shard_*, world > 1) driver.  */
int kmc_invariant_reports(const kmc_ctx* ctx, kmc_invariant_report_t* out, size_t cap, size_t* n, int32_t* complete);
/* i-th state of the counterexample of invariant `invariant` (0 = an initial state), as kmc_trace_state.           */
int kmc_invariant_trace_state(const kmc_ctx* ctx, int32_t invariant, uint32_t i, uint64_t* buf, size_t cap_words,
                              uint32_t* action_id);
/* copy packed states [first, first+count) of the state store to host memory               */
int kmc_copy_states(const kmc_ctx* ctx, uint64_t first, uint64_t count, uint64_t* buf);
/* parent words of the same range: bits 0..39 store index, 40..47 owner rank of the parent,
 * 56..63 action id; low 48 bits all ones = initial state (TLC's trace file)                 */
int kmc_copy_parents(const kmc_ctx* ctx, uint64_t first, uint64_t count, uint64_t* buf);
/* One transition of the state graph (kmc_edges): `src` is the global store index of the source state, `src_fp` and
 * `dst_fp` the set-identity fingerprints of source and successor (state_fp: under SYMMETRY that of the orbit, the
 * fingerprint kmc_violation reports), `action` the action id of model.json.                                          */
typedef struct {
  uint64_t src;
  uint64_t src_fp;
  uint64_t dst_fp;
  uint32_t action;
  uint32_t pad;
} kmc_edge_t;
/* Every transition out of the stored states [first, first+count) of the last kmc_run (TLC -dump dot): each successor
 * the lowered Next generates and the CONSTRAINT keeps, duplicates and self-loops included, in no particular order.  The
 * states are expanded again on the GPU (the non-fused expand kernel, then k_edges), in chunks that fit the candidate
 * buffer; spilled states are staged from host memory.  The run is left exactly as it was: stats, coverage, violations,
 * reports and the store.  Up to cap edges are written, *n receives the full count.  One GPU only: KMC_E_BADARG on a
 * "gpus" > 1 or world > 1 context; KMC_E_STATE before a kmc_run; KMC_E_LAYOUT_OVERFLOW when a successor of the range
 * does not fit the layout (the unexpanded last level of a stopped run can hold such a state).                        */
int kmc_edges(kmc_ctx* ctx, uint64_t first, uint64_t count, kmc_edge_t* out, size_t cap, size_t* n);
/* out[i] = set-identity fingerprint (as kmc_edge_t.src_fp) of stored state first + i, computed on the host; the
 * same conditions as kmc_edges.                                                                                        */
int kmc_fingerprints(kmc_ctx* ctx, uint64_t first, uint64_t count, uint64_t* out);
/* this rank's offending state (packed words) and its parent word -- the starting point of a trace
 * walk that crosses ranks (a multi-rank driver follows parent words through kmc_copy_*)      */
int kmc_violation_record(const kmc_ctx* ctx, uint64_t* words, size_t cap_words, uint64_t* parent_word);
const char* kmc_strerror(const kmc_ctx* ctx, int code);

/* ---- fingerprint set alone (FPSet.put / contains / size) ------------------------------ */
/* fps: n host fingerprints; out_seen[i] = 1 if already present (TLC's put() contract).
 * Fingerprint 0 is stored as 1 (0 marks an empty 8-byte slot), so 0 and 1 are the same key.  */
int kmc_fpset_put(kmc_ctx* ctx, const uint64_t* fps, size_t n, uint8_t* out_seen);
int kmc_fpset_contains(kmc_ctx* ctx, const uint64_t* fps, size_t n, uint8_t* out_present);
int kmc_fpset_size(const kmc_ctx* ctx, uint64_t* out);

/* ---- per-level building blocks for a fingerprint-sharded multi-rank driver ------------ */
/* All pointers returned are DEVICE pointers owned by the ctx.                              */
typedef struct {
  uint64_t* cand;           /* candidate rows: (words + 1) uint64 each; region d starts at */
  uint64_t region_rows;     /*   cand + d * region_rows * (words + 1), d = owner rank      */
  uint64_t* cand_counts;    /* device array [world]: rows produced for each owner          */
  uint64_t* recv;           /* receive buffer for rows owned by this rank                  */
  uint64_t recv_rows_cap;
  int32_t row_words;        /* words + 1                                                   */
} kmc_shard_buffers_t;

int kmc_shard_begin(kmc_ctx* ctx);                           /* reset set/store/counters   */
int kmc_shard_buffers(kmc_ctx* ctx, kmc_shard_buffers_t* out);
int kmc_shard_seed_init(kmc_ctx* ctx);                       /* init states -> cand regions */
/* expand frontier states [first, first+count) of this rank's current level into cand      */
int kmc_shard_expand(kmc_ctx* ctx, uint64_t first, uint64_t count);
int kmc_shard_counts(kmc_ctx* ctx, uint64_t* host_counts /* [world] */);
int kmc_shard_reset_cand(kmc_ctx* ctx);
/* insert `rows` received rows from `rows_dev` (device) into this rank's set; new states are
 * appended to the store; returns the new store tail                                       */
int kmc_shard_insert(kmc_ctx* ctx, const uint64_t* rows_dev, uint64_t rows, uint64_t* new_tail);
int kmc_shard_level_done(kmc_ctx* ctx, uint64_t* level_first, uint64_t* level_count);
int kmc_shard_sync(kmc_ctx* ctx);

/* ---- fused expand + exchange over peer memory (NVLink): replaces counts/exchange/insert above ------
 * Every rank owns an inbox (two buffers); kmc_shard_ipc_handle exports it (64-byte CUDA IPC handle),
 * kmc_shard_open_peers maps all ranks' inboxes.  Per round: kmc_shard_expand_p2p (the expand kernel
 * stores each successor row directly into its owner's inbox and publishes the row counts there) ->
 * a cross-rank barrier enqueued by the caller on the engine's stream -> kmc_shard_insert_p2p.       */
int kmc_shard_ipc_handle(kmc_ctx* ctx, void* out64);
int kmc_shard_open_peers(kmc_ctx* ctx, const void* handles /* world x 64 bytes */, uint32_t world);
int kmc_shard_seed_p2p(kmc_ctx* ctx);
int kmc_shard_expand_p2p(kmc_ctx* ctx, uint64_t first, uint64_t count);
int kmc_shard_insert_p2p(kmc_ctx* ctx);

/* ---- the same with DEVICE-SIDE cross-rank synchronisation (no NCCL collective, no host wait inside a level) ----
 * A sync page in front of every inbox holds per-source "ready" and per-destination "done" round counters and a
 * level board; peers push into it over NVLink, its owner polls it locally from tiny wait kernels on the stream.
 * kmc_shard_round_p2p   one expand (or, seed != 0, initial states) -> exchange -> insert round; every rank calls it
 *                       the same number of times per level (count = 0 on ranks without work)
 * kmc_shard_level_sync  invariants + publish this rank's level summary to all ranks + wait for all summaries; the ONE
 *                       host synchronisation of a level.  board receives world x 8 words per rank:
 *                       {level id, new states, violations, store tail, generated, fail, deadlocks,
 *                        invariants first violated at this level (bit mask, "continue" runs)}
 * kmc_shard_inbox_ptr / kmc_shard_open_peers_direct: peers inside one process (one ctx per GPU, host threads):
 *                       direct device pointers + cudaDeviceEnablePeerAccess instead of CUDA IPC handles.           */
int kmc_shard_round_p2p(kmc_ctx* ctx, uint64_t first, uint64_t count, int seed);
int kmc_shard_level_sync(kmc_ctx* ctx, uint64_t* board /* world x 8 */);
int kmc_shard_inbox_ptr(kmc_ctx* ctx, void** out);
int kmc_shard_open_peers_direct(kmc_ctx* ctx, void* const* inboxes, const int* devices, uint32_t world);

#ifdef __cplusplus
}
#endif
#endif /* KSPECMC_H */
