// kspecmc.cpp -- libkspecmc.so: the model-agnostic front of the C ABI in include/kspecmc.h.
//
// A lowered model is a shared library (libkmc_<model>.so: the engine kernels specialised to the
// spec's packed layout and Next/invariant switch table, see kmc_engine.cu).  kmc_create dlopens it
// and every other call forwards to it, so that JNI / ctypes / cgo bindings link against one
// stable library whatever the spec.  No computation happens here, and there is no CPU fallback:
// if the model library or the GPU is missing the call fails with KMC_E_MODEL / KMC_E_NO_GPU.
#include <dlfcn.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>

#include "kspecmc.h"

struct kmcm_ctx;

struct kmc_ctx {
  void* dl = nullptr;
  kmcm_ctx* inner = nullptr;
  std::string error;
  int (*create)(const char*, kmcm_ctx**) = nullptr;
  void (*destroy)(kmcm_ctx*) = nullptr;
  int (*model_info)(const kmcm_ctx*, kmc_model_info_t*) = nullptr;
  int (*run)(kmcm_ctx*) = nullptr;
  int (*stats)(const kmcm_ctx*, kmc_stats_t*) = nullptr;
  int (*level_widths)(const kmcm_ctx*, uint64_t*, size_t, size_t*) = nullptr;
  int (*action_counts)(const kmcm_ctx*, uint64_t*, size_t, size_t*) = nullptr;
  int (*coverage)(const kmcm_ctx*, uint64_t*, uint64_t*, size_t, uint64_t*, size_t, size_t*, size_t*, int32_t*) = nullptr;
  int (*violation)(const kmcm_ctx*, kmc_violation_t*) = nullptr;
  int (*trace_state)(const kmcm_ctx*, uint32_t, uint64_t*, size_t, uint32_t*) = nullptr;
  int (*copy_states)(const kmcm_ctx*, uint64_t, uint64_t, uint64_t*) = nullptr;
  int (*copy_parents)(const kmcm_ctx*, uint64_t, uint64_t, uint64_t*) = nullptr;
  int (*edges)(kmcm_ctx*, uint64_t, uint64_t, kmc_edge_t*, size_t, size_t*) = nullptr;
  int (*fingerprints)(kmcm_ctx*, uint64_t, uint64_t, uint64_t*) = nullptr;
  int (*violation_record)(const kmcm_ctx*, uint64_t*, size_t, uint64_t*) = nullptr;
  int (*invariant_reports)(const kmcm_ctx*, kmc_invariant_report_t*, size_t, size_t*, int32_t*) = nullptr;
  int (*invariant_trace_state)(const kmcm_ctx*, int32_t, uint32_t, uint64_t*, size_t, uint32_t*) = nullptr;
  const char* (*strerror_)(const kmcm_ctx*, int) = nullptr;
  int (*fpset_put)(kmcm_ctx*, const uint64_t*, size_t, uint8_t*) = nullptr;
  int (*fpset_contains)(kmcm_ctx*, const uint64_t*, size_t, uint8_t*) = nullptr;
  int (*fpset_size)(const kmcm_ctx*, uint64_t*) = nullptr;
  int (*shard_begin)(kmcm_ctx*) = nullptr;
  int (*shard_buffers)(kmcm_ctx*, kmc_shard_buffers_t*) = nullptr;
  int (*shard_seed_init)(kmcm_ctx*) = nullptr;
  int (*shard_expand)(kmcm_ctx*, uint64_t, uint64_t) = nullptr;
  int (*shard_counts)(kmcm_ctx*, uint64_t*) = nullptr;
  int (*shard_reset_cand)(kmcm_ctx*) = nullptr;
  int (*shard_insert)(kmcm_ctx*, const uint64_t*, uint64_t, uint64_t*) = nullptr;
  int (*shard_level_done)(kmcm_ctx*, uint64_t*, uint64_t*) = nullptr;
  int (*shard_sync)(kmcm_ctx*) = nullptr;
  int (*shard_ipc_handle)(kmcm_ctx*, void*) = nullptr;
  int (*shard_open_peers)(kmcm_ctx*, const void*, uint32_t) = nullptr;
  int (*shard_seed_p2p)(kmcm_ctx*) = nullptr;
  int (*shard_expand_p2p)(kmcm_ctx*, uint64_t, uint64_t) = nullptr;
  int (*shard_insert_p2p)(kmcm_ctx*) = nullptr;
  int (*shard_round_p2p)(kmcm_ctx*, uint64_t, uint64_t, int) = nullptr;
  int (*shard_level_sync)(kmcm_ctx*, uint64_t*) = nullptr;
  int (*shard_inbox_ptr)(kmcm_ctx*, void**) = nullptr;
  int (*shard_open_peers_direct)(kmcm_ctx*, void* const*, const int*, uint32_t) = nullptr;
};

template <class F>
static bool bind(kmc_ctx* c, F& fn, const char* name) {
  fn = reinterpret_cast<F>(dlsym(c->dl, name));
  if (!fn) {
    c->error = std::string("model library lacks symbol ") + name;
    return false;
  }
  return true;
}

extern "C" {

int kmc_create(const char* model_lib, const char* options_json, kmc_ctx** out) {
  if (!out || !model_lib) return KMC_E_BADARG;
  kmc_ctx* c = new kmc_ctx();
  *out = c;
  c->dl = dlopen(model_lib, RTLD_NOW | RTLD_LOCAL);
  if (!c->dl) {
    const char* e = dlerror();
    c->error = std::string("cannot load lowered model '") + model_lib + "': " + (e ? e : "?");
    return KMC_E_MODEL;
  }
  bool ok = bind(c, c->create, "kmcm_create") && bind(c, c->destroy, "kmcm_destroy") &&
            bind(c, c->model_info, "kmcm_model_info") && bind(c, c->run, "kmcm_run") &&
            bind(c, c->stats, "kmcm_stats") && bind(c, c->level_widths, "kmcm_level_widths") &&
            bind(c, c->action_counts, "kmcm_action_counts") && bind(c, c->coverage, "kmcm_coverage") &&
            bind(c, c->violation, "kmcm_violation") &&
            bind(c, c->trace_state, "kmcm_trace_state") && bind(c, c->copy_states, "kmcm_copy_states") &&
            bind(c, c->copy_parents, "kmcm_copy_parents") && bind(c, c->violation_record, "kmcm_violation_record") &&
            bind(c, c->edges, "kmcm_edges") && bind(c, c->fingerprints, "kmcm_fingerprints") &&
            bind(c, c->invariant_reports, "kmcm_invariant_reports") &&
            bind(c, c->invariant_trace_state, "kmcm_invariant_trace_state") &&
            bind(c, c->strerror_, "kmcm_strerror") && bind(c, c->fpset_put, "kmcm_fpset_put") &&
            bind(c, c->fpset_contains, "kmcm_fpset_contains") && bind(c, c->fpset_size, "kmcm_fpset_size") &&
            bind(c, c->shard_begin, "kmcm_shard_begin") && bind(c, c->shard_buffers, "kmcm_shard_buffers") &&
            bind(c, c->shard_seed_init, "kmcm_shard_seed_init") && bind(c, c->shard_expand, "kmcm_shard_expand") &&
            bind(c, c->shard_counts, "kmcm_shard_counts") && bind(c, c->shard_reset_cand, "kmcm_shard_reset_cand") &&
            bind(c, c->shard_insert, "kmcm_shard_insert") && bind(c, c->shard_level_done, "kmcm_shard_level_done") &&
            bind(c, c->shard_sync, "kmcm_shard_sync") && bind(c, c->shard_ipc_handle, "kmcm_shard_ipc_handle") &&
            bind(c, c->shard_open_peers, "kmcm_shard_open_peers") && bind(c, c->shard_seed_p2p, "kmcm_shard_seed_p2p") &&
            bind(c, c->shard_expand_p2p, "kmcm_shard_expand_p2p") && bind(c, c->shard_insert_p2p, "kmcm_shard_insert_p2p") &&
            bind(c, c->shard_round_p2p, "kmcm_shard_round_p2p") && bind(c, c->shard_level_sync, "kmcm_shard_level_sync") &&
            bind(c, c->shard_inbox_ptr, "kmcm_shard_inbox_ptr") && bind(c, c->shard_open_peers_direct, "kmcm_shard_open_peers_direct");
  if (!ok) return KMC_E_MODEL;
  return c->create(options_json, &c->inner);
}

void kmc_destroy(kmc_ctx* c) {
  if (!c) return;
  if (c->inner && c->destroy) c->destroy(c->inner);
  // the model library stays mapped until the process exits: a process usually re-creates contexts of the
  // same model, and a loaded-library audit of the process (/proc/self/maps) then shows which lowered model ran
  delete c;
}

const char* kmc_strerror(const kmc_ctx* c, int code) {
  if (c && !c->inner) return c->error.empty() ? "model not loaded" : c->error.c_str();
  if (c && c->strerror_) return c->strerror_(c->inner, code);
  return code == KMC_OK ? "ok" : "error (no context)";
}

#define FWD(name, ...)                            \
  if (!c || !c->inner) return KMC_E_BADARG;       \
  return c->name(c->inner, ##__VA_ARGS__)

int kmc_model_info(const kmc_ctx* c, kmc_model_info_t* out) { FWD(model_info, out); }
int kmc_run(kmc_ctx* c) { FWD(run); }
int kmc_stats(const kmc_ctx* c, kmc_stats_t* out) { FWD(stats, out); }
int kmc_level_widths(const kmc_ctx* c, uint64_t* out, size_t cap, size_t* n) { FWD(level_widths, out, cap, n); }
int kmc_action_counts(const kmc_ctx* c, uint64_t* out, size_t cap, size_t* n) { FWD(action_counts, out, cap, n); }
int kmc_coverage(const kmc_ctx* c, uint64_t* action_gen, uint64_t* action_dist, size_t action_cap, uint64_t* site_gen,
                 size_t site_cap, size_t* n_actions, size_t* n_sites, int32_t* complete) {
  FWD(coverage, action_gen, action_dist, action_cap, site_gen, site_cap, n_actions, n_sites, complete);
}
int kmc_violation(const kmc_ctx* c, kmc_violation_t* out) { FWD(violation, out); }
int kmc_trace_state(const kmc_ctx* c, uint32_t i, uint64_t* buf, size_t cap, uint32_t* a) { FWD(trace_state, i, buf, cap, a); }
int kmc_copy_states(const kmc_ctx* c, uint64_t first, uint64_t count, uint64_t* buf) { FWD(copy_states, first, count, buf); }
int kmc_copy_parents(const kmc_ctx* c, uint64_t first, uint64_t count, uint64_t* buf) { FWD(copy_parents, first, count, buf); }
int kmc_edges(kmc_ctx* c, uint64_t first, uint64_t count, kmc_edge_t* out, size_t cap, size_t* n) {
  FWD(edges, first, count, out, cap, n);
}
int kmc_fingerprints(kmc_ctx* c, uint64_t first, uint64_t count, uint64_t* out) { FWD(fingerprints, first, count, out); }
int kmc_violation_record(const kmc_ctx* c, uint64_t* words, size_t cap, uint64_t* meta) { FWD(violation_record, words, cap, meta); }
int kmc_invariant_reports(const kmc_ctx* c, kmc_invariant_report_t* out, size_t cap, size_t* n, int32_t* complete) {
  FWD(invariant_reports, out, cap, n, complete);
}
int kmc_invariant_trace_state(const kmc_ctx* c, int32_t inv, uint32_t i, uint64_t* buf, size_t cap, uint32_t* a) {
  FWD(invariant_trace_state, inv, i, buf, cap, a);
}
int kmc_fpset_put(kmc_ctx* c, const uint64_t* fps, size_t n, uint8_t* seen) { FWD(fpset_put, fps, n, seen); }
int kmc_fpset_contains(kmc_ctx* c, const uint64_t* fps, size_t n, uint8_t* out) { FWD(fpset_contains, fps, n, out); }
int kmc_fpset_size(const kmc_ctx* c, uint64_t* out) { FWD(fpset_size, out); }
int kmc_shard_begin(kmc_ctx* c) { FWD(shard_begin); }
int kmc_shard_buffers(kmc_ctx* c, kmc_shard_buffers_t* out) { FWD(shard_buffers, out); }
int kmc_shard_seed_init(kmc_ctx* c) { FWD(shard_seed_init); }
int kmc_shard_expand(kmc_ctx* c, uint64_t first, uint64_t count) { FWD(shard_expand, first, count); }
int kmc_shard_counts(kmc_ctx* c, uint64_t* host_counts) { FWD(shard_counts, host_counts); }
int kmc_shard_reset_cand(kmc_ctx* c) { FWD(shard_reset_cand); }
int kmc_shard_insert(kmc_ctx* c, const uint64_t* rows, uint64_t n, uint64_t* tail) { FWD(shard_insert, rows, n, tail); }
int kmc_shard_level_done(kmc_ctx* c, uint64_t* first, uint64_t* count) { FWD(shard_level_done, first, count); }
int kmc_shard_sync(kmc_ctx* c) { FWD(shard_sync); }
int kmc_shard_ipc_handle(kmc_ctx* c, void* out64) { FWD(shard_ipc_handle, out64); }
int kmc_shard_open_peers(kmc_ctx* c, const void* h, uint32_t world) { FWD(shard_open_peers, h, world); }
int kmc_shard_seed_p2p(kmc_ctx* c) { FWD(shard_seed_p2p); }
int kmc_shard_expand_p2p(kmc_ctx* c, uint64_t first, uint64_t count) { FWD(shard_expand_p2p, first, count); }
int kmc_shard_insert_p2p(kmc_ctx* c) { FWD(shard_insert_p2p); }
int kmc_shard_round_p2p(kmc_ctx* c, uint64_t first, uint64_t count, int seed) { FWD(shard_round_p2p, first, count, seed); }
int kmc_shard_level_sync(kmc_ctx* c, uint64_t* board) { FWD(shard_level_sync, board); }
int kmc_shard_inbox_ptr(kmc_ctx* c, void** out) { FWD(shard_inbox_ptr, out); }
int kmc_shard_open_peers_direct(kmc_ctx* c, void* const* inboxes, const int* devices, uint32_t world) {
  FWD(shard_open_peers_direct, inboxes, devices, world);
}

}  // extern "C"
