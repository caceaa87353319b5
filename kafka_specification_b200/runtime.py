"""ctypes binding of ``libkspecmc.so`` (include/kspecmc.h) -- the host side above the C ABI.

Mirrors the reference-facing interface of the replaced path (TLC's ``ModelChecker``: run a
model, read "states generated / distinct states / depth", fetch the error trace).  There is no
CPU fallback: if the library, the lowered model or the GPU is missing, construction raises.
"""
from __future__ import annotations

import ctypes
import json
import os
import time
from dataclasses import dataclass, field

import numpy as np

from .frontend.values import fmt
from .lower.layout import Layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "build")

KMC_ERRORS = {
    0: "KMC_OK", -1: "KMC_E_BADARG", -2: "KMC_E_CUDA", -3: "KMC_E_OOM", -4: "KMC_E_TABLE_FULL",
    -5: "KMC_E_STORE_FULL", -6: "KMC_E_LAYOUT_OVERFLOW", -7: "KMC_E_MODEL", -8: "KMC_E_STATE", -9: "KMC_E_NO_GPU",
    -10: "KMC_E_CAND_FULL", -11: "KMC_E_PEER_TIMEOUT", -12: "KMC_E_SET_TIMEOUT",
}


class KmcError(RuntimeError):
    def __init__(self, code: int, text: str):
        super().__init__(f"{KMC_ERRORS.get(code, code)}: {text}")
        self.code = code


class Stats(ctypes.Structure):
    _fields_ = [
        ("distinct", ctypes.c_uint64), ("generated", ctypes.c_uint64), ("queue", ctypes.c_uint64),
        ("depth", ctypes.c_uint64), ("deadlocks", ctypes.c_uint64), ("out_of_model", ctypes.c_uint64),
        ("probes", ctypes.c_uint64), ("levels", ctypes.c_uint64),
        ("gpu_ms_total", ctypes.c_double), ("gpu_ms_expand", ctypes.c_double), ("gpu_ms_insert", ctypes.c_double),
        ("launches_expand", ctypes.c_uint64), ("launches_insert", ctypes.c_uint64), ("launches_other", ctypes.c_uint64),
        ("wall_ms", ctypes.c_double), ("table_slots", ctypes.c_uint64), ("max_states", ctypes.c_uint64),
        ("complete", ctypes.c_uint64), ("gpu_ms_invariant", ctypes.c_double), ("slot_bytes", ctypes.c_uint64),
        ("set_flushes", ctypes.c_uint64), ("set_host_keys", ctypes.c_uint64), ("set_filtered", ctypes.c_uint64),
        ("gpu_ms_set_spill", ctypes.c_double), ("set_link_bytes", ctypes.c_uint64),
        ("init_generated", ctypes.c_uint64), ("init_candidates", ctypes.c_uint64), ("gpu_ms_init", ctypes.c_double),
    ]

    def as_dict(self) -> dict:
        return {n: getattr(self, n) for n, _ in self._fields_}


class Violation(ctypes.Structure):
    _fields_ = [("kind", ctypes.c_int32), ("invariant", ctypes.c_int32), ("level", ctypes.c_uint64),
                ("trace_len", ctypes.c_uint64), ("fingerprint", ctypes.c_uint64)]


class InvariantReport(ctypes.Structure):
    _fields_ = [("invariant", ctypes.c_int32), ("level", ctypes.c_uint64), ("violators_first_level", ctypes.c_uint64),
                ("violators", ctypes.c_uint64), ("trace_len", ctypes.c_uint64), ("fingerprint", ctypes.c_uint64)]


class ModelInfo(ctypes.Structure):
    _fields_ = [("words", ctypes.c_int32), ("state_bits", ctypes.c_int32), ("num_actions", ctypes.c_int32),
                ("num_invariants", ctypes.c_int32), ("num_init", ctypes.c_int32), ("max_fanout", ctypes.c_int32),
                ("check_deadlock", ctypes.c_int32), ("exact", ctypes.c_int32),
                ("name", ctypes.c_char * 128), ("digest", ctypes.c_char * 32), ("init_candidates", ctypes.c_uint64)]


# kmc_edge_t as a numpy record: Checker.edges returns arrays of it, which kmc_edges fills in place
EDGE_DTYPE = np.dtype([("src", np.uint64), ("src_fp", np.uint64), ("dst_fp", np.uint64), ("action", np.uint32),
                       ("pad", np.uint32)])


class ShardBuffers(ctypes.Structure):
    _fields_ = [("cand", ctypes.c_void_p), ("region_rows", ctypes.c_uint64), ("cand_counts", ctypes.c_void_p),
                ("recv", ctypes.c_void_p), ("recv_rows_cap", ctypes.c_uint64), ("row_words", ctypes.c_int32)]


_LIB = None


def load_library(path: str | None = None) -> ctypes.CDLL:
    """Loads libkspecmc.so; fails loudly when it has not been built."""
    global _LIB
    if _LIB is not None and path is None:
        return _LIB
    path = path or os.path.join(BUILD, "libkspecmc.so")
    if not os.path.exists(path):
        raise KmcError(-7, f"{path} is missing: run `python -m kafka_specification_b200.build --all` "
                           f"(there is no CPU fallback)")
    lib = ctypes.CDLL(path)
    vp, u64p = ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint64)
    lib.kmc_create.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.POINTER(vp)]
    lib.kmc_destroy.argtypes = [vp]
    lib.kmc_destroy.restype = None
    lib.kmc_model_info.argtypes = [vp, ctypes.POINTER(ModelInfo)]
    lib.kmc_run.argtypes = [vp]
    lib.kmc_stats.argtypes = [vp, ctypes.POINTER(Stats)]
    lib.kmc_level_widths.argtypes = [vp, u64p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t)]
    lib.kmc_action_counts.argtypes = [vp, u64p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t)]
    lib.kmc_coverage.argtypes = [vp, u64p, u64p, ctypes.c_size_t, u64p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t),
                                 ctypes.POINTER(ctypes.c_size_t), ctypes.POINTER(ctypes.c_int32)]
    lib.kmc_violation.argtypes = [vp, ctypes.POINTER(Violation)]
    lib.kmc_trace_state.argtypes = [vp, ctypes.c_uint32, u64p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint32)]
    lib.kmc_copy_states.argtypes = [vp, ctypes.c_uint64, ctypes.c_uint64, vp]
    lib.kmc_copy_parents.argtypes = [vp, ctypes.c_uint64, ctypes.c_uint64, vp]
    lib.kmc_violation_record.argtypes = [vp, u64p, ctypes.c_size_t, u64p]
    lib.kmc_edges.argtypes = [vp, ctypes.c_uint64, ctypes.c_uint64, vp, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t)]
    lib.kmc_fingerprints.argtypes = [vp, ctypes.c_uint64, ctypes.c_uint64, vp]
    lib.kmc_invariant_reports.argtypes = [vp, ctypes.POINTER(InvariantReport), ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t),
                                          ctypes.POINTER(ctypes.c_int32)]
    lib.kmc_invariant_trace_state.argtypes = [vp, ctypes.c_int32, ctypes.c_uint32, u64p, ctypes.c_size_t,
                                              ctypes.POINTER(ctypes.c_uint32)]
    lib.kmc_strerror.argtypes = [vp, ctypes.c_int]
    lib.kmc_strerror.restype = ctypes.c_char_p
    lib.kmc_fpset_put.argtypes = [vp, vp, ctypes.c_size_t, vp]
    lib.kmc_fpset_contains.argtypes = [vp, vp, ctypes.c_size_t, vp]
    lib.kmc_fpset_size.argtypes = [vp, u64p]
    lib.kmc_shard_begin.argtypes = [vp]
    lib.kmc_shard_buffers.argtypes = [vp, ctypes.POINTER(ShardBuffers)]
    lib.kmc_shard_seed_init.argtypes = [vp]
    lib.kmc_shard_expand.argtypes = [vp, ctypes.c_uint64, ctypes.c_uint64]
    lib.kmc_shard_counts.argtypes = [vp, u64p]
    lib.kmc_shard_reset_cand.argtypes = [vp]
    lib.kmc_shard_insert.argtypes = [vp, vp, ctypes.c_uint64, u64p]
    lib.kmc_shard_level_done.argtypes = [vp, u64p, u64p]
    lib.kmc_shard_sync.argtypes = [vp]
    lib.kmc_shard_ipc_handle.argtypes = [vp, vp]
    lib.kmc_shard_open_peers.argtypes = [vp, vp, ctypes.c_uint32]
    lib.kmc_shard_seed_p2p.argtypes = [vp]
    lib.kmc_shard_expand_p2p.argtypes = [vp, ctypes.c_uint64, ctypes.c_uint64]
    lib.kmc_shard_insert_p2p.argtypes = [vp]
    lib.kmc_shard_round_p2p.argtypes = [vp, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_int]
    lib.kmc_shard_level_sync.argtypes = [vp, u64p]
    lib.kmc_shard_inbox_ptr.argtypes = [vp, ctypes.POINTER(vp)]
    lib.kmc_shard_open_peers_direct.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_int), ctypes.c_uint32]
    for fn in ("kmc_create", "kmc_model_info", "kmc_run", "kmc_stats", "kmc_level_widths", "kmc_action_counts", "kmc_coverage",
               "kmc_violation", "kmc_trace_state", "kmc_copy_states", "kmc_copy_parents", "kmc_violation_record", "kmc_edges", "kmc_fingerprints", "kmc_invariant_reports", "kmc_invariant_trace_state", "kmc_fpset_put", "kmc_fpset_contains",
               "kmc_fpset_size", "kmc_shard_begin", "kmc_shard_buffers", "kmc_shard_seed_init", "kmc_shard_expand",
               "kmc_shard_counts", "kmc_shard_reset_cand", "kmc_shard_insert", "kmc_shard_level_done", "kmc_shard_sync",
               "kmc_shard_ipc_handle", "kmc_shard_open_peers", "kmc_shard_seed_p2p", "kmc_shard_expand_p2p",
               "kmc_shard_insert_p2p", "kmc_shard_round_p2p", "kmc_shard_level_sync", "kmc_shard_inbox_ptr",
               "kmc_shard_open_peers_direct"):
        getattr(lib, fn).restype = ctypes.c_int
    _LIB = lib
    return lib


def model_paths(name: str) -> tuple[str, str]:
    d = os.path.join(BUILD, "models", name)
    return os.path.join(d, f"libkmc_{name}.so"), os.path.join(d, "model.json")


class StateDecoder:
    """Rebuilds TLA+ values from packed words with the lowering's layout types, rebuilt from model.json."""

    def __init__(self, meta: dict):
        self.meta = meta
        self.layout = Layout.from_description(meta["layout"])
        self.variables = self.layout.variables

    def decode(self, words) -> dict:
        return self.layout.py_unpack(words)

    def text(self, words) -> str:
        st = self.decode(words)
        return "\n".join(f"/\\ {v} = {fmt(st[v])}" for v in self.variables)

    def texts(self, rows) -> list[str]:
        """TLC-style text of MANY packed states (rows: [n, W] uint64): the atom codes are extracted with numpy, and
        every variable is decoded once per DISTINCT value it takes in the batch (a few thousand for millions of
        states), so that state-set digests of 10^6..10^7 states take seconds instead of minutes."""
        lay = self.layout
        rows = np.ascontiguousarray(rows, dtype=np.uint64).reshape(-1, lay.words)
        n = rows.shape[0]
        if n == 0:
            return []
        codes = np.empty((n, len(lay.atoms)), dtype=np.int64)
        for a in lay.atoms:
            codes[:, a.index] = ((rows[:, a.word] >> np.uint64(a.shift)) & np.uint64(a.mask)).astype(np.int64)
        parts = []
        for v in self.variables:
            b, e = lay.spans[v]
            uniq, inv = np.unique(codes[:, b:e], axis=0, return_inverse=True)
            table = [f"/\\ {v} = {fmt(lay.var_types[v].py_read(dict(zip(range(b, e), map(int, u)))))}" for u in uniq]
            parts.append([table[j] for j in np.asarray(inv).reshape(-1)])
        return ["\n".join(p) for p in zip(*parts)]


# ---------------------------------------------------------------------------
@dataclass
class RunResult:
    distinct: int
    generated: int
    depth: int
    queue: int
    deadlocks: int
    complete: bool
    levels: list[int]
    stats: dict
    violation: dict | None = None
    trace: list[dict] = field(default_factory=list)
    # with "continue": every violated invariant (Checker.invariant_reports), ordered by (level, cfg index)
    invariant_violations: list[dict] = field(default_factory=list)
    # Init solutions, duplicates included, and (device Init) the candidate assignments decoded on the GPU
    init_generated: int = 0
    init_candidates: int = 0


class Checker:
    """One GPU-resident model checker instance (one ``kmc_ctx``).  ``options`` are kmc_create's JSON options
    (include/kspecmc.h), e.g. ``table_log2=27, max_states=N, spill=True, set_spill=True, exact_set=True``; ``cont``
    stands for ``continue``."""

    def __init__(self, model: str, model_lib: str | None = None, model_json: str | None = None, **options):
        self.lib = load_library()
        lib_path, json_path = model_paths(model)
        self.model_lib = model_lib or lib_path
        json_path = model_json or json_path
        if not os.path.exists(self.model_lib):
            raise KmcError(-7, f"lowered model library {self.model_lib} is missing (build it first; no CPU fallback)")
        with open(json_path) as f:
            self.meta = json.load(f)
        self.decoder = StateDecoder(self.meta)
        self.ctx = ctypes.c_void_p()
        opts = {("continue" if k == "cont" else k): v for k, v in options.items() if k not in ("p2p", "device_sync")}
        self.cont = bool(opts.get("continue"))
        rc = self.lib.kmc_create(self.model_lib.encode(), json.dumps(opts).encode(), ctypes.byref(self.ctx))
        if rc != 0:
            msg = self.lib.kmc_strerror(self.ctx, rc).decode() if self.ctx else "kmc_create failed"
            if self.ctx:
                self.lib.kmc_destroy(self.ctx)
                self.ctx = None
            raise KmcError(rc, msg)
        self.info = ModelInfo()
        self._check(self.lib.kmc_model_info(self.ctx, ctypes.byref(self.info)))
        if self.info.digest.decode() != self.meta["digest"]:
            raise KmcError(-7, "model.json does not belong to the loaded model library (digest mismatch)")
        self.words = self.info.words

    def _check(self, rc: int):
        if rc != 0:
            raise KmcError(rc, self.lib.kmc_strerror(self.ctx, rc).decode())

    def close(self):
        if getattr(self, "ctx", None):
            self.lib.kmc_destroy(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # -- full BFS ------------------------------------------------------------
    def stats(self) -> dict:
        st = Stats()
        self._check(self.lib.kmc_stats(self.ctx, ctypes.byref(st)))
        return st.as_dict()

    def level_widths(self) -> list[int]:
        buf = (ctypes.c_uint64 * 4096)()
        n = ctypes.c_size_t()
        self._check(self.lib.kmc_level_widths(self.ctx, buf, 4096, ctypes.byref(n)))
        return [int(buf[i]) for i in range(min(n.value, 4096))]

    def action_counts(self) -> dict:
        """Successors generated per action by the last run."""
        cap = len(self.meta["actions"])
        buf = (ctypes.c_uint64 * cap)()
        n = ctypes.c_size_t()
        self._check(self.lib.kmc_action_counts(self.ctx, buf, cap, ctypes.byref(n)))
        return {a["name"]: int(buf[i]) for i, a in enumerate(self.meta["actions"]) if i < n.value}

    def coverage(self) -> dict:
        """TLC's coverage report of the last run:

        * ``init``: the initial predicate (name, module, source span) with ``distinct`` / ``generated`` initial states;
        * ``actions``: per action of model.json, ``{name, module, location, generated, distinct}``;
        * ``sites``: successors generated per emit site of the lowered Next (model.json ``sites`` gives each one's action);
        * ``complete``: False after recovering from a checkpoint without per-site counts (generated is then partial).

        Generated per action is deterministic, and so is generated per site without SYMMETRY; distinct per action
        depends on which generator of a new state won the insert (as in TLC with several workers).
        """
        acts, n_sites_meta = self.meta["actions"], len(self.meta.get("sites", []))
        na, ns = len(acts), max(n_sites_meta, 1)
        gen, dist, site = (ctypes.c_uint64 * na)(), (ctypes.c_uint64 * na)(), (ctypes.c_uint64 * ns)()
        n_a, n_s, complete = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_int32()
        self._check(self.lib.kmc_coverage(self.ctx, gen, dist, na, site, ns, ctypes.byref(n_a), ctypes.byref(n_s),
                                          ctypes.byref(complete)))
        if n_a.value != na or n_s.value != n_sites_meta:
            raise KmcError(-7, "model.json does not describe the loaded model library's actions and emit sites")
        st = self.stats()
        actions = [{"name": a["name"], "module": a.get("module"), "location": {k: a[k] for k in ("line", "col", "end_line", "end_col") if k in a},
                    "generated": int(gen[i]), "distinct": int(dist[i])} for i, a in enumerate(acts)]
        init_distinct = st["distinct"] - sum(a["distinct"] for a in actions)
        init = dict(self.meta.get("init", {"name": "Init"}))
        # a device-form Init (model.json init.device) has no table: its generated count comes from the run
        device = bool(init.pop("device", False))
        init.pop("candidates", None)
        init.pop("branches", None)
        return {"init": {**init, "distinct": init_distinct,
                         "generated": st["init_generated"] if device else len(self.meta["init_states"])},
                "actions": actions, "sites": [int(site[i]) for i in range(n_s.value)], "complete": bool(complete.value)}

    def violation(self) -> dict | None:
        v = Violation()
        self._check(self.lib.kmc_violation(self.ctx, ctypes.byref(v)))
        if v.kind == 0:
            return None
        return {"kind": "invariant" if v.kind == 1 else "deadlock",
                "invariant": self.meta["invariants"][v.invariant] if v.kind == 1 else None,
                "level": int(v.level), "trace_len": int(v.trace_len), "fingerprint": int(v.fingerprint)}

    def _trace_entry(self, i: int, buf, act) -> dict:
        words = [int(buf[k]) for k in range(self.words)]
        a = self.meta["actions"][act.value] if (i > 0 and act.value < len(self.meta["actions"])) else None
        return {"words": words, "action": a, "state": self.decoder.decode(words), "text": self.decoder.text(words)}

    def trace(self) -> list[dict]:
        v = self.violation()
        if v is None:
            return []
        out = []
        buf = (ctypes.c_uint64 * self.words)()
        act = ctypes.c_uint32()
        for i in range(v["trace_len"]):
            self._check(self.lib.kmc_trace_state(self.ctx, i, buf, self.words, ctypes.byref(act)))
            out.append(self._trace_entry(i, buf, act))
        return out

    def invariant_reports(self) -> list[dict]:
        """Every invariant the last ``continue`` run found violated, ordered by (level, cfg index): ``invariant`` (name),
        ``index`` (in the cfg), ``level`` (its first violating level), ``violators_first_level``, ``violators``,
        ``fingerprint``, ``trace_len``, ``trace`` (decoded like ``trace()``: the counterexample ending in the smallest-
        fingerprint violator of that level) and ``complete`` (False after a recover: only the levels searched since)."""
        n, complete = ctypes.c_size_t(), ctypes.c_int32()
        self._check(self.lib.kmc_invariant_reports(self.ctx, None, 0, ctypes.byref(n), ctypes.byref(complete)))
        reps = (InvariantReport * max(n.value, 1))()
        self._check(self.lib.kmc_invariant_reports(self.ctx, reps, n.value, ctypes.byref(n), ctypes.byref(complete)))
        buf = (ctypes.c_uint64 * self.words)()
        act = ctypes.c_uint32()
        out = []
        for r in reps[:n.value]:
            trace = []
            for i in range(r.trace_len):
                self._check(self.lib.kmc_invariant_trace_state(self.ctx, r.invariant, i, buf, self.words, ctypes.byref(act)))
                trace.append(self._trace_entry(i, buf, act))
            out.append({"invariant": self.meta["invariants"][r.invariant], "index": int(r.invariant), "level": int(r.level),
                        "violators_first_level": int(r.violators_first_level), "violators": int(r.violators),
                        "fingerprint": int(r.fingerprint), "trace_len": int(r.trace_len), "trace": trace,
                        "complete": bool(complete.value)})
        return out

    def run(self, raise_on_error: bool = True) -> RunResult:
        self.last_rc = self.lib.kmc_run(self.ctx)
        if self.last_rc != 0 and raise_on_error:
            self._check(self.last_rc)
        return self.result()

    def error_text(self, rc: int) -> str:
        return self.lib.kmc_strerror(self.ctx, rc).decode()

    def result(self) -> RunResult:
        st = self.stats()
        viol = self.violation()
        # (a model with more than 64 invariants has no per-invariant report)
        reports = self.invariant_reports() if self.cont and len(self.meta["invariants"]) <= 64 else []
        return RunResult(distinct=st["distinct"], generated=st["generated"], depth=st["depth"], queue=st["queue"],
                         deadlocks=st["deadlocks"], complete=bool(st["complete"]), levels=self.level_widths(),
                         stats=st, violation=viol, trace=self.trace() if viol else [], invariant_violations=reports,
                         init_generated=st["init_generated"], init_candidates=st["init_candidates"])

    def violation_record(self):
        """(packed words, parent word) of this rank's offending state, or None."""
        buf = (ctypes.c_uint64 * self.words)()
        meta = ctypes.c_uint64()
        rc = self.lib.kmc_violation_record(self.ctx, buf, self.words, ctypes.byref(meta))
        if rc != 0:
            return None
        return [int(buf[k]) for k in range(self.words)], int(meta.value)

    def state_and_parent(self, idx: int):
        st = self.copy_states(idx, 1)[0]
        par = np.empty(1, dtype=np.uint64)
        self._check(self.lib.kmc_copy_parents(self.ctx, idx, 1, par.ctypes.data))
        return [int(x) for x in st], int(par[0])

    def copy_states(self, first: int, count: int) -> np.ndarray:
        buf = np.empty((count, self.words), dtype=np.uint64)
        if count:
            self._check(self.lib.kmc_copy_states(self.ctx, first, count, buf.ctypes.data))
        return buf

    # -- the state set and the state graph (TLC -dump) ------------------------
    def level_ranges(self) -> list[tuple[int, int]]:
        """(first, count) of every BFS level in the store; the last one is the queue when the run stopped early."""
        out, first = [], 0
        for w in self.level_widths():
            out.append((first, w))
            first += w
        distinct = self.stats()["distinct"]
        if distinct > first:
            out.append((first, distinct - first))
        return out

    def edges(self, first: int, count: int, chunk: int = 1 << 20) -> np.ndarray:
        """Every transition out of the stored states [first, first+count) as an ``EDGE_DTYPE`` array: the successors the
        lowered Next generates and the CONSTRAINT keeps, duplicates and self-loops included, in no particular order
        (kmc_edges, enumerated on the GPU; the run's results are left as they were).  The states go to kmc_edges ``chunk``
        at a time; a chunk whose edges outgrow the buffer (sized for min(max_fanout, 8) per state, then for the largest
        count seen) is asked for again with room for all of them."""
        parts, n = [], ctypes.c_size_t()
        per_state = max(1, min(self.info.max_fanout, 8))
        for off in range(first, first + count, chunk):
            m = min(chunk, first + count - off)
            cap = m * per_state
            while True:
                buf = np.empty(cap, dtype=EDGE_DTYPE)
                self._check(self.lib.kmc_edges(self.ctx, off, m, buf.ctypes.data, cap, ctypes.byref(n)))
                if n.value <= cap:
                    break
                cap = n.value
            per_state = max(per_state, -(-n.value // m))
            parts.append(buf[:n.value])
        return np.concatenate(parts) if parts else np.empty(0, dtype=EDGE_DTYPE)

    def fingerprints(self, first: int, count: int) -> np.ndarray:
        """Set-identity fingerprint of each stored state [first, first+count) (``edges()``'s ``src_fp``)."""
        out = np.empty(count, dtype=np.uint64)
        if count:
            self._check(self.lib.kmc_fingerprints(self.ctx, first, count, out.ctypes.data))
        return out

    def dump_states(self, path: str, batch: int = 1 << 20) -> dict:
        """Writes every stored state to ``path`` as TLC's ``-dump`` does (``State k:`` and the state's text, see
        ``dump.py``), level by level; within a level the states are ordered by their packed words, so that the file does
        not depend on which insert won (identical across runs, ``spill`` and ``set_spill`` without SYMMETRY).  Returns
        the states written and the seconds spent decoding and writing."""
        from . import dump
        t = {"states": 0, "decode_s": 0.0, "write_s": 0.0}
        with open(path, "w") as f:
            for first, count in self.level_ranges():
                rows = dump.sorted_rows(self.copy_states(first, count))
                for b in range(0, count, batch):
                    t0 = time.perf_counter()
                    texts = self.decoder.texts(rows[b:b + batch])
                    t1 = time.perf_counter()
                    t["states"] += dump.write_states(f, texts, t["states"] + 1)
                    t["write_s"] += time.perf_counter() - t1
                    t["decode_s"] += t1 - t0
        return t

    def dump_dot(self, path: str, actionlabels: bool = False, colorize: bool = False) -> dict:
        """Writes the state graph to ``path`` in TLC's DotStateWriter layout (``dump.write_dot``): a node per stored
        state, initial states filled, and one edge per distinct (source, successor, action) out of the expanded states
        (``distinct - queue``: a stopped run shows the graph explored so far)."""
        from . import dump
        st = self.stats()
        ranges = self.level_ranges()
        nodes_fp, texts = [], []
        for first, count in ranges:
            rows = self.copy_states(first, count)
            order = dump.row_order(rows)
            nodes_fp.append(self.fingerprints(first, count)[order])
            texts += self.decoder.texts(rows[order])
        n_init = ranges[0][1] if ranges else 0
        edges = self.edges(0, st["distinct"] - st["queue"])
        actions = [a["name"] for a in self.meta["actions"]]
        fps = np.concatenate(nodes_fp) if nodes_fp else np.empty(0, dtype=np.uint64)
        with open(path, "w") as f:
            return dump.write_dot(f, fps, texts, n_init, edges, actions, actionlabels=actionlabels, colorize=colorize)

    # -- fingerprint set alone (FPSet.put / contains / size) -----------------
    def fpset_put(self, fps: np.ndarray) -> np.ndarray:
        fps = np.ascontiguousarray(fps, dtype=np.uint64)
        seen = np.zeros(len(fps), dtype=np.uint8)
        self._check(self.lib.kmc_fpset_put(self.ctx, fps.ctypes.data, len(fps), seen.ctypes.data))
        return seen.astype(bool)

    def fpset_contains(self, fps: np.ndarray) -> np.ndarray:
        fps = np.ascontiguousarray(fps, dtype=np.uint64)
        out = np.zeros(len(fps), dtype=np.uint8)
        self._check(self.lib.kmc_fpset_contains(self.ctx, fps.ctypes.data, len(fps), out.ctypes.data))
        return out.astype(bool)

    def fpset_size(self) -> int:
        n = ctypes.c_uint64()
        self._check(self.lib.kmc_fpset_size(self.ctx, ctypes.byref(n)))
        return int(n.value)
