"""Test support: a lowered model compiled for the host (host_model.cpp), its sequential BFS and per-state calls.

One library per pair of header texts (model.h and invariants.h), built under build/hosttest/ on first use: headers
lowered inside a test and the same headers from build() share it."""
from __future__ import annotations

import ctypes
import functools
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from kafka_specification_b200.build import device_init_registry, registry, tla_search_dirs  # noqa: E402
from kafka_specification_b200.lower.model import LoweredModel, lower_model  # noqa: E402,F401

BUILD = os.path.join(ROOT, "build", "hosttest")
SOURCE = os.path.join(HERE, "host_model.cpp")
M64 = (1 << 64) - 1

_i32, _u32, _u64, _vp = ctypes.c_int, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_void_p
_u64p, _i64p = ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_int64)
# (restype, argtypes) of every entry point of host_model.cpp
SIGNATURES = {
    **{fn: (_i32, []) for fn in ("hm_words", "hm_state_bits", "hm_all_ones_possible", "hm_has_symmetry", "hm_num_actions",
                                 "hm_num_sites", "hm_num_invariants", "hm_num_init", "hm_check_deadlock", "hs_row_words")},
    "hm_digest": (ctypes.c_char_p, []),
    "hm_site_action": (_i32, [_i32]),
    "hm_successors": (_i32, [_vp, _i32, _vp, _vp, _i32]),
    "hm_first_violated": (_i32, [_vp]),
    "hm_mask": (_u64, [_vp]),
    "hm_in_model": (_i32, [_vp]),
    "hm_init_state": (None, [_i32, _vp]),
    "hm_init_branches": (_i32, []),
    "hm_init_space": (_u64, [_i32]),
    "hm_init_candidate": (_i32, [_i32, _u64, _vp]),
    "hm_init_solutions": (_i32, [_vp, _u64, _vp]),
    "hm_canonicalize": (None, [_vp, _u64, _vp]),
    "hm_bfs": (None, [_i32, _u64]),
    "hm_bfs_array": (_u64p, [_i32, _vp]),
    "hm_bfs_clear": (None, []),
    "audit_store": (_i32, [_vp, _vp, _vp, _u64, _vp, _u32, _u32, _i32, _vp, _u64, _vp, _vp, _vp, _vp, ctypes.c_char_p,
                           ctypes.c_size_t]),
    "audit_violator_rows": (_u64, [_vp, _u64]),
    "hs_create": (_vp, [_u32, _u32]),
    **{fn: (None, [_vp]) for fn in ("hs_destroy", "hs_begin", "hs_seed_init", "hs_reset_cand")},
    "hs_expand": (None, [_vp, _u64, _u64]),
    "hs_counts": (None, [_vp, _vp]),
    "hs_send_ptr": (_i64p, [_vp, _u32]),
    "hs_insert": (None, [_vp, _vp, _u64]),
    "hs_level_done": (None, [_vp, _vp, _vp]),
    "hs_stats": (None, [_vp, _vp]),
    "hs_violation_record": (_i32, [_vp, _vp]),
    "hs_state_and_parent": (None, [_vp, _u64, _vp]),
}
# hm_bfs_array's arrays, in its order
BFS_ARRAYS = ("totals", "states", "parents", "widths", "action_generated", "site_generated", "invariant_first_level",
              "invariant_violators", "mask_first_level", "mask_violators_first_level", "mask_violators", "mask_pick")


def _library_path(header_text: str, invariants_text: str) -> str:
    """host_model.cpp compiled against `header_text` and `invariants_text`; written through pid-unique temporaries, so
    that test processes building the same headers at once never see a partial file."""
    with open(SOURCE) as f:
        tag = hashlib.sha256((header_text + "\0" + invariants_text + "\0" + f.read()).encode()).hexdigest()[:16]
    so = os.path.join(BUILD, f"{tag}.so")
    if not os.path.exists(so):
        os.makedirs(BUILD, exist_ok=True)
        tmp = f".{os.getpid()}.tmp"
        hdr, inv = os.path.join(BUILD, f"{tag}.h"), os.path.join(BUILD, f"{tag}.inv.h")
        for path, text in ((hdr, header_text), (inv, invariants_text)):
            with open(path + tmp, "w") as f:
                f.write(text)
            os.replace(path + tmp, path)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", f'-DKMC_MODEL_HEADER="{hdr}"',
                               f'-DKMC_INVARIANTS_HEADER="{inv}"', SOURCE, "-o", so + tmp])
        os.replace(so + tmp, so)
    return so


@functools.lru_cache(maxsize=None)
def lower_registered(name: str) -> LoweredModel:
    """The registered model `name` (build.registry() or build.device_init_registry()) lowered from its module and cfg
    as build() lowers it, once per process; `lower_registered.__wrapped__(name)` lowers it afresh."""
    spec = {**registry(), **device_init_registry()}[name]
    with open(os.path.join(ROOT, spec["cfg"])) as f:
        return lower_model(spec["module"], tla_search_dirs(), f.read(), name=name)


@functools.lru_cache(maxsize=None)
def _load(so: str) -> ctypes.CDLL:
    lib = ctypes.CDLL(so)
    for fn, (res, args) in SIGNATURES.items():
        getattr(lib, fn).restype = res
        getattr(lib, fn).argtypes = args
    return lib


class HostModel:
    """host_model.cpp compiled against one model's model.h and invariants.h."""

    def __init__(self, name: str, header_text: str, invariants_text: str):
        self.name = name
        self.lib = lib = _load(_library_path(header_text, invariants_text))
        self.words = lib.hm_words()
        self.state_bits = lib.hm_state_bits()
        self.all_ones_possible = bool(lib.hm_all_ones_possible())
        self.symmetry = bool(lib.hm_has_symmetry())
        self.num_actions = lib.hm_num_actions()
        self.num_sites = lib.hm_num_sites()
        self.num_invariants = lib.hm_num_invariants()
        self.num_init = lib.hm_num_init()
        self.check_deadlock = bool(lib.hm_check_deadlock())
        self.digest = lib.hm_digest().decode()
        self.site_action = [lib.hm_site_action(i) for i in range(self.num_sites)]
        self.init_space = [int(lib.hm_init_space(b)) for b in range(lib.hm_init_branches())]   # device form only

    @classmethod
    def from_lowered(cls, model: LoweredModel):
        return cls(model.name, model.header, model.invariants_header)

    @classmethod
    def for_registered(cls, name: str):
        """The headers lower_registered(name) lowers, without build/."""
        return cls.from_lowered(lower_registered(name))

    @classmethod
    def for_built_model(cls, name: str):
        """build/models/<name>/model.h and invariants.h, the headers libkmc_<name>.so was compiled from."""
        d = os.path.join(ROOT, "build", "models", name)
        with open(os.path.join(d, "model.h")) as f, open(os.path.join(d, "invariants.h")) as g:
            h = cls(name, f.read(), g.read())
        with open(os.path.join(d, "model.json")) as f:
            digest = json.load(f)["digest"]
        if h.digest != digest:
            raise AssertionError(f"digest: model.h ({h.digest}) and model.json ({digest}) of {name} disagree")
        return h

    def _state(self, words) -> np.ndarray:
        return np.ascontiguousarray(words, dtype=np.uint64).reshape(self.words)

    def successors(self, state, sites: bool = False) -> tuple[np.ndarray, np.ndarray]:
        """[n, W] successors of one state and their action ids, under expand() or the two-phase form."""
        s = self._state(state)
        cap = 64
        while True:
            out = np.zeros((cap, self.words), dtype=np.uint64)
            act = np.zeros(cap, dtype=np.int32)
            n = self.lib.hm_successors(s.ctypes.data, int(sites), out.ctypes.data, act.ctypes.data, cap)
            if n < 0:
                raise RuntimeError(f"{self.name}: layout trap expanding {[int(x) for x in s]}")
            if n <= cap:
                return out[:n], act[:n]
            cap = n

    def first_violated(self, state) -> int:
        """Index of the first violated invariant, or -1."""
        return self.lib.hm_first_violated(self._state(state).ctypes.data)

    def mask(self, state) -> int:
        """Bit i set iff INVARIANT i is violated (violated_invariants)."""
        return int(self.lib.hm_mask(self._state(state).ctypes.data))

    def in_model(self, state) -> bool:
        return bool(self.lib.hm_in_model(self._state(state).ctypes.data))

    def init_states(self) -> np.ndarray:
        out = np.zeros((self.num_init, self.words), dtype=np.uint64)
        for i in range(self.num_init):
            self.lib.hm_init_state(i, out[i].ctypes.data)
        return out

    def init_candidate(self, branch: int, idx: int) -> tuple[str, np.ndarray | None]:
        """Candidate idx of one branch of the device form of Init: ("solution", its words), ("rejected", None) or
        ("trapped", None) for a solution that does not fit the layout."""
        out = np.zeros(self.words, dtype=np.uint64)
        r = self.lib.hm_init_candidate(branch, idx, out.ctypes.data)
        return ("solution", out) if r > 0 else ("rejected", None) if r == 0 else ("trapped", None)

    def init_solutions(self) -> np.ndarray:
        """[n, W] every generated initial state of either form of Init, duplicates included: the table, or every
        solution of every candidate of every branch in branch and candidate order."""
        cap = 1 << 16
        while True:
            out = np.zeros((cap, self.words), dtype=np.uint64)
            n = ctypes.c_uint64()
            code = self.lib.hm_init_solutions(out.ctypes.data, cap, ctypes.byref(n))
            if code:
                raise RuntimeError(f"{self.name}: an initial state traps the layout (code {code})")
            if n.value <= cap:
                return out[: n.value]
            cap = n.value

    def canonicalize(self, rows: np.ndarray) -> np.ndarray:
        rows = np.ascontiguousarray(rows, dtype=np.uint64).reshape(-1, self.words)
        out = np.empty_like(rows)
        if len(rows):
            self.lib.hm_canonicalize(rows.ctypes.data, len(rows), out.ctypes.data)
        return out

    def bfs(self, sites: bool = False, stop_at: int = 0) -> dict:
        """Level-ordered BFS past violations (see hm_bfs): the store in the engine's format (states in BFS order, parent
        words index | action << 56) and the run's statistics.  Successors come from expand() or, with `sites`, from the
        two-phase form, which also counts them per emit site.  Stops, as incomplete, at the first level end holding
        >= stop_at states (0: never)."""
        self.lib.hm_bfs(int(sites), stop_at)
        r = {}
        for i, key in enumerate(BFS_ARRAYS):
            n = ctypes.c_uint64()
            p = self.lib.hm_bfs_array(i, ctypes.byref(n))
            r[key] = np.ctypeslib.as_array(p, shape=(n.value,)).copy() if n.value else np.zeros(0, dtype=np.uint64)
        self.lib.hm_bfs_clear()
        t = [int(x) for x in r.pop("totals")]
        r["states"] = r["states"].reshape(-1, self.words)
        for key in BFS_ARRAYS[3:]:
            r[key] = [int(x) for x in r[key]]
        r.update(generated=t[0], deadlocks=t[1], fail=t[2], complete=bool(t[3]), n_expanded=t[4], max_fanout=t[5],
                 first_invariant=None if t[6] == M64 else t[6], first_invariant_level=t[7], mask_mismatches=t[8])
        return r

    def invariant_report(self, invariants: list[str]) -> dict:
        """What kmc_invariant_reports reports, from a full host BFS checked through the mask: {invariant name: {level,
        violators_first_level, violators, fingerprint}} of the violated invariants, and the number of checked states
        where the mask and first_violated_invariant disagree (key None)."""
        assert len(invariants) == self.num_invariants
        r = self.bfs()
        if r["fail"]:
            raise RuntimeError(f"{self.name}: layout trap (code {r['fail']}) during the host BFS")
        out = {name: {"level": r["mask_first_level"][i], "violators_first_level": r["mask_violators_first_level"][i],
                      "violators": r["mask_violators"][i], "fingerprint": r["mask_pick"][i]}
               for i, name in enumerate(invariants) if r["mask_first_level"][i]}
        out[None] = r["mask_mismatches"]
        return out


def run_host(model: LoweredModel, max_states: int = 0, dump: bool = False, items: bool = False) -> dict:
    """Full BFS of `model` on the host (through the two-phase form with `items`), stopped at the first level end that
    holds >= max_states states (0: never).  With `dump`, "states" are the canonical identities in BFS order."""
    hm = HostModel.from_lowered(model)
    r = hm.bfs(sites=items, stop_at=max_states)
    res = {
        "distinct": len(r["parents"]), "generated": r["generated"], "depth": len(r["widths"]), "deadlocks": r["deadlocks"],
        "fail": r["fail"], "complete": r["complete"],
        "first_violated": None if r["first_invariant"] is None else model.invariants[r["first_invariant"]],
        "first_violated_level": r["first_invariant_level"], "max_fanout_seen": r["max_fanout"],
        "first_violation_level": {name: (r["invariant_first_level"][i] or None) for i, name in enumerate(model.invariants)},
        "levels": r["widths"],
        "per_action": {a["name"]: r["action_generated"][i] for i, a in enumerate(model.actions)},
    }
    if dump:
        res["states"] = hm.canonicalize(r["states"])
    return res


def site_coverage(model: LoweredModel) -> dict:
    """Full BFS of `model` on the host through the two-phase form the expand kernel runs: successors generated per emit
    site, the sites' actions as compiled into the header (SITE_ACTION), distinct and generated."""
    hm = HostModel.from_lowered(model)
    r = hm.bfs(sites=True)
    if r["fail"]:
        raise RuntimeError(f"{model.name}: layout trap (code {r['fail']}) during the host BFS")
    return {"distinct": len(r["parents"]), "generated": r["generated"], "sites": r["site_generated"],
            "site_action": hm.site_action}
