"""Test support: host_invariants.cpp compiled against a lowered model.h and its invariants.h (one library per header pair,
under build/hosttest/), and the per-invariant report of its host BFS."""
from __future__ import annotations

import ctypes
import functools
import hashlib
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
BUILD = os.path.join(ROOT, "build", "hosttest")
SOURCE = os.path.join(HERE, "host_invariants.cpp")


@functools.lru_cache(maxsize=None)
def _load(header: str, invariants_header: str) -> ctypes.CDLL:
    with open(SOURCE) as f:
        tag = hashlib.sha256((header + invariants_header + f.read()).encode()).hexdigest()[:16]
    so = os.path.join(BUILD, f"inv_{tag}.so")
    if not os.path.exists(so):
        os.makedirs(BUILD, exist_ok=True)
        tmp = f".{os.getpid()}.tmp"
        paths = []
        for suffix, text in (("h", header), ("inv.h", invariants_header)):
            p = os.path.join(BUILD, f"inv_{tag}.{suffix}")
            with open(p + tmp, "w") as f:
                f.write(text)
            os.replace(p + tmp, p)
            paths.append(p)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", f'-DKMC_MODEL_HEADER="{paths[0]}"',
                               f'-DKMC_INVARIANTS_HEADER="{paths[1]}"', SOURCE, "-o", so + tmp])
        os.replace(so + tmp, so)
    lib = ctypes.CDLL(so)
    lib.hi_mask.restype, lib.hi_mask.argtypes = ctypes.c_uint64, [ctypes.c_void_p]
    lib.hi_first.restype, lib.hi_first.argtypes = ctypes.c_int, [ctypes.c_void_p]
    lib.hi_num_invariants.restype, lib.hi_num_invariants.argtypes = ctypes.c_int, []
    lib.hi_bfs.restype, lib.hi_bfs.argtypes = ctypes.c_int64, [ctypes.c_void_p] * 4
    return lib


class HostInvariants:
    def __init__(self, header: str, invariants_header: str, invariants: list[str]):
        self.lib = _load(header, invariants_header)
        self.invariants = invariants
        assert self.lib.hi_num_invariants() == len(invariants)

    @classmethod
    def from_lowered(cls, model):
        return cls(model.header, model.invariants_header, model.invariants)

    @classmethod
    def for_built_model(cls, name: str, invariants: list[str]):
        d = os.path.join(ROOT, "build", "models", name)
        with open(os.path.join(d, "model.h")) as f, open(os.path.join(d, "invariants.h")) as g:
            return cls(f.read(), g.read(), invariants)

    def mask(self, words) -> int:
        return int(self.lib.hi_mask(np.ascontiguousarray(words, dtype=np.uint64).ctypes.data))

    def first(self, words) -> int:
        return int(self.lib.hi_first(np.ascontiguousarray(words, dtype=np.uint64).ctypes.data))

    def report(self) -> dict:
        """{invariant name: {level, violators_first_level, violators, fingerprint}} of the violated invariants, and the
        number of checked states where the mask and first_violated_invariant disagree (key None)."""
        n = max(len(self.invariants), 1)
        arrs = [np.zeros(n, dtype=np.uint64) for _ in range(4)]
        mismatches = self.lib.hi_bfs(*[a.ctypes.data for a in arrs])
        if mismatches < 0:
            raise RuntimeError("layout trap during the host BFS")
        first_level, first_count, total, pick = arrs
        out = {name: {"level": int(first_level[i]), "violators_first_level": int(first_count[i]),
                      "violators": int(total[i]), "fingerprint": int(pick[i])}
               for i, name in enumerate(self.invariants) if first_level[i]}
        out[None] = int(mismatches)
        return out
