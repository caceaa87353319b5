"""Test support: per-emit-site coverage of a lowered model, computed on the host (see host_coverage.cpp)."""
from __future__ import annotations

import ctypes
import hashlib
import os
import subprocess

import numpy as np

from hostmodel import BUILD, HERE


def site_coverage(model) -> dict:
    """Full BFS of ``model`` (a LoweredModel) on the host: successors generated per emit site, the sites' actions
    as compiled into the header (SITE_ACTION), distinct and generated."""
    os.makedirs(BUILD, exist_ok=True)
    src = os.path.join(HERE, "host_coverage.cpp")
    tag = hashlib.sha256((model.header + open(src).read()).encode()).hexdigest()[:16]
    hdr = os.path.join(BUILD, f"cov_{model.name}_{tag}.h")
    so = os.path.join(BUILD, f"cov_{model.name}_{tag}.so")
    if not os.path.exists(so):
        with open(hdr, "w") as f:
            f.write(model.header)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", f'-DKMC_MODEL_HEADER="{hdr}"', src, "-o", so])
    lib = ctypes.CDLL(so)
    n = lib.kmc_cov_num_sites()
    stats = np.zeros(3, dtype=np.uint64)
    sites = np.zeros(max(n, 1), dtype=np.uint64)
    lib.kmc_cov_bfs(ctypes.c_void_p(stats.ctypes.data), ctypes.c_void_p(sites.ctypes.data))
    if stats[2]:
        raise RuntimeError(f"{model.name}: layout trap (code {int(stats[2])}) during the host BFS")
    return {"distinct": int(stats[0]), "generated": int(stats[1]), "sites": [int(x) for x in sites[:n]],
            "site_action": [lib.kmc_cov_site_action(i) for i in range(n)]}
