"""Ahead-of-time build: ``.tla`` + ``.cfg``  ->  lowered header  ->  ``libkmc_<model>.so`` (sm_90a).

    python -m kafka_specification_b200.build --all            # every model in models/ and tests/specs/MODELS.json
    python -m kafka_specification_b200.build Kip320 models/Kip320.cfg --name kip320

Artifacts go to ``build/`` (git-ignored):

    build/libkspecmc.so                 the C-ABI dispatcher (include/kspecmc.h)
    build/models/<name>/model.h         the lowered switch table
    build/models/<name>/model.json      layout / actions / invariants (for trace printing)
    build/models/<name>/libkmc_<name>.so

The Kafka specification's ``.tla`` files are not part of this repository.  The lowering searches
``KSPEC_TLA_PATH``, then ``SPEC_DIR`` -- the unchanged, git-ignored copy of the specification's
checkout that ``make -C oracle`` takes -- then the project's own modules in ``models/`` and ``tests/specs/``.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "build")
CSRC = os.path.join(ROOT, "kafka_specification_b200", "csrc")
INCLUDE = os.path.join(ROOT, "include")
MODELS_DIR = os.path.join(ROOT, "models")
TEST_SPECS_DIR = os.path.join(ROOT, "tests", "specs")

NVCC_ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
SPEC_DIR = os.path.join(ROOT, "oracle", "_ref", "spec")


def tla_search_dirs() -> list[str]:
    dirs = []
    env = os.environ.get("KSPEC_TLA_PATH")
    if env:
        dirs += env.split(os.pathsep)
    dirs += [SPEC_DIR, MODELS_DIR, TEST_SPECS_DIR]
    return [d for d in dirs if os.path.isdir(d)]


def nvcc_path() -> str:
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _run(cmd: list[str], log: str | None = None):
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if log:
        with open(log, "w") as f:
            f.write(" ".join(cmd) + "\n" + p.stdout)
    if p.returncode != 0:
        raise RuntimeError(f"command failed ({p.returncode}): {' '.join(cmd)}\n{p.stdout[-4000:]}")
    return p.stdout


def build_dispatcher(force: bool = False) -> str:
    os.makedirs(BUILD, exist_ok=True)
    out = os.path.join(BUILD, "libkspecmc.so")
    src = os.path.join(CSRC, "kspecmc.cpp")
    hdr = os.path.join(INCLUDE, "kspecmc.h")
    if not force and os.path.exists(out) and os.path.getmtime(out) >= max(os.path.getmtime(src), os.path.getmtime(hdr)):
        return out
    _run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", f"-I{INCLUDE}", src, "-o", out, "-ldl"])
    return out


def model_dir(name: str) -> str:
    return os.path.join(BUILD, "models", name)


def model_lib_path(name: str) -> str:
    return os.path.join(model_dir(name), f"libkmc_{name}.so")


def _engine_stamp() -> str:
    h = hashlib.sha256()
    for p in (os.path.join(CSRC, "kmc_engine.cu"), os.path.join(INCLUDE, "kspecmc.h")):
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()[:16]


def lower_to_dir(module: str, cfg_path: str, name: str):
    """Lower and write model.h / model.json; returns the LoweredModel."""
    import time
    from .lower.model import lower_model
    with open(cfg_path) as f:
        cfg_text = f.read()
    t0 = time.time()
    m = lower_model(module, tla_search_dirs(), cfg_text, name=name)
    lower_seconds = time.time() - t0
    d = model_dir(name)
    os.makedirs(d, exist_ok=True)
    hdr = os.path.join(d, "model.h")
    old = open(hdr).read() if os.path.exists(hdr) else None
    if old != m.header:
        with open(hdr, "w") as f:
            f.write(m.header)
    meta = m.meta()
    meta["cfg"] = os.path.relpath(cfg_path, ROOT)
    meta["lower_seconds"] = round(lower_seconds, 2)      # parse + lower on the build host (part of a cold start)
    with open(os.path.join(d, "model.json"), "w") as f:
        json.dump(meta, f, indent=1)
    return m


def _nvcc_cmd(hdr: str, out_so: str) -> list[str]:
    """nvcc of the engine with a lowered header.  The engine runs the two-phase form of the lowered Next only, so
    -DKMC_NO_ONE_PHASE drops the one-phase form from the translation unit (it would only add nvcc time)."""
    return [nvcc_path(), *NVCC_ARCH, "-lineinfo", "-O3", "-std=c++17", "-shared", "-Xcompiler", "-fPIC",
            "-diag-suppress", "177", "-DKMC_NO_ONE_PHASE",
            f"-I{INCLUDE}", "-include", hdr, os.path.join(CSRC, "kmc_engine.cu"), "-o", out_so]


def compile_model(name: str, force: bool = False, verbose_ptxas: bool = True) -> str:
    d = model_dir(name)
    hdr = os.path.join(d, "model.h")
    so = model_lib_path(name)
    stamp_file = os.path.join(d, "build.stamp")
    with open(hdr, "rb") as f:
        stamp = hashlib.sha256(f.read()).hexdigest()[:16] + ":" + _engine_stamp()
    if not force and os.path.exists(so) and os.path.exists(stamp_file) and open(stamp_file).read() == stamp:
        return so
    cmd = _nvcc_cmd(hdr, so)
    if verbose_ptxas:
        cmd[1:1] = ["-Xptxas", "-v"]
    import time
    t0 = time.time()
    log = os.path.join(d, "nvcc.log")
    _run(cmd, log=log)
    with open(log, "a") as f:
        f.write(f"nvcc wall time: {time.time() - t0:.1f} s\n")
    with open(stamp_file, "w") as f:
        f.write(stamp)
    return so


def compile_model_to(name: str, out_so: str) -> str:
    """Plain nvcc of the prebuilt lowered header into `out_so` (no stamp, no log): the cold-start timing of bench.py."""
    _run(_nvcc_cmd(os.path.join(model_dir(name), "model.h"), out_so))
    return out_so


def build_model(module: str, cfg_path: str, name: str, force: bool = False) -> str:
    """Lower (when the .tla sources are reachable) and compile; returns the library path."""
    have_sources = any(os.path.exists(os.path.join(d, module + ".tla")) for d in tla_search_dirs())
    if have_sources:
        lower_to_dir(module, cfg_path, name)
    elif not os.path.exists(os.path.join(model_dir(name), "model.h")):
        raise RuntimeError(f"{module}.tla is not reachable and build/models/{name}/model.h was not prebuilt")
    return compile_model(name, force=force)


def registry() -> dict:
    """Every model build_all() compiles: the project's models (models/MODELS.json) and the models that exist only to
    test the engine (tests/specs/MODELS.json, specs kept with the tests; absent from a tree without the test suite)."""
    with open(os.path.join(MODELS_DIR, "MODELS.json")) as f:
        reg = json.load(f)
    test_registry = os.path.join(TEST_SPECS_DIR, "MODELS.json")
    if not os.path.exists(test_registry):
        return reg
    with open(test_registry) as f:
        test_models = json.load(f)
    clash = set(reg) & set(test_models)
    if clash:
        raise RuntimeError(f"models registered twice: {sorted(clash)}")
    return {**reg, **test_models}


def build_all(force: bool = False, only: list[str] | None = None, verbose: bool = True, jobs: int = 0) -> dict[str, str]:
    """Lower (sequentially, it is fast) and compile (in parallel: nvcc dominates) every registered model."""
    from concurrent.futures import ThreadPoolExecutor
    build_dispatcher(force)
    todo = []
    for name, spec in registry().items():
        if only and name not in only:
            continue
        module, cfg_path = spec["module"], os.path.join(ROOT, spec["cfg"])
        have_sources = any(os.path.exists(os.path.join(d, module + ".tla")) for d in tla_search_dirs())
        if have_sources:
            lower_to_dir(module, cfg_path, name)
        elif not os.path.exists(os.path.join(model_dir(name), "model.h")):
            raise RuntimeError(f"{module}.tla is not reachable and build/models/{name}/model.h was not prebuilt")
        todo.append(name)
    jobs = jobs or min(8, os.cpu_count() or 1)

    def one(name):
        so = compile_model(name, force=force)
        if verbose:
            print(f"[build] {name}: {so}", flush=True)
        return name, so

    with ThreadPoolExecutor(max_workers=jobs) as ex:
        return dict(ex.map(one, todo))


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("module", nargs="?")
    ap.add_argument("cfg", nargs="?")
    ap.add_argument("--name")
    ap.add_argument("--all", action="store_true")
    ap.add_argument("--force", action="store_true")
    a = ap.parse_args(argv)
    if a.all or not a.module:
        for n, p in build_all(force=a.force).items():
            print(n, p)
        return 0
    build_dispatcher(a.force)
    name = a.name or a.module
    print(build_model(a.module, a.cfg, name, force=a.force))
    return 0


if __name__ == "__main__":
    sys.exit(main())
