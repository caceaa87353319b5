"""``tlc2.TLC``-compatible command line on top of the C ABI.

    python -m kafka_specification_b200.tlc2 [-config F.cfg] [-workers N|auto] [-deadlock] [-continue]
                                             [-fpbits N] [-maxstates N] [-I dir] [-metadir d] [-checkpoint MIN]
                                             [-recover DIR] [-spill] [-setspill] [-exactset] [-coverage N] [-tool]
                                             [-dump FILE | -dump dot[,actionlabels][,colorize][,snapshot] FILE] SPEC

``SPEC`` is a module name or a path to ``SPEC.tla``; modules it EXTENDS / INSTANCEs are resolved
from the same directory (and ``-I`` directories), like TLC does.  The spec and its ``.cfg`` are
lowered ahead of time into a CUDA switch table (cached under ``build/models/``), the BFS runs on
the GPU through ``libkspecmc.so``, and the summary / error trace are printed in TLC's format.
``-workers N`` selects N GPUs of this machine (fingerprint-sharded inside the library, option ``"gpus": N`` of
kmc_create); ``-workers auto`` = one GPU (the GPU grid replaces TLC's worker threads).  ``-tool`` wraps the
messages in TLC's tool-mode markers (``@!@!@STARTMSG code:class @!@!@`` ... ``@!@!@ENDMSG code @!@!@``).
``-coverage N`` prints TLC's action-level coverage table ("distinct:generated" per action) once, at the end of the
run (also after a violation): TLC repeats it every N minutes, but a search here takes seconds.
``-setspill`` (an extension, like ``-spill``) moves the fingerprint set's keys to host memory whenever its table fills,
so that a state space larger than the table still finishes (one GPU; see ``set_spill`` in include/kspecmc.h).
``-exactset`` (an extension as well) keys the fingerprint set by the packed state itself instead of a hashed
fingerprint, so that "No error has been found" is exact on every model (one GPU; see ``exact_set`` in
include/kspecmc.h); the collision estimate is then 0.  Models whose key is exact already are unchanged by it.
``-continue`` searches past violations and prints one error block per violated invariant, ordered by (first violating
level, cfg index), each with the counterexample that ends in the smallest-fingerprint violator of that level; the first
block is the one a run without ``-continue`` prints.  TLC under ``-continue`` prints a trace for every violating state
it meets (as far as its published behaviour goes: TLC cannot be run here to compare); here it is one per invariant.
A deadlock found on the way keeps its block and its exit status, ahead of the invariant blocks.
``-dump FILE`` writes every reachable state to ``FILE.dump``; ``-dump dot,... FILE`` writes the state graph, its
transitions enumerated on the GPU, to ``FILE.dot`` (one GPU; see ``dump.py`` for the layouts and how they differ from
TLC's).  The file is written once, at the end of the run, after a violation too; ``snapshot`` is accepted and ignored.

Exit status follows TLC: 0 no error, 12 safety (invariant) violation, 11 deadlock,
10 assumption failure, 150 spec/config error, 1 runtime failure (no GPU, table full, ...).
"""
from __future__ import annotations

import argparse
import hashlib
import math
import os
import re
import sys
import time

from . import build as B
from .frontend.cfg import CfgError
from .frontend.modules import ModuleError
from .frontend.tla_lexer import TlaSyntaxError
from .lower.svals import LowerError
from .dump import split_dump_args
from .runtime import Checker, KmcError

EXIT_OK, EXIT_VIOLATION_ASSUMPTION, EXIT_VIOLATION_DEADLOCK, EXIT_VIOLATION_SAFETY, EXIT_ERROR_SPEC = 0, 10, 11, 12, 150


def parse_args(argv):
    ap = argparse.ArgumentParser(prog="tlc2.TLC", add_help=True, prefix_chars="-")
    ap.add_argument("-config")
    ap.add_argument("-workers", default="auto")
    ap.add_argument("-deadlock", action="store_true", help="do NOT check for deadlock (TLC semantics)")
    ap.add_argument("-continue", dest="cont", action="store_true")
    ap.add_argument("-fpbits", type=int, default=0, help="log2 of the fingerprint-set slots")
    ap.add_argument("-maxstates", type=int, default=0)
    ap.add_argument("-I", action="append", default=[])
    ap.add_argument("-metadir", help="directory for checkpoints (TLC: states/<timestamp>)")
    ap.add_argument("-checkpoint", type=float, default=None, help="minutes between checkpoints (TLC default 30; 0 = every level)")
    ap.add_argument("-recover", help="resume from the checkpoint in this directory")
    ap.add_argument("-spill", action="store_true",
                    help="extension: keep only the live BFS window in HBM and move older levels to host memory")
    ap.add_argument("-setspill", action="store_true",
                    help="extension: move the fingerprint set's keys to host memory whenever its HBM table fills")
    ap.add_argument("-exactset", action="store_true",
                    help="extension: key the fingerprint set by the packed state itself (no fingerprint collisions)")
    ap.add_argument("-tool", action="store_true")
    ap.add_argument("-device", type=int, default=0)
    ap.add_argument("-cleanup", action="store_true")
    ap.add_argument("-nowarning", action="store_true")
    ap.add_argument("-fp", type=int, default=0)
    ap.add_argument("-fpmem", type=float, default=0)
    ap.add_argument("-coverage", type=int, default=0, help="print the coverage table at the end of the run (N > 0)")
    ap.add_argument("spec")
    return ap.parse_args(argv)


# TLC's -tool mode wraps every message as  @!@!@STARTMSG <code>:<class> @!@!@ / text / @!@!@ENDMSG <code> @!@!@
# (class 0 = info, 1 = error, 4 = a state of an error trace).  The codes are those of TLC's tlc2.output.EC as
# published (TLC is not in the reference tree and cannot run here, so they are reproduced, not verified).
EC = {"version": 2262, "mode": 2187, "sany_start": 2220, "sany_end": 2219, "starting": 2185, "init": 2189,
      "init_done": 2190, "inv_initial": 2107, "inv_behavior": 2110, "deadlock": 2114, "behavior": 2121,
      "state": 2217, "success": 2193, "collision": 2201, "stats": 2199, "depth": 2194, "finished": 2186,
      "general": 1000,
      # coverage (TLC >= 1.7, action level).  TLC publishes 2201 for the start of the coverage report; the entry
      # "collision" above already uses 2201, and both are kept as they are.
      "coverage_start": 2201, "coverage_init": 2772, "coverage_next": 2773, "coverage_end": 2202}
_TOOL = False


def msg(kind: str, text: str, cls: int = 0):
    if _TOOL:
        code = EC[kind]
        print(f"@!@!@STARTMSG {code}:{cls} @!@!@\n{text}\n@!@!@ENDMSG {code} @!@!@")
    else:
        print(text)


def collision_probability(distinct: int, generated: int) -> float:
    """TLC's 'calculated (optimistic)' estimate: n * (g - n) / 2^64."""
    return distinct * max(generated - distinct, 1) / 2.0 ** 64


def action_location(a: dict | None) -> str:
    if a is None:
        return "<Initial predicate>"
    if "line" in a and a.get("end_line"):
        return (f"<{a['name']} line {a['line']}, col {a['col']} to line {a['end_line']}, col {a['end_col']} "
                f"of module {a['module']}>")
    return f"<{a['name']} of module {a.get('module', '?')}>"


def coverage_lines(cov: dict, when: str) -> list[tuple[str, str]]:
    """(EC kind, text) of TLC's coverage report for a ``Checker.coverage()`` dict: the initial predicate, then one
    line per action in model.json order (actions that never fired included, as 0:0)."""
    def loc(a):
        return action_location({"name": a["name"], "module": a.get("module") or "?", **a.get("location", {})})
    init = cov["init"]
    out = [("coverage_start", f"The coverage statistics at {when}"),
           ("coverage_init", f"{action_location(init)}: {init['distinct']}:{init['generated']}")]
    out += [("coverage_next", f"{loc(a)}: {a['distinct']}:{a['generated']}") for a in cov["actions"]]
    out.append(("coverage_end", "End of statistics."))
    return out


def print_coverage(cov: dict):
    if not cov["complete"]:
        msg("general", "Warning: the run recovered from a checkpoint without per-site counts; the generated counts "
                       "below cover only the levels searched since.")
    for kind, text in coverage_lines(cov, time.strftime("%Y-%m-%d %H:%M:%S")):
        msg(kind, text)


def trace_messages(trace: list[dict]) -> list[tuple[str, str, int]]:
    return [("state", f"State {i + 1}: {action_location(t['action'])}\n{t['text']}\n", 4) for i, t in enumerate(trace)]


def invariant_messages(name: str, level: int, trace: list[dict]) -> list[tuple[str, str, int]]:
    """TLC's error block of one violated invariant: (EC kind, text, class) per message."""
    if level == 1:
        head = [("inv_initial", f"Error: Invariant {name} is violated by the initial state:", 1)]
    else:
        head = [("inv_behavior", f"Error: Invariant {name} is violated.", 1),
                ("behavior", "Error: The behavior up to this point is:", 1)]
    return head + trace_messages(trace)


def error_messages(violation: dict | None, trace: list[dict], reports: list[dict]) -> tuple[list[tuple[str, str, int]], int]:
    """The error blocks of a run and its exit status.  `violation` / `trace`: the run's first violation (RunResult);
    `reports`: its per-invariant reports under -continue (RunResult.invariant_violations, empty otherwise), whose
    first block is the one of `violation` when that is an invariant violation."""
    out, code = [], EXIT_OK
    if violation and violation["kind"] == "deadlock":
        out = [("deadlock", "Error: Deadlock reached.", 1), ("behavior", "Error: The behavior up to this point is:", 1)]
        out += trace_messages(trace)
        code = EXIT_VIOLATION_DEADLOCK
    elif violation and not reports:
        out = invariant_messages(violation["invariant"], violation["level"], trace)
    for r in sorted(reports, key=lambda r: (r["level"], r["index"])):
        out += invariant_messages(r["invariant"], r["level"], r["trace"])
    if code == EXIT_OK and (violation or reports):
        code = EXIT_VIOLATION_SAFETY
    return out, code


def write_dump(ck: Checker, req) -> None:
    if req.dot:
        ck.dump_dot(req.path, actionlabels=req.actionlabels, colorize=req.colorize)
    else:
        ck.dump_states(req.path)


def main(argv=None) -> int:
    try:
        argv, dump_req = split_dump_args(list(argv if argv is not None else sys.argv[1:]))
    except ValueError as e:
        print(f"Error: {e}")
        return EXIT_ERROR_SPEC
    a = parse_args(argv)
    spec_path = a.spec[:-4] if a.spec.endswith(".tla") else a.spec
    spec_dir = os.path.dirname(os.path.abspath(spec_path)) if os.path.dirname(spec_path) else os.getcwd()
    module = os.path.basename(spec_path)
    cfg_path = a.config or os.path.join(spec_dir, module + ".cfg")
    if not cfg_path.endswith(".cfg"):
        cfg_path += ".cfg"
    t0 = time.time()
    global _TOOL
    _TOOL = bool(a.tool)
    msg("version", "TLC2-compatible front end of kspec-mc (H100-native explicit-state model checker)")
    try:
        n_gpus = 1 if a.workers == "auto" else max(1, int(a.workers))
    except ValueError:
        print(f"Error: -workers takes a number or auto, not {a.workers!r}")
        return EXIT_ERROR_SPEC
    msg("mode", f"Running breadth-first search Model-Checking on {n_gpus} GPU{'s' if n_gpus > 1 else ''} "
                f"(-workers {a.workers}).")
    try:
        cfg_text = open(cfg_path).read()
    except OSError as e:
        print(f"Error: cannot read the configuration file {cfg_path}: {e}")
        return EXIT_ERROR_SPEC
    os.environ["KSPEC_TLA_PATH"] = os.pathsep.join([spec_dir] + a.I + [os.environ.get("KSPEC_TLA_PATH", "")]).strip(os.pathsep)
    name = re.sub(r"[^A-Za-z0-9_]", "_", module).lower() + "_" + hashlib.sha256(cfg_text.encode()).hexdigest()[:10]
    try:
        msg("sany_start", f"Parsing file {os.path.join(spec_dir, module + '.tla')}")
        model = B.lower_to_dir(module, cfg_path, name)
        for w in model.warnings:
            if not a.nowarning:
                print(f"Warning: {w}")
        msg("sany_end", f"Semantic processing of module {module}")
        B.build_dispatcher()
        B.compile_model(name)
    except (TlaSyntaxError, ModuleError, CfgError) as e:
        msg("general", f"Error: {e}", 1)
        return EXIT_ERROR_SPEC
    except LowerError as e:
        text = str(e)
        msg("general", f"Error: {text}", 1)
        return EXIT_VIOLATION_ASSUMPTION if "ASSUME" in text else EXIT_ERROR_SPEC
    msg("starting", f"Starting... ({time.strftime('%Y-%m-%d %H:%M:%S')})")
    opts = {"device": a.device}
    if n_gpus > 1:
        opts["gpus"] = n_gpus
    if a.fpbits:
        opts["table_log2"] = a.fpbits
    if a.maxstates:
        opts["max_states"] = a.maxstates
    if a.cont:
        opts["cont"] = True
    if a.deadlock:
        opts["check_deadlock"] = False
    if a.metadir or a.checkpoint is not None:
        ckdir = a.metadir or os.path.join("states", time.strftime("%y-%m-%d-%H-%M-%S"))
        os.makedirs(ckdir, exist_ok=True)
        opts["checkpoint_dir"] = ckdir
        opts["checkpoint_minutes"] = 30.0 if a.checkpoint is None else a.checkpoint
    if a.recover:
        opts["recover"] = a.recover
    if a.spill:
        opts["spill"] = True
    if a.setspill:
        opts["set_spill"] = True
    if a.exactset:
        opts["exact_set"] = True
    try:
        ck = Checker(name, **opts)
    except KmcError as e:
        msg("general", f"Error: {e}", 1)
        return 1
    msg("init", "Computing initial states...")
    try:
        r = ck.run(raise_on_error=False)
        st = r.stats
        if ck.last_rc != 0:
            print(f"Error: {ck.error_text(ck.last_rc)}")
            return 1
    except KmcError as e:
        msg("general", f"Error: {e}", 1)
        return 1
    n_init = len(model.init_states)
    if model.init.get("device"):
        # the device form of Init has no table: the initial states are level 1 of the run (all of the states found
        # when the run stopped in level 1)
        n_init = r.levels[0] if r.levels else r.distinct
    msg("init_done", f"Finished computing initial states: {n_init} distinct state{'s' if n_init != 1 else ''} generated.")
    blocks, exit_code = error_messages(r.violation, r.trace, r.invariant_violations)
    if dump_req is not None:
        try:
            write_dump(ck, dump_req)
        except (KmcError, OSError) as e:
            msg("general", f"Error: cannot write {dump_req.path}: {e}", 1)
            return 1
    for kind, text, cls in blocks:
        msg(kind, text, cls)
    if not blocks:
        msg("success", "Model checking completed. No error has been found.\n"
                       "  Estimates of the probability that TLC did not check all reachable states\n"
                       "  because two distinct states had the same fingerprint:")
        if a.exactset and ck.info.exact:
            msg("collision", "  calculated (optimistic):  val = 0 (exact: the set key is the packed state)")
        elif ck.info.exact:
            msg("collision", "  calculated (optimistic):  val = 0 (the set key is a bijection of the packed state: exact)")
        else:
            p128 = collision_probability(r.distinct, r.generated) / 2.0 ** 65
            msg("collision", f"  calculated (optimistic):  val = {p128:.1E} (128-bit fingerprints)")
    if a.coverage > 0:
        print_coverage(ck.coverage())
    msg("stats", f"{r.generated} states generated, {r.distinct} distinct states found, {r.queue} states left on queue.")
    if r.complete:
        msg("depth", f"The depth of the complete state graph search is {r.depth}.")
    dt = time.time() - t0
    msg("finished", f"Finished in {int(dt // 60):02d}min {int(dt % 60):02d}s at ({time.strftime('%Y-%m-%d %H:%M:%S')}); "
                    f"GPU search time {st['gpu_ms_total']:.1f} ms "
                    f"({r.distinct / max(st['gpu_ms_total'], 1e-6) * 1000:.3g} distinct states/s)")
    ck.close()
    return exit_code


if __name__ == "__main__":
    sys.exit(main())
