"""Generates tests/golden/goldens.json -- run after `make -C oracle` (needs oracle/_ref/spec), commit the output.

For every registered model (models/MODELS.json and the test-only tests/specs/MODELS.json):
  * Oracle B (oracle/kspec_oracle.c, hand-written C restatement) runs the full BFS;
  * if the entry is marked "oracle_a", Oracle A (oracle/tla_interp.py, direct interpreter of the
    unchanged .tla text) runs it too, and both must agree on distinct / generated / depth /
    per-level widths / deadlocks / per-invariant first-violation level;  Oracle A also provides a
    digest of the set of reachable states (canonical TLC-style text), which the lowered model must
    reproduce state for state, and the number of states a CONSTRAINT discards (out_of_model: initial
    states and every generation of a successor);
  * analytic closed forms (IdSequence, FiniteReplicatedLog) are asserted where they exist.
The reference ships no goldens of its own (parity unpinned, see oracle/tla_interp.py).
"""
import hashlib
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import kso  # noqa: E402
import tla_interp  # noqa: E402
from kafka_specification_b200.frontend.cfg import parse_cfg  # noqa: E402


def state_digest(texts) -> str:
    """Order-independent digest of a set of canonical state texts."""
    acc = 0
    for t in texts:
        acc = (acc + int.from_bytes(hashlib.sha256(t.encode()).digest()[:8], "little")) % (1 << 64)
    return f"{acc:016x}"


def closed_form(module, cfg):
    c = cfg.constants
    if module == "IdSequence":
        n = c["MaxId"] + 2
        return {"distinct": n, "generated": n, "depth": n}
    if module == "FiniteReplicatedLog":
        nrep, L, R = len(c["Replicas"]), c["LogSize"], len(c["LogRecords"])
        return {"distinct": sum(R ** e for e in range(L + 1)) ** nrep, "depth": nrep * L + 1}
    if module == "MiniWide" and c["Max"] == 1 and not cfg.symmetry:
        return miniwide_closed_form(len(c["Procs"]) * c["Slots"], c["Budget"], c["Limit"], cfg.invariants)
    return {}


def miniwide_closed_form(n, budget, limit, invariants):
    """MiniWide with Max = 1 over n cells: a state is its set of full cells, one more per step, so level i + 1 holds the
    C(n, i) states with i full cells, up to the Budget of the CONSTRAINT.  Each state with i full cells generates n - i
    successors; those of the last level all have Budget + 1 full cells and are discarded (and no deadlock).  FewFull
    (fewer than Limit full cells, Limit <= Budget) is first violated at level Limit + 1 by C(n, Limit) states, and
    violated by every later state and every discarded successor."""
    from math import comb
    b = min(budget, n)
    assert limit <= b, "the closed form covers a Limit the stored states reach"
    levels = [comb(n, i) for i in range(b + 1)]
    out = comb(n, b) * (n - b)
    return {"distinct": sum(levels), "levels": levels, "depth": b + 1,
            "generated": 1 + sum(comb(n, i) * (n - i) for i in range(b + 1)),
            "deadlocks": 1 if b == n else 0, "out_of_model": out,
            "first_violation_level": {inv: limit + 1 if inv == "FewFull" else None for inv in invariants},
            "violators_first_level": {"FewFull": comb(n, limit)},
            "violating_states": {inv: sum(levels[limit:]) + out if inv == "FewFull" else 0 for inv in invariants}}


def main():
    from kafka_specification_b200.build import registry
    reg = registry()
    only = sys.argv[1:]
    out_path = os.path.join(HERE, "goldens.json")
    out = json.load(open(out_path)) if os.path.exists(out_path) else {}
    for name, spec in reg.items():
        if only and name not in only:
            continue
        if spec.get("large") and name not in only:
            continue                    # minutes of CPU and tens of GB: only when asked for by name
        cfg_text = open(os.path.join(ROOT, spec["cfg"])).read()
        cfg = parse_cfg(cfg_text)
        t0 = time.time()
        dirs = [os.path.join(ROOT, "oracle", "_ref", "spec"), os.path.join(ROOT, "models"), os.path.join(ROOT, "tests", "specs")]
        if "kso" in spec:
            model, params = spec["kso"]
            b = kso.run(model, params, max_states=spec.get("max_states", 4_000_000), invariants=cfg.invariants,
                        symmetry=bool(spec.get("symmetry")))
            src = ["oracle_b"]
        else:
            # a spec Oracle B has no hand-written restatement of (synthetic front-end tests): Oracle A alone
            b = tla_interp.run_bfs(spec["module"], dirs, cfg_text + "\nCHECK_DEADLOCK FALSE\n", stop_on_violation=False)
            src = []
        g = {"module": spec["module"], "cfg": spec["cfg"], "kso": spec.get("kso"), "symmetry": bool(spec.get("symmetry")),
             "distinct": b["distinct"], "generated": b["generated"], "depth": b["depth"], "levels": b["levels"],
             "deadlocks": b["deadlocks"], "first_violation_level": b["first_violation_level"],
             "check_deadlock": cfg.check_deadlock, "sources": src}
        if spec.get("oracle_a"):
            # full-space statistics: never stop at a violation, deadlock checking off
            stats_cfg = cfg_text + "\nCHECK_DEADLOCK FALSE\n"
            a = tla_interp.run_bfs(spec["module"], dirs, stats_cfg, collect_states=True, stop_on_violation=False)
            for k in ("distinct", "generated", "depth", "levels", "deadlocks"):
                assert a[k] == g[k], (name, k, a[k], g[k])
            for inv, lvl in b["first_violation_level"].items():
                assert a["first_violation_level"].get(inv) == lvl, (name, inv, a["first_violation_level"], lvl)
            g["first_violation_level"] = a["first_violation_level"]     # includes TypeOk
            g["out_of_model"] = a["out_of_model"]
            if not spec.get("symmetry"):       # under SYMMETRY the choice of orbit representatives is free
                g["state_digest"] = state_digest(a["states"])
            g["sources"].append("oracle_a")
        cf = closed_form(spec["module"], cfg)
        for k, v in cf.items():
            if k in g:
                assert g[k] == v, (name, k, g[k], v)
        if cf and spec.get("oracle_a") and "violating_states" in cf:
            assert a["violating_states"] == cf["violating_states"], (name, a["violating_states"])
        if cf:
            g["sources"].append("closed_form")
        out[name] = g
        print(f"{name}: distinct={g['distinct']} generated={g['generated']} depth={g['depth']} "
              f"viol={g['first_violation_level']} sources={g['sources']} ({time.time() - t0:.1f}s)", flush=True)
        with open(out_path, "w") as f:
            json.dump(out, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
