"""Generates tests/golden/coverage.json -- run after `make -C oracle` (needs oracle/_ref/spec), commit the output.

For every registered model that is not marked "large": successors generated per action and per emit site over a
full BFS (past violations, like -continue), the numbers a GPU run's coverage report must reproduce.

  * per action: Oracle A with its successors labelled by TLC's rule (tests/support/oracle_a_actions.py) where the
    interpreter finishes in seconds; elsewhere the lowered model's own labels, counted by the sequential host
    harness (tests/support/hostmodel.run_host);
  * per site: Oracle A has no emit sites, so these come from the lowered header on the host: the popcount of each
    site_mask bit over the states the host BFS expands (tests/support/host_coverage.py).  Under SYMMETRY these
    depend on which member of each orbit is stored (the first one found here, the insert's winner on the GPU), so
    they are exact only for models without it; per action they are the same either way.

Each entry records its sources.  The large models (10^7..10^8 states, the benchmark's headline among them) are
left out: their coverage is checked on the GPU through sums and run-to-run determinism only.

    python tests/golden/make_coverage.py [model ...]
"""
import json
import os
import sys
from concurrent.futures import ProcessPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests", "support")):
    sys.path.insert(0, p)

# Oracle A finishes these in seconds to a minute on one CPU core
ORACLE_A = ["idsequence", "idsequence_deadlock", "frl_tiny", "kip320_n2", "trunchw_n2", "kip101_n2", "kip279_n2",
            "firsttry_n2", "kip320sym_n2", "asyncisr_v2", "minilock", "minimsgs", "miniqueue", "miniwindow"]


def one(name: str, spec: dict) -> tuple[str, dict]:
    from kafka_specification_b200.build import tla_search_dirs
    from kafka_specification_b200.lower.model import lower_model
    from host_coverage import site_coverage
    from hostmodel import run_host
    cfg_text = open(os.path.join(ROOT, spec["cfg"])).read()
    model = lower_model(spec["module"], tla_search_dirs(), cfg_text, name=name)
    names = [a["name"] for a in model.actions]
    cov = site_coverage(model)
    if name in ORACLE_A:
        from oracle_a_actions import run_bfs_by_action
        r = run_bfs_by_action(spec["module"], tla_search_dirs(), cfg_text)
        unknown = set(r["per_action"]) - set(names)
        if unknown:
            raise SystemExit(f"{name}: Oracle A labels {sorted(unknown)} are not actions of the lowered model {names}")
        per_action, source = {n: r["per_action"].get(n, 0) for n in names}, "oracle_a"
    else:
        r = run_host(model)
        per_action, source = {n: r["per_action"][n] for n in names}, "host_bfs"
    if r["generated"] != cov["generated"]:
        raise SystemExit(f"{name}: generated {r['generated']} ({source}) != {cov['generated']} (host site BFS)")
    return name, {
        "actions": names, "num_init": len(model.init_states), "generated": cov["generated"], "distinct": cov["distinct"],
        "per_action": per_action, "per_action_source": source,
        "per_site": cov["sites"], "site_action": cov["site_action"], "per_site_source": "host_site_mask",
    }


def main():
    reg = json.load(open(os.path.join(ROOT, "models", "MODELS.json")))
    only = sys.argv[1:]
    todo = [(n, s) for n, s in reg.items() if (n in only if only else not s.get("large"))]
    out_path = os.path.join(HERE, "coverage.json")
    out = json.load(open(out_path)) if os.path.exists(out_path) else {}
    with ProcessPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        for name, entry in ex.map(one, *zip(*todo)):
            out[name] = entry
            print(f"{name}: {entry['per_action_source']} {entry['per_action']}", flush=True)
    with open(out_path, "w") as f:
        json.dump({k: out[k] for k in sorted(out)}, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
