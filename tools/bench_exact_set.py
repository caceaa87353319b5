"""What exact_set costs: config #5 (asyncisr_deep, 294 million states of three words) with its set keyed by a 128-bit
fingerprint (16-byte slots) against the same set keyed by the packed state (32-byte slots), both in a 2^30-slot table.

    python tools/bench_exact_set.py [--rounds N]

The two configurations alternate, N rounds each, after one warm-up run each; every run is checked bit-exact against
the golden (distinct, generated, depth, per-level widths) before anything is printed.  The --dump-style outputs of the
two are compared on miniwide_w5 (every reachable state, and the state graph) byte for byte.  One JSON line: the median, minimum
and maximum of each configuration's gpu_ms_total, its probes and slot bytes, and the card's name and power limit, read
(not set) in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODEL = "asyncisr_deep"
BASE = {"table_log2": 30, "max_states": 300_000_000}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=30)
    name, power = (x.strip() for x in q.stdout.strip().splitlines()[0].split(","))
    return name, power


def run(opts, golden):
    from kafka_specification_b200.runtime import Checker
    with Checker(MODEL, **opts) as ck:
        r = ck.run()
    got = (r.distinct, r.generated, r.depth, r.levels)
    want = (golden["distinct"], golden["generated"], golden["depth"], golden["levels"])
    if got != want or not r.complete:
        raise SystemExit(f"PARITY FAILURE with {opts}: got {got[:3]}, golden {want[:3]}")
    return r.stats


def dumps_identical():
    from kafka_specification_b200.runtime import Checker
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for exact in (False, True):
            with Checker("miniwide_w5", exact_set=exact, cont=True, table_log2=16) as ck:
                ck.run()
                ck.dump_states(os.path.join(d, f"s{exact}"))
                ck.dump_dot(os.path.join(d, f"d{exact}"), actionlabels=True)
            out[exact] = [open(os.path.join(d, f"{k}{exact}"), "rb").read() for k in ("s", "d")]
    return out[False] == out[True]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    with open(os.path.join(ROOT, "tests", "golden", "goldens.json")) as f:
        golden = json.load(f)[MODEL]
    name, power = card()
    exact_opts = {**BASE, "exact_set": True}
    run(BASE, golden)                                 # warm-up: module load, first touch of the allocations
    run(exact_opts, golden)
    runs = {"default": [], "exact_set": []}
    for _ in range(a.rounds):
        for key, opts in (("default", BASE), ("exact_set", exact_opts)):
            runs[key].append(run(opts, golden))
    summary = {}
    for key, sts in runs.items():
        ms = [s["gpu_ms_total"] for s in sts]
        summary[key] = {"gpu_ms_total_median": round(statistics.median(ms), 1), "gpu_ms_total_min": round(min(ms), 1),
                        "gpu_ms_total_max": round(max(ms), 1), "gpu_ms_total": [round(x, 1) for x in ms],
                        "probes": sts[-1]["probes"], "slot_bytes": sts[-1]["slot_bytes"],
                        "table_slots": sts[-1]["table_slots"]}
    print(json.dumps({
        "model": MODEL, "distinct": golden["distinct"], "parity": "bit-exact vs tests/golden/goldens.json",
        "rounds": a.rounds, **summary,
        "exact_over_default": round(summary["exact_set"]["gpu_ms_total_median"] / summary["default"]["gpu_ms_total_median"], 3),
        "miniwide_w5_dumps_identical": dumps_identical(),
        "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
