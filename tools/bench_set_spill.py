"""What set_spill costs on the headline model: Kip320 R4E3 (340 million states) through a 2^27-slot table (2^26 keys per
epoch, so several flushes, some in the middle of a level) against the default sizing, which holds every key in HBM.

    python tools/bench_set_spill.py [--rounds N]

The two configurations alternate, N rounds each (other work shares the host); every run is checked bit-exact against
the golden (distinct, generated, depth, per-level widths) before anything is printed.  One JSON line: the median of
each configuration's gpu_ms_total, set_spill's flush and filter time (gpu_ms_set_spill, CUDA events), its flushes, the
keys in host memory, the key bytes moved over the host link, and the card's name and power limit, read (not set) in
the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODEL = "kip320_3x4_r4e3"
SET_SPILL = {"table_log2": 27, "max_states": 350_000_000, "set_spill": True}


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


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    with open(os.path.join(ROOT, "tests", "golden", "goldens.json")) as f:
        golden = json.load(f)[MODEL]
    name, power = card()
    spill, default = [], []
    run(SET_SPILL, golden)                       # warm-up: module load, first-touch of host memory
    for _ in range(a.rounds):
        spill.append(run(SET_SPILL, golden))
        default.append(run({}, golden))
    med = lambda runs, k: statistics.median(s[k] for s in runs)
    s = spill[-1]
    print(json.dumps({
        "model": MODEL, "distinct": golden["distinct"], "parity": "bit-exact vs tests/golden/goldens.json",
        "rounds": a.rounds,
        "set_spill": {"table_slots": s["table_slots"], "gpu_ms_total": med(spill, "gpu_ms_total"),
                      "gpu_ms_set_spill": med(spill, "gpu_ms_set_spill"), "set_flushes": s["set_flushes"],
                      "set_host_keys": s["set_host_keys"], "set_filtered": s["set_filtered"],
                      "host_link_bytes": s["set_link_bytes"], "wall_ms": med(spill, "wall_ms")},
        "default": {"table_slots": default[-1]["table_slots"], "gpu_ms_total": med(default, "gpu_ms_total"),
                    "wall_ms": med(default, "wall_ms")},
        "gpu": name, "power_limit": power,
    }))


if __name__ == "__main__":
    main()
