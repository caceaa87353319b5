"""What the device form of Init costs: FiniteReplicatedLog's type as an Init (frl_typeinit_3x4x3: 1280^3 =
2,097,152,000 candidate assignments, 1,771,561 solutions) against the same state space searched from the table
model's one initial state (frl_3x4x3, 13 levels).

    python tools/bench_device_init.py [--rounds N] [--out DIR]

The two models alternate, N rounds each after one warm-up run of each (other work shares the host); every run is
checked against the closed form before anything is printed.  One JSON line: the medians of k_init's time
(gpu_ms_init, CUDA events around its launches), candidates per second over that time, the whole run (gpu_ms_total)
of both models, and the card's name and power limit, read (not set) in the same run.  With --out the line is also
written to DIR/bench_device_init.json.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEVICE, TABLE = "frl_typeinit_3x4x3", "frl_3x4x3"
CANDIDATES, STATES = 1280 ** 3, 121 ** 3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=30)
    name, power = (x.strip() for x in q.stdout.strip().splitlines()[0].split(","))
    return name, power


def run(model):
    from kafka_specification_b200.runtime import Checker
    with Checker(model, table_log2=23) as ck:
        r = ck.run()
    if r.distinct != STATES or not r.complete:
        raise SystemExit(f"PARITY FAILURE on {model}: {r.distinct} distinct states, complete {r.complete}")
    if model == DEVICE and (r.init_candidates != CANDIDATES or r.init_generated != STATES or r.levels != [STATES]):
        raise SystemExit(f"PARITY FAILURE on {model}: {r.init_candidates} candidates, {r.init_generated} solutions")
    return r.stats


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", help="also write the line to DIR/bench_device_init.json")
    a = ap.parse_args()
    name, power = card()
    run(DEVICE), run(TABLE)                                  # warm-up: module loads, first allocations
    dev, tab = [], []
    for _ in range(a.rounds):
        dev.append(run(DEVICE))
        tab.append(run(TABLE))
    med = lambda xs, k: statistics.median(x[k] for x in xs)  # noqa: E731
    ms_init = med(dev, "gpu_ms_init")
    out = {"model": DEVICE, "candidates": CANDIDATES, "solutions": STATES, "rounds": a.rounds,
           "k_init_ms": round(ms_init, 3), "candidates_per_s": round(CANDIDATES / (ms_init / 1e3)),
           "k_init_ms_spread": [round(min(x["gpu_ms_init"] for x in dev), 3), round(max(x["gpu_ms_init"] for x in dev), 3)],
           "device_init_run_ms": round(med(dev, "gpu_ms_total"), 3),
           "table_model": TABLE, "table_run_ms": round(med(tab, "gpu_ms_total"), 3),
           "gpu": name, "power_limit": power}
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_device_init.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
