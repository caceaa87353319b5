"""What TLC's -dump costs, and that it costs the search nothing.

    python tools/bench_dump.py [--parent TREE] [--rounds N] [--steps K] [--warmup W] [--dump-stop N]

* The headline ``bench.py`` line (Kip320 R4E3, one GPU), alternated N rounds with the same command in ``--parent``, a
  checkout of the commit before kmc_edges with its dispatcher and headline model built: the expand and insert kernels
  are unchanged, so the two must agree.
* kmc_edges over every expanded state of the headline store, edges counted and discarded (cap = 0: nothing crosses
  the host link but the per-chunk counts), host clock around the call (it ends in a stream synchronisation), checked
  against generated - init_generated - out_of_model.
* dump_states: wall time, and its split into decoding and writing, for kip320_small and for the headline model stopped
  at its first level end with >= --dump-stop states (the whole headline dump is ~10^11 bytes of text).

One JSON line, with the card's name, power limit and SM clock limit, read (not set) in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODEL = "kip320_3x4_r4e3"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=30)
    return [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]


def bench_line(tree, steps, warmup):
    p = subprocess.run([sys.executable, "bench.py", "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup),
                        "--no-cold", "--no-cpu-baseline"], cwd=tree, capture_output=True, text=True, timeout=3000)
    lines = [l for l in p.stdout.splitlines() if l.startswith("{")]
    if p.returncode or not lines:
        raise SystemExit(f"bench.py in {tree} failed ({p.returncode}):\n{p.stdout[-2000:]}\n{p.stderr[-2000:]}")
    return json.loads(lines[-1])


def edge_pass():
    import ctypes
    from kafka_specification_b200.runtime import Checker
    with Checker(MODEL, table_log2=30, max_states=1 << 29) as ck:
        r = ck.run()
        st = ck.stats()
        n = ctypes.c_size_t()
        t0 = time.perf_counter()
        ck._check(ck.lib.kmc_edges(ck.ctx, 0, st["distinct"] - st["queue"], None, 0, ctypes.byref(n)))
        ms = (time.perf_counter() - t0) * 1e3
        if n.value + st["out_of_model"] != st["generated"] - st["init_generated"]:
            raise SystemExit(f"edge count {n.value} does not match generated - init - out_of_model")
        return {"states": r.distinct, "edges": n.value, "edge_row_bytes": n.value * 32, "ms": round(ms, 1),
                "run_gpu_ms_expand": round(st["gpu_ms_expand"], 1)}


def state_dump(name, **opts):
    from kafka_specification_b200.runtime import Checker
    with Checker(name, **opts) as ck:
        ck.run()
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "s.dump")
            t0 = time.perf_counter()
            t = ck.dump_states(path)
            wall = time.perf_counter() - t0
            size = os.path.getsize(path)
    return {"model": name, "states": t["states"], "bytes": size, "wall_s": round(wall, 2),
            "decode_s": round(t["decode_s"], 2), "write_s": round(t["write_s"], 2)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--parent", help="tree of the previous commit, built (dispatcher + headline model)")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dump-stop", type=int, default=10_000_000)
    a = ap.parse_args()
    gpu, power, sm_clock = card()
    out = {"gpu": gpu, "power_limit": power, "sm_clock_max": sm_clock}
    if a.parent:
        lines = {"this": [], "parent": []}
        for _ in range(a.rounds):
            lines["parent"].append(bench_line(a.parent, a.steps, a.warmup))
            lines["this"].append(bench_line(ROOT, a.steps, a.warmup))
        out["bench"] = {k: [l.get("value", l) for l in v] for k, v in lines.items()}
        out["bench_lines"] = lines
    out["edges"] = edge_pass()
    out["dump_states"] = [state_dump("kip320_small", table_log2=22),
                          state_dump(MODEL, table_log2=30, max_states=1 << 29, stop_after_states=a.dump_stop)]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
