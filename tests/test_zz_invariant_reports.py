"""-continue reports every violated invariant: its first level, its violators and its own shortest counterexample
(kmc_invariant_reports), on every registered model that violates an invariant, on each engine path."""
import os
import subprocess
import sys

import pytest

import gpu_runs
from conftest import ROOT
from gpu_runs import assert_oracle_b_trace, report_summary as summary
from hostmodel import HostModel
from oracle_a_actions import OracleA

pytestmark = pytest.mark.gpu

KAFKA = ["trunchw_n2", "kip101_n2", "trunchw_small", "kip101_small", "kip279_small", "firsttry_small",
         "kip320_with279_small", "trunchw_3x4_r3e3", "kip101_3x4_r3e3", "kip279_3x4_r3e3", "firsttry_3x4_r3e3"]
MINI = ["minibound", "minibound_mixed", "minibound_init", "minibound_sym", "asyncisr_bounded"]
RING = 1 << 16


def checker(name, **opts):
    """A set of 2^24 slots for the small models, the engine's default size for the others."""
    if name.endswith("_n2") or name.startswith("mini") or name == "asyncisr_bounded":
        opts.setdefault("table_log2", 24)
    return gpu_runs.checker(name, **opts)


def assert_kafka_trace(name, ck, rep):
    """Oracle B checks every step; only the reported invariant must hold on the earlier states and fail on the last
    one."""
    import kso
    if rep["invariant"] in kso.INVARIANTS:
        assert_oracle_b_trace(name, rep["trace"], ck.decoder, [rep["invariant"]])


def assert_mini_trace(oa, rep):
    """The trace replays under Oracle A (OracleA.replay); every state but the last is in the model and satisfies the
    reported invariant, and the last one violates it."""
    states = oa.replay(rep["trace"])
    for st in states[:-1]:
        assert oa.in_model(st) and oa.holds(rep["invariant"], st)
    assert not oa.holds(rep["invariant"], states[-1])


@pytest.mark.parametrize("name", KAFKA + MINI + ["leaderinisr_init"])
def test_every_violated_invariant_is_reported(name, goldens):
    g = goldens[name]
    want = {i: l for i, l in g["first_violation_level"].items() if l is not None}
    with checker(name, cont=True) as ck:
        r = ck.run()
        reps = r.invariant_violations
        assert {x["invariant"]: x["level"] for x in reps} == want
        assert [(x["level"], x["index"]) for x in reps] == sorted((x["level"], x["index"]) for x in reps)
        for x in reps:
            assert x["trace_len"] == x["level"] == len(x["trace"]) and x["complete"]
            assert 1 <= x["violators_first_level"] <= x["violators"]
        # the run's first violation, unless it is a deadlock, is its invariant's entry
        v = r.violation
        if v["kind"] == "invariant":
            e = next(x for x in reps if x["invariant"] == v["invariant"])
            assert (e["level"], e["fingerprint"], e["trace_len"]) == (v["level"], v["fingerprint"], v["trace_len"])
            assert [t["words"] for t in e["trace"]] == [t["words"] for t in r.trace]
        # the picks and counts against an independent host BFS of the lowered model, where the first level fits the ring
        host = HostModel.for_built_model(name).invariant_report(ck.meta["invariants"]) if g["distinct"] < 3_000_000 else None
        for x in reps:
            if host is not None:
                h = host[x["invariant"]]
                assert (x["violators_first_level"], x["violators"]) == (h["violators_first_level"], h["violators"])
                if h["violators_first_level"] <= RING:
                    assert x["fingerprint"] == h["fingerprint"]
            if name in KAFKA:
                assert_kafka_trace(name, ck, x)
        if name in MINI:
            oa = OracleA(name)
            for x in reps:
                assert_mini_trace(oa, x)
        words = name != "minibound_sym"
        first = summary(reps, words)
        r2 = ck.run()
        assert summary(r2.invariant_violations, words) == first, "a second run picks differently"


def test_without_continue_nothing_is_collected():
    with checker("firsttry_small") as ck:
        r = ck.run()
        assert r.violation is not None and r.invariant_violations == []
        assert ck.invariant_reports() == []


def shard_path_reports(name):
    """The reports of the two-kernel kmc_shard_* path at world 1 (gpu_runs.shard_levels)."""
    with checker(name, cont=True) as ck:
        gpu_runs.shard_levels(ck, cont=True)
        ck._check(ck.lib.kmc_shard_sync(ck.ctx))
        return summary(ck.invariant_reports())


@pytest.mark.parametrize("name", ["firsttry_small", "minibound_mixed", "asyncisr_bounded"])
def test_shard_path_at_world_1_reports_the_same(name):
    with checker(name, cont=True) as ck:
        fused = summary(ck.run().invariant_violations)
    assert shard_path_reports(name) == fused


def test_spill_and_a_small_ring_report_the_same():
    with checker("firsttry_small", cont=True) as ck:
        want = summary(ck.run().invariant_violations)
    with checker("firsttry_small", cont=True, spill=True, max_states=1 << 19) as ck:
        r = ck.run()
        assert r.complete
        assert summary(r.invariant_violations) == want


def test_two_gpus_report_the_same():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    with checker("firsttry_small", cont=True) as ck:
        want = ck.run().invariant_violations
    with checker("firsttry_small", cont=True, gpus=2) as ck:
        got = ck.run().invariant_violations
    # the picks and their traces are the same states; the parent words differ (another store layout)
    assert [(x["invariant"], x["level"], x["violators_first_level"], x["violators"], x["fingerprint"],
             [t["words"][0] for t in x["trace"][-1:]]) for x in got] == \
           [(x["invariant"], x["level"], x["violators_first_level"], x["violators"], x["fingerprint"],
             [t["words"][0] for t in x["trace"][-1:]]) for x in want]


@pytest.mark.parametrize("tool", [False, True])
def test_cli_continue_prints_weakisr_then_strongisr(tool):
    cmd = [sys.executable, "-m", "kafka_specification_b200.tlc2", "-continue", "-config",
           os.path.join(ROOT, "models", "Kip320FirstTry_small.cfg")] + (["-tool"] if tool else []) + \
          [os.path.join(ROOT, "oracle", "_ref", "spec", "Kip320FirstTry")]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 12, p.stdout[-3000:] + p.stderr[-3000:]
    out = p.stdout
    w, s = out.index("Error: Invariant WeakIsr is violated."), out.index("Error: Invariant StrongIsr is violated.")
    assert w < s
    assert "State 12:" in out[w:s] and "State 13:" not in out[w:s]
    assert "State 13:" in out[s:] and "State 14:" not in out[s:]
    if tool:
        assert out.count("@!@!@STARTMSG 2110:1 @!@!@") == 2
        assert out.count("@!@!@STARTMSG 2217:4 @!@!@") == 12 + 13
