"""-continue reports every violated invariant: its first level, its violators and its own shortest counterexample
(kmc_invariant_reports), on every registered model that violates an invariant, on each engine path."""
import os
import subprocess
import sys

import pytest

from conftest import ROOT
from hostinvariants import HostInvariants
from test_gpu_parity import _assert_trace_is_behaviour
from test_zz_constraint_violations import OracleA

pytestmark = pytest.mark.gpu

KAFKA = ["trunchw_n2", "kip101_n2", "trunchw_small", "kip101_small", "kip279_small", "firsttry_small",
         "kip320_with279_small", "trunchw_3x4_r3e3", "kip101_3x4_r3e3", "kip279_3x4_r3e3", "firsttry_3x4_r3e3"]
MINI = ["minibound", "minibound_mixed", "minibound_init", "minibound_sym", "asyncisr_bounded"]
RING = 1 << 16


def checker(name, **kw):
    from kafka_specification_b200.runtime import Checker
    kw.setdefault("table_log2", 24 if name.endswith("_n2") or name.startswith("mini") or name == "asyncisr_bounded" else 0)
    if not kw["table_log2"]:
        del kw["table_log2"]
    return Checker(name, **kw)


def summary(reports, words=True):
    """What a run reports per invariant.  (The states before the last one are not part of it: a state's parent is the
    generator whose insert won, which may differ from run to run, as for kmc_violation's trace; under SYMMETRY
    neither is the last one: the pick is an orbit, and the member stored is the one whose insert won.)"""
    return [(r["invariant"], r["level"], r["violators_first_level"], r["violators"], r["fingerprint"], r["trace_len"],
             r["trace"][-1]["words"] if r["trace"] and words else None) for r in reports]


def assert_kafka_trace(name, ck, rep):
    """Oracle B checks every step (as _assert_trace_is_behaviour); only the reported invariant must hold on the earlier
    states and fail on the last one."""
    import kso
    saved = ck.meta["invariants"]
    ck.meta["invariants"] = [rep["invariant"]]
    try:
        if rep["invariant"] in kso.INVARIANTS:
            _assert_trace_is_behaviour(name, rep["trace"], ck)
    finally:
        ck.meta["invariants"] = saved


def assert_mini_trace(oa, rep):
    assert rep["trace"][0]["action"] is None
    by_text = {oa.text(s): s for s in oa.inits}
    states = [by_text[rep["trace"][0]["text"]]]
    for i, t in enumerate(rep["trace"][1:], start=1):
        nxt = [s1 for s1, label in oa.it.labelled_successors(oa.next_e, states[-1])
               if label == t["action"]["name"] and oa.text(s1) == t["text"]]
        assert nxt, f"trace state {i + 1} is not a {t['action']['name']} successor of state {i}"
        states.append(nxt[0])
    for st in states[:-1]:
        assert oa.in_model(st) and oa.holds(rep["invariant"], st)
    assert not oa.holds(rep["invariant"], states[-1])


@pytest.fixture(scope="module")
def all_models():
    from kafka_specification_b200.build import registry
    return registry()


@pytest.mark.parametrize("name", KAFKA + MINI + ["leaderinisr_init"])
def test_every_violated_invariant_is_reported(name, goldens, all_models):
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
        host = HostInvariants.for_built_model(name, ck.meta["invariants"]).report() if g["distinct"] < 3_000_000 else None
        for x in reps:
            if host is not None:
                h = host[x["invariant"]]
                assert (x["violators_first_level"], x["violators"]) == (h["violators_first_level"], h["violators"])
                if h["violators_first_level"] <= RING:
                    assert x["fingerprint"] == h["fingerprint"]
            if name in KAFKA:
                assert_kafka_trace(name, ck, x)
        if name in MINI:
            oa = OracleA(all_models, name)
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


def _shard_run(name, **opts):
    """The two-kernel kmc_shard_* path at world 1 (expand into the candidate buffer, k_insert, level end)."""
    import numpy as np
    from kafka_specification_b200.runtime import Checker
    with Checker(name, cont=True, **opts) as ck:
        lib, c = ck.lib, ck.ctx
        assert lib.kmc_shard_begin(c) == 0 and lib.kmc_shard_seed_init(c) == 0
        from kafka_specification_b200.runtime import ShardBuffers
        import ctypes
        b = ShardBuffers()
        assert lib.kmc_shard_buffers(c, ctypes.byref(b)) == 0
        tail, first, count = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64()
        counts = np.zeros(8, dtype=np.uint64)
        assert lib.kmc_shard_counts(c, counts.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64))) == 0
        assert lib.kmc_shard_insert(c, b.recv, int(counts[0]), ctypes.byref(tail)) == 0
        assert lib.kmc_shard_level_done(c, ctypes.byref(first), ctypes.byref(count)) == 0
        chunk = max(1, b.region_rows // 32)
        while count.value:
            f, n = first.value, count.value
            for off in range(0, n, chunk):
                k = min(chunk, n - off)
                assert lib.kmc_shard_reset_cand(c) == 0
                assert lib.kmc_shard_expand(c, f + off, k) == 0
                assert lib.kmc_shard_counts(c, counts.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64))) == 0
                assert lib.kmc_shard_insert(c, b.recv, int(counts[0]), ctypes.byref(tail)) == 0
            assert lib.kmc_shard_level_done(c, ctypes.byref(first), ctypes.byref(count)) == 0
        assert lib.kmc_shard_sync(c) == 0
        return summary(ck.invariant_reports())


@pytest.mark.parametrize("name", ["firsttry_small", "minibound_mixed", "asyncisr_bounded"])
def test_shard_path_at_world_1_reports_the_same(name):
    with checker(name, cont=True) as ck:
        fused = summary(ck.run().invariant_violations)
    tl = {"table_log2": 24} if not name.startswith("first") else {}
    assert _shard_run(name, **tl) == fused


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
