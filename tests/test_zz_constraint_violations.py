"""Invariant violations that only a CONSTRAINT-discarded state produces, on the GPU, and the counterexample rule under
SYMMETRY.

A successor that a CONSTRAINT discards is generated and invariant-checked but never stored: on the fused single-GPU
path the expand kernel's insert records it in the violator ring itself, with the parent word of the state it came
from, and build_trace reports level + 1 for a trace whose last state is in no store.  An initial state outside the
constraint goes the same way through k_insert.  The models (tests/specs/MiniBound.tla, tests/specs/MCAsyncIsrBounded.tla)
are described in test_constraint_violations_host.py, which checks them against Oracle A on the CPU.  Here every run is
checked against the goldens, its whole store and violator ring against the host audit (store_audit.audit_checker),
and every state of its counterexample against Oracle A, transition by transition.
"""
import functools
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import gpu_runs
from conftest import ROOT
from gpu_runs import CONSTRAINT_MODELS, compare_runs, fused_run, two_kernel_run
from kafka_specification_b200 import build
from oracle_a_actions import OracleA

pytestmark = pytest.mark.gpu

DISCARDED_FIRST = {"minibound", "minibound_init", "asyncisr_bounded"}     # every first violator is a discarded state

checker = functools.partial(gpu_runs.checker, table_log2=16)
audited_run = functools.partial(gpu_runs.audited_run, table_log2=16)


@pytest.fixture(scope="module")
def coverage_golden():
    with open(os.path.join(ROOT, "tests", "golden", "coverage.json")) as f:
        return json.load(f)


def assert_trace_is_an_oracle_a_behaviour(oa, trace, violation):
    """The trace replays under Oracle A (OracleA.replay), every state but the last is in the model and violates
    nothing, and the last one's first violated invariant is the reported one.  Returns the Oracle A state of the last
    one."""
    assert len(trace) == violation["trace_len"] == violation["level"]
    states = oa.replay(trace)
    for i, st in enumerate(states[:-1]):
        assert oa.in_model(st) and not oa.violated(st), f"trace state {i + 1} of {len(states)} violates something"
    last = states[-1]
    assert violation["invariant"] in oa.violated(last) and oa.violated(last)[0] == violation["invariant"]
    return last


def first_violation(g):
    levels = {k: v for k, v in g["first_violation_level"].items() if v}
    if not levels:
        return None, set()
    lvl = min(levels.values())
    return lvl, {k for k, v in levels.items() if v == lvl}


@pytest.mark.parametrize("cont", [False, True])
@pytest.mark.parametrize("name", CONSTRAINT_MODELS)
def test_fused_run_against_golden_audit_and_oracle_a(name, cont, goldens, coverage_golden):
    from golden.make_golden import state_digest
    g = goldens[name]
    r, rep = audited_run(name, details=True, cont=cont)
    lvl, invs = first_violation(g)
    if cont or lvl is None:
        assert r.complete and r.queue == 0
        assert (r.distinct, r.generated, r.depth, r.levels, r.deadlocks, r.stats["out_of_model"]) == (
            g["distinct"], g["generated"], g["depth"], g["levels"], g["deadlocks"], g["out_of_model"])
        # coverage.json: successors per action (discarded ones included, from Oracle A) and, without SYMMETRY, per
        # emit site; the stored states decode to Oracle A's set
        c, cov = coverage_golden[name], rep["coverage"]
        assert {a["name"]: a["generated"] for a in cov["actions"]} == c["per_action"]
        assert cov["init"]["generated"] == c["num_init"] and cov["complete"]
        if not build.registry()[name].get("symmetry"):
            assert cov["sites"] == c["per_site"]
            assert state_digest(rep["texts"]) == g["state_digest"]
    else:
        # stopped at the end of the level whose expansion (or, at level 1, whose insert) found the violation
        assert not r.complete and r.levels == g["levels"][: lvl - 1]
        assert r.stats["out_of_model"] == rep["found"]["out_of_model"] > 0
    assert r.stats["slot_bytes"] == (16 if name == "asyncisr_bounded" else 8)
    if lvl is None:
        assert r.violation is None and rep["violation"] is None
        return
    v = r.violation
    assert v["kind"] == "invariant" and v["level"] == lvl and v["invariant"] in invs and v["trace_len"] == lvl
    assert rep["violation"]["level_end"] == lvl - 1
    oa = OracleA(name)
    last = assert_trace_is_an_oracle_a_behaviour(oa, r.trace, v)
    if name in DISCARDED_FIRST:
        assert not oa.in_model(last) and not oa.holds("Bound", last)
    # the reported record is the trace's last state, with the parent word of the previous trace state
    record = rep["record"]
    assert record[0] == r.trace[-1]["words"]
    if lvl > 1:
        assert (record[1] >> 56) == [a["name"] for a in registry_actions(name)].index(r.trace[-1]["action"]["name"])


def registry_actions(name):
    return json.load(open(os.path.join(ROOT, "build", "models", name, "model.json")))["actions"]


def test_discarded_successors_of_a_state_are_not_a_deadlock(goldens):
    """minibound_nodead checks deadlocks; its state with every counter at Max has only discarded successors."""
    g = goldens["minibound_nodead"]
    with checker("minibound_nodead") as ck:
        r = ck.run()
    assert r.complete and r.violation is None and r.deadlocks == 0
    assert (r.distinct, r.generated, r.stats["out_of_model"]) == (g["distinct"], g["generated"], g["out_of_model"])


def test_every_initial_state_discarded_leaves_an_empty_store(goldens):
    for cont in (False, True):
        with checker("minibound_allout", cont=cont) as ck:
            r = ck.run()
            cov = ck.coverage()
        assert r.complete and r.violation is None and r.trace == []
        assert (r.distinct, r.depth, r.levels, r.generated, r.stats["out_of_model"]) == (0, 0, [], 3, 3)
        assert cov["init"] == {**cov["init"], "distinct": 0, "generated": 3}


@pytest.mark.parametrize("name,cont", [(n, c) for n in CONSTRAINT_MODELS if n != "minibound_allout"
                                       for c in (False, True)])
def test_two_kernel_pipeline_reports_the_same_violation(name, cont):
    """kmc_shard_* at world 1 (expand -> candidate buffer -> k_insert): the same counts, widths and violation -- kind,
    invariant, level, trace length and fingerprint -- as the fused path."""
    compare_runs(fused_run(name, cont=cont, table_log2=16), two_kernel_run(name, cont=cont, table_log2=16),
                 symmetric=name == "minibound_sym")


@pytest.mark.parametrize("cont,ring", [(False, 1 << 9), (True, 1 << 11)])
def test_discarded_counterexample_through_spilled_levels(cont, ring, goldens):
    """asyncisr_bounded (4,088 states) with a spilling ring: levels below the one being expanded live in host memory,
    so the trace of the level-6 violator (a discarded successor) walks from the ring into the spilled levels."""
    g = goldens["asyncisr_bounded"]
    r, rep = audited_run("asyncisr_bounded", cont=cont, spill=True, max_states=ring)
    assert r.stats["max_states"] == ring < g["distinct"]
    if cont:
        assert r.complete and (r.distinct, r.levels, r.stats["out_of_model"]) == (g["distinct"], g["levels"], g["out_of_model"])
    assert r.violation["level"] == 6 and r.violation["invariant"] == "VersionInBound"
    last = assert_trace_is_an_oracle_a_behaviour(OracleA("asyncisr_bounded"), r.trace, r.violation)
    assert not OracleA("asyncisr_bounded").in_model(last)


@pytest.mark.parametrize("cont", [False, True])
def test_checkpoint_before_the_violating_level_and_recover(tmp_path, cont, goldens):
    """A bounded run of asyncisr_bounded stops (with a checkpoint) after level 5 is stored, before its expansion finds
    the discarded violators; the recovered run finds the same violation as an uninterrupted one, and out_of_model
    carries over: counted before the checkpoint plus after it."""
    g = goldens["asyncisr_bounded"]
    d = str(tmp_path)
    with checker("asyncisr_bounded", checkpoint_dir=d, stop_after_states=150) as ck:
        a = ck.run()
    assert not a.complete and a.violation is None and a.levels == g["levels"][:4]
    with checker("asyncisr_bounded", cont=cont) as ck:
        want = ck.run()
    r, rep = audited_run("asyncisr_bounded", recover=d, cont=cont)
    assert r.stats["out_of_model"] == want.stats["out_of_model"] == rep["found"]["out_of_model"]
    assert 0 < a.stats["out_of_model"] < r.stats["out_of_model"]
    if cont:
        assert r.complete and r.stats["out_of_model"] == g["out_of_model"] and r.levels == g["levels"]
    v, w = r.violation, want.violation
    assert (v["kind"], v["invariant"], v["level"], v["trace_len"]) == (w["kind"], w["invariant"], w["level"], w["trace_len"])
    assert v["fingerprint"] == w["fingerprint"] == rep["violation"]["fingerprint"]


def test_cli_reports_a_discarded_violator():
    """tlc2 on MiniBound: TLC's invariant-violation message, a four-state trace whose last state has a counter at
    Max + 1 (a state the CONSTRAINT discards), and TLC's exit code for a safety violation."""
    specs = os.path.join(ROOT, "tests", "specs")
    p = subprocess.run([sys.executable, "-m", "kafka_specification_b200.tlc2", "-config", os.path.join(specs, "MiniBound.cfg"),
                        os.path.join(specs, "MiniBound")], cwd=ROOT, capture_output=True, text=True, timeout=600)
    out = p.stdout + p.stderr
    assert p.returncode == 12, out
    assert "Error: Invariant NotOver is violated." in out and "Error: The behavior up to this point is:" in out
    assert "State 4: <Inc line" in out and "State 5:" not in out
    last = out[out.index("State 4:"):]
    assert ":> 3" in last.split("\n\n")[0], last


def test_symmetry_counterexample_is_the_rule_pick_over_orbits():
    """minibound_sym: OneFull is first violated at level 3 by three orbits, reached only through members that are not
    their canonical form.  The reported counterexample is the rule's pick over orbits -- deadlocks first, then the
    smallest fingerprint of the canonical form -- computed on the host from the lowered model's own BFS, whichever
    member the GPU stored; and two runs report the same orbit."""
    from store_audit import AuditLib, expected_orbit, fingerprint, host_audit
    a = AuditLib.for_built_model("minibound_sym")
    _, _, found = host_audit("minibound_sym")
    orbit, fp = expected_orbit(a, found)
    got = []
    for _ in range(2):
        r, _ = audited_run("minibound_sym")
        v = r.violation
        assert (v["kind"], v["invariant"], v["level"]) == ("invariant", "OneFull", 3)
        words = np.asarray([r.trace[-1]["words"]], dtype=np.uint64)
        canon = a.canonicalize(words)
        assert not np.array_equal(canon, words)            # the stored member is not the canonical form
        assert [int(x) for x in canon[0]] == orbit and v["fingerprint"] == fp == int(fingerprint(canon, a.state_bits)[0])
        got.append(([int(x) for x in canon[0]], v["fingerprint"]))
    assert got[0] == got[1]
