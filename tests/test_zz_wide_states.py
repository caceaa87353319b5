"""The engine at the state widths and set-key forms that no Kafka model reaches, on the GPU.

The expand kernel and the set are compiled per model, and several of their code paths depend on the width W of the
packed state: the tile holds SPT = 4, 4, 4, 3, 2, 1, 1 states per thread for W = 1 .. 7, stage rows are W + 1 words,
the tile load is 64-bit at odd W, and the set key is a 128-bit fingerprint from W = 3 on.  Two narrower forms change the
key as well: one word with all 64 bits used (no bijection: a hashed 8-byte key) and two words that can pack to all-ones
(no exact 16-byte key: the fingerprint instead).  tests/specs/MiniWide.tla reaches all of them (its cfgs are checked on
the CPU in test_wide_states_host.py).  Every expected number here comes from Oracle A (the goldens) or from the closed
form of MiniWide (make_golden.closed_form), and every stored state, parent link and counterexample from the audit of
the whole store against the lowered Next compiled for the host (store_audit.audit_checker).
"""
import functools
import os

import numpy as np
import pytest

import gpu_runs
from conftest import ROOT
from golden.make_golden import closed_form, state_digest
from gpu_runs import compare_runs, fused_run, two_kernel_run
from hostmodel import HostModel
from kafka_specification_b200.build import registry
from kafka_specification_b200.frontend.cfg import parse_cfg
from oracle_a_actions import OracleA
from store_audit import VIOL_RING, audit_checker

pytestmark = pytest.mark.gpu

# (model, words, set slot bytes); every one hashes its set key (kmc_model_info.exact = 0)
SMALL = [("miniwide_one64", 1, 8), ("miniwide_two128", 2, 16), ("miniwide_w5", 5, 16), ("miniwide_w6", 6, 16),
         ("miniwide_w7", 7, 16)]
SMALL_NAMES = [n for n, _, _ in SMALL]
# levels wider than 132 SMs x TILE at W = 6, 7 (TILE = 1024): each CTA loops over several tiles
LARGE = [("miniwide_w5_large", 5), ("miniwide_w6_large", 6), ("miniwide_w7_large", 7)]
H100_SMS = 132

checker = functools.partial(gpu_runs.checker, table_log2=16)


def expected(name):
    """The closed form of a MiniWide cfg without SYMMETRY."""
    cfg = parse_cfg(open(os.path.join(ROOT, registry()[name]["cfg"])).read())
    return closed_form("MiniWide", cfg)


def run_and_audit(name, **opts):
    """One kmc_run and the audit of its whole store: (RunResult, audit report, kmc_model_info (words, exact))."""
    with checker(name, **opts) as ck:
        r = ck.run()
        rep = audit_checker(ck, r.levels, r.distinct)
        rep["texts"] = ck.decoder.texts(rep["states"])
        info = (ck.info.words, ck.info.exact)
    assert sum(rep["widths"]) == r.distinct
    return r, rep, info


def assert_complete(r, want):
    assert r.complete and r.queue == 0
    assert (r.distinct, r.generated, r.depth, r.levels, r.deadlocks, r.stats["out_of_model"]) == (
        want["distinct"], want["generated"], want["depth"], want["levels"], want["deadlocks"], want["out_of_model"])


def assert_oracle_a_trace(name, trace, violation):
    """The counterexample replays under Oracle A, transition by transition, and only its last state violates FewFull."""
    oa = OracleA(name)
    assert len(trace) == violation["trace_len"] == violation["level"]
    states = oa.replay(trace)
    assert all(not oa.violated(st) for st in states[:-1])
    assert oa.violated(states[-1]) == ["FewFull"]


def host_reports(name):
    """kmc_invariant_reports of a -continue run, from the host BFS of the lowered model."""
    hm = HostModel.for_built_model(name)
    rep = hm.invariant_report(["TypeOk", "FewFull"])
    assert rep.pop(None) == 0
    return rep


def assert_reports(r, name, want):
    """The per-invariant reports of a -continue run: FewFull only, at the closed form's level and first-level violator
    count, with the host BFS's totals and pick.  Every discarded successor violates FewFull; where one level has more of
    them than the engine's stage holds (VIOL_RING), the report says it is incomplete and counts fewer violators, and
    where the first level has more violators than the ring holds, its pick is one of them, not the host's."""
    host = host_reports(name)["FewFull"]
    assert [v["invariant"] for v in r.invariant_violations] == ["FewFull"]
    v = r.invariant_violations[0]
    assert v["level"] == want["first_violation_level"]["FewFull"] == host["level"]
    assert v["violators_first_level"] == want["violators_first_level"]["FewFull"] == host["violators_first_level"]
    assert v["trace_len"] == v["level"]
    if want["out_of_model"] <= VIOL_RING:
        assert v["complete"] and v["violators"] == host["violators"] == want["violating_states"]["FewFull"]
    else:
        assert not v["complete"] and v["violators"] < host["violators"] == want["violating_states"]["FewFull"]
    if v["violators_first_level"] <= VIOL_RING:
        assert v["fingerprint"] == host["fingerprint"]


def without_pick(run):
    """A fused_run / two_kernel_run result without the fingerprint of its counterexample: at a first violating level with
    more violators than the ring holds, the pick is not deterministic."""
    summary, levels = run
    return {**summary, "violation": {k: x for k, x in summary["violation"].items() if k != "fingerprint"}}, levels


@pytest.mark.parametrize("name,words,slot_bytes", SMALL)
def test_full_run_against_golden_closed_form_and_oracle_a_states(name, words, slot_bytes, goldens):
    g, want = goldens[name], expected(name)
    r, rep, info = run_and_audit(name, cont=True)
    assert_complete(r, g)
    assert_complete(r, want)
    assert info == (words, 0) and r.stats["slot_bytes"] == slot_bytes
    assert state_digest(rep["texts"]) == g["state_digest"]
    assert_reports(r, name, want)
    assert_oracle_a_trace(name, r.invariant_violations[0]["trace"], r.invariant_violations[0])


@pytest.mark.parametrize("name", SMALL_NAMES)
def test_run_stopped_at_the_first_violation(name, goldens):
    g, want = goldens[name], expected(name)
    r, rep, _ = run_and_audit(name)
    lvl = want["first_violation_level"]["FewFull"]
    assert not r.complete and r.levels == g["levels"][: lvl - 1]
    v = r.violation
    assert (v["kind"], v["invariant"], v["level"], v["trace_len"]) == ("invariant", "FewFull", lvl, lvl)
    assert rep["violation"]["count"] == want["violators_first_level"]["FewFull"]
    assert_oracle_a_trace(name, r.trace, v)


@pytest.mark.parametrize("cand_bytes", [0, 1 << 16])
@pytest.mark.parametrize("name", SMALL_NAMES)
def test_two_kernel_pipeline_finds_the_same_levels(name, cand_bytes):
    """kmc_shard_* at world 1 (expand -> candidate buffer -> k_insert of W + 1-word rows) against the fused path; a
    64 KB candidate buffer cuts every level into chunks of a few states."""
    opts = {"cand_bytes": cand_bytes} if cand_bytes else {}
    compare_runs(fused_run(name, cont=True, table_log2=16, **opts), two_kernel_run(name, cont=True, table_log2=16, **opts))


@pytest.mark.parametrize("name,table_log2", [("miniwide_one64", 4), ("miniwide_two128", 4), ("miniwide_w5", 6),
                                             ("miniwide_w6", 6), ("miniwide_w7", 6)])
def test_set_spill_through_many_flushes(name, table_log2, goldens):
    """The set's hashed keys (8 bytes at W = 1, 16 bytes at the all-ones W = 2 and from W = 3 on) move to host memory
    whenever half the table is used, also in the middle of a level, and the run ends with the golden's states."""
    g = goldens[name]
    r, rep, _ = run_and_audit(name, cont=True, set_spill=True, table_log2=table_log2, max_states=g["distinct"] + 4096)
    assert_complete(r, g)
    assert state_digest(rep["texts"]) == g["state_digest"]
    st = r.stats
    assert st["table_slots"] == 1 << table_log2 and st["set_host_keys"] <= r.distinct
    if name == "miniwide_one64":            # 16 states through 8 keys of room
        assert st["set_flushes"] >= 1
    else:
        assert st["set_flushes"] >= 5 and st["set_flushes"] > r.depth and st["set_filtered"] > 0


@pytest.mark.parametrize("name,ring", [("miniwide_w5_large", 1 << 17), ("miniwide_w7_large", 1 << 19)])
def test_spill_ring_smaller_than_the_state_space(name, ring):
    """A store ring that holds the two widest adjacent levels but not the whole run: rows of 5 and 7 words wrap the ring
    and move to host memory."""
    want = expected(name)
    r, _, _ = run_and_audit(name, cont=True, spill=True, max_states=ring, table_log2=21)
    assert r.stats["max_states"] == ring < r.distinct
    assert_complete(r, want)
    assert_reports(r, name, want)


@pytest.mark.parametrize("name", SMALL_NAMES)
def test_checkpoint_and_recover(name, tmp_path, goldens):
    """A run stopped (with a checkpoint) at the end of level 3, recovered into a new context: W-word rows through the
    checkpoint file, and the recovered run ends at the golden's counts."""
    g = goldens[name]
    d = str(tmp_path)
    with checker(name, checkpoint_dir=d, stop_after_states=sum(g["levels"][:2]) + 1, cont=True) as ck:
        a = ck.run()
    assert not a.complete and a.levels == g["levels"][:2] and a.distinct == sum(g["levels"][:3])
    r, rep, _ = run_and_audit(name, recover=d, cont=True)
    assert_complete(r, g)
    assert state_digest(rep["texts"]) == g["state_digest"]


def test_symmetry_at_six_words(goldens):
    """canonicalize over six words: the orbit count and levels of Oracle A, with an audited store."""
    g = goldens["miniwide_w6_sym"]
    r, rep, info = run_and_audit("miniwide_w6_sym", cont=True)
    assert info == (6, 0)
    assert_complete(r, g)
    assert r.invariant_violations[0]["level"] == g["first_violation_level"]["FewFull"]
    rs, _, _ = run_and_audit("miniwide_w6_sym")
    assert rs.violation["level"] == g["first_violation_level"]["FewFull"]
    assert_oracle_a_trace("miniwide_w6_sym", rs.trace, rs.violation)


@pytest.mark.parametrize("name,words", LARGE)
def test_large_levels_against_closed_form_and_host_bfs(name, words):
    want = expected(name)
    r, rep, info = run_and_audit(name, cont=True, table_log2=21)
    assert info == (words, 0)
    assert_complete(r, want)
    assert_reports(r, name, want)
    if words >= 6:
        assert max(r.levels) > H100_SMS * 1024
    host = HostModel.for_built_model(name).bfs()
    assert host["widths"] == r.levels and host["generated"] == r.generated
    assert np.array_equal(gpu_runs.sorted_rows(host["states"]), gpu_runs.sorted_rows(rep["states"]))


@pytest.mark.parametrize("name", [n for n, _ in LARGE])
def test_large_two_kernel_pipeline_in_many_chunks(name):
    compare_runs(without_pick(fused_run(name, cont=True, table_log2=21, cand_bytes=1 << 22)),
                 without_pick(two_kernel_run(name, cont=True, table_log2=21, cand_bytes=1 << 22)))


def test_stopped_large_run_reports_the_audited_pick():
    """Stops at FewFull's first level, whose C(21, 7) = 116,280 violators are more than the violator ring keeps: the
    audit checks that the reported state is one of them."""
    want = expected("miniwide_w6_large")
    r, rep, _ = run_and_audit("miniwide_w6_large", table_log2=21)
    lvl = want["first_violation_level"]["FewFull"]
    assert r.violation["level"] == lvl and r.levels == want["levels"][: lvl - 1]
    assert rep["violation"]["count"] == want["violators_first_level"]["FewFull"]
