"""Invariant violations that only a CONSTRAINT-discarded state produces, on the CPU.

TLC counts a successor that a CONSTRAINT discards as generated and checks it against the invariants every time it is
generated, but never stores or explores it; an initial state outside the constraint is treated the same way.  The
models here (tests/specs/MiniBound.tla and its cfgs, tests/specs/MCAsyncIsrBounded.tla) make that rule decide:
  minibound         the first violation (NotOver, level 4) comes only from discarded successors
  minibound_mixed   one level end holds stored violators (OneFull) and discarded ones (NotOver)
  minibound_init    some initial states are discarded, and they violate NotOver
  minibound_allout  every initial state is discarded: nothing is stored
  minibound_nodead  a state whose successors are all discarded is not a deadlock (CHECK_DEADLOCK TRUE)
  minibound_sym     SYMMETRY, OneFull first violated by stored states of three orbits at once, none of them stored
                    as its canonical form
  asyncisr_bounded  two-word states (16-byte set keys), violated only by discarded successors
Oracle A (oracle/tla_interp.py) against the lowered model compiled for the host, and the whole-store audit over the
host BFS's store, whose violator rows are what the engine's ring must hold."""
import os

import numpy as np
import pytest

from conftest import HAVE_REFERENCE, ROOT
from golden.make_golden import state_digest

NEEDS_REFERENCE = {"asyncisr_bounded"}          # extends the reference's AsyncIsr
MODELS = ["minibound", "minibound_mixed", "minibound_init", "minibound_allout", "minibound_nodead", "minibound_sym",
          "asyncisr_bounded"]


@pytest.fixture(scope="module")
def all_models():
    """The registry build() compiles: these models are test-only, registered in tests/specs/MODELS.json."""
    from kafka_specification_b200.build import registry
    return registry()


def _skip_without_reference(name):
    if name in NEEDS_REFERENCE and not HAVE_REFERENCE:
        pytest.skip("oracle/_ref/spec is missing: run build() first")


def _cfg_text(all_models, name):
    return open(os.path.join(ROOT, all_models[name]["cfg"])).read()


_LOWERED = {}


def lowered(all_models, name):
    from hostmodel import lower_model
    from kafka_specification_b200.build import tla_search_dirs
    if name not in _LOWERED:
        _LOWERED[name] = lower_model(all_models[name]["module"], tla_search_dirs(), _cfg_text(all_models, name), name=name)
    return _LOWERED[name]


def audit_lib(all_models, name):
    from store_audit import AuditLib
    m = lowered(all_models, name)
    return AuditLib(name, m.header, m.invariants_header)


_ORACLE = {}


def oracle_a(all_models, name):
    """Oracle A over the whole state space (past violations, deadlocks unchecked, as the goldens are made) and its first
    violation under the cfg's own settings (stopping there, as TLC does)."""
    import tla_interp
    from kafka_specification_b200.build import tla_search_dirs
    if name not in _ORACLE:
        text = _cfg_text(all_models, name)
        full = tla_interp.run_bfs(all_models[name]["module"], tla_search_dirs(), text + "\nCHECK_DEADLOCK FALSE\n",
                                  collect_states=True, stop_on_violation=False)
        first = tla_interp.run_bfs(all_models[name]["module"], tla_search_dirs(), text)
        _ORACLE[name] = (full, first)
    return _ORACLE[name]


@pytest.mark.parametrize("name", MODELS)
def test_golden_is_oracle_a(name, all_models, goldens):
    """The committed golden is what Oracle A computes now, out_of_model included."""
    _skip_without_reference(name)
    a, _ = oracle_a(all_models, name)
    g = goldens[name]
    for k in ("distinct", "generated", "depth", "levels", "deadlocks", "out_of_model", "first_violation_level"):
        assert g[k] == a[k], k
    if not all_models[name].get("symmetry"):
        assert g["state_digest"] == state_digest(a["states"])


@pytest.mark.parametrize("name", MODELS)
@pytest.mark.parametrize("items", [False, True])
def test_lowered_model_agrees_with_oracle_a(name, items, all_models):
    from hostmodel import run_host
    _skip_without_reference(name)
    a, first = oracle_a(all_models, name)
    m = lowered(all_models, name)
    r = run_host(m, dump=True, items=items)
    assert r["complete"] and not r["fail"]
    assert (r["distinct"], r["generated"], r["depth"], r["levels"], r["deadlocks"]) == (
        a["distinct"], a["generated"], a["depth"], a["levels"], a["deadlocks"])
    assert r["first_violation_level"] == {k: v for k, v in a["first_violation_level"].items()}
    if first["violation"] is None:
        assert r["first_violated"] is None
    else:
        assert r["first_violated_level"] == first["violation"]["level"]
        if name != "minibound_mixed":           # there two invariants are first violated at the same level
            assert r["first_violated"] == first["violation"]["invariant"]
    if not all_models[name].get("symmetry"):
        assert state_digest([m.state_text(row) for row in r["states"]]) == state_digest(a["states"])


@pytest.mark.parametrize("name,level", [("minibound", 4), ("asyncisr_bounded", 6)])
def test_first_violation_comes_from_a_successor_that_is_not_stored(name, level, all_models, goldens):
    """No stored state violates an invariant, yet the run has a violation at `level`: a discarded successor's."""
    _skip_without_reference(name)
    from hostmodel import HostModel
    hm = HostModel.from_lowered(lowered(all_models, name))
    r = hm.bfs()
    assert len(r["states"]) == goldens[name]["distinct"]
    assert all(hm.first_violated(s) < 0 for s in r["states"])
    assert r["first_invariant_level"] == level == min(v for v in goldens[name]["first_violation_level"].values() if v)
    # the violating successor is a successor of a stored state of the level before, and the constraint discards it
    bounds = np.concatenate([[0], np.cumsum(r["widths"])])
    found = 0
    for s in r["states"][bounds[level - 2]:bounds[level - 1]]:
        rows, _ = hm.successors(s)
        found += sum(1 for t in rows if hm.first_violated(t) >= 0 and not hm.in_model(t))
    assert found > 0


def test_all_initial_states_discarded(all_models, goldens):
    from hostmodel import HostModel
    g = goldens["minibound_allout"]
    assert (g["distinct"], g["depth"], g["levels"], g["generated"], g["out_of_model"]) == (0, 0, [], 3, 3)
    hm = HostModel.from_lowered(lowered(all_models, "minibound_allout"))
    assert hm.num_init == 3 and not any(hm.in_model(s) for s in hm.init_states())
    r = hm.bfs()
    assert len(r["states"]) == 0 and r["widths"] == [] and r["generated"] == 3 and r["first_invariant"] is None


def test_discarded_successors_are_not_a_deadlock(all_models, goldens):
    """minibound_nodead: the state with every counter at Max has successors, all of them discarded; it is counted as
    generating them and is no deadlock, although deadlocks are checked."""
    from hostmodel import HostModel
    g = goldens["minibound_nodead"]
    hm = HostModel.from_lowered(lowered(all_models, "minibound_nodead"))
    assert hm.check_deadlock and g["check_deadlock"] and g["deadlocks"] == 0
    r = hm.bfs()
    assert r["deadlocks"] == 0 and len(r["states"]) == g["distinct"]
    succ = [hm.successors(s)[0] for s in r["states"]]
    all_out = [s for s, rows in zip(r["states"], succ) if len(rows) and not any(hm.in_model(t) for t in rows)]
    assert len(all_out) == 1
    m = lowered(all_models, "minibound_nodead")
    assert "cnt = (p1 :> 2 @@ p2 :> 2 @@ p3 :> 2)" in m.state_text(all_out[0])


# ------------------------------------------------------------------------------------------------ the store audit
def _host_audit(all_models, name, sites=True):
    a = audit_lib(all_models, name)
    st = a.host_bfs(sites=sites)
    found = a.check_store(st["states"], st["parents"], st["widths"], st["n_expanded"], check_deadlock=a.check_deadlock)
    return a, st, found


@pytest.mark.parametrize("name", MODELS)
def test_audit_of_the_host_store_counts_the_discarded_states(name, all_models, goldens):
    """The audit recomputes generated, deadlocks and out_of_model from the stored states alone; out_of_model matches
    Oracle A's independent count, and the violators it lists are exactly Oracle A's violating generations."""
    _skip_without_reference(name)
    a, st, found = _host_audit(all_models, name)
    g = goldens[name]
    assert (found["generated"], found["deadlocks"], found["out_of_model"]) == (g["generated"], g["deadlocks"], g["out_of_model"])
    full, _ = oracle_a(all_models, name)
    # a violator is listed once per first violated invariant; Oracle A counts it once per invariant it violates
    per_inv = [n for n in full["violating_states"].values() if n]
    assert max(per_inv, default=0) <= sum(found["violators_per_level_end"]) <= sum(per_inv)
    levels = [l for l in g["first_violation_level"].values() if l]
    ends = [e for e, c in enumerate(found["violators_per_level_end"]) if c]
    assert ends[:1] == [min(levels) - 1 for _ in levels[:1]]


def _level_of(widths):
    return np.repeat(np.arange(1, len(widths) + 1), widths)


@pytest.mark.parametrize("name,level_end", [("minibound", 3), ("asyncisr_bounded", 5), ("minibound_init", 0)])
def test_audit_lists_the_discarded_violators_at_their_level_end(name, level_end, all_models, goldens):
    """Every violator row of the first level end is a discarded state: a successor, under the action its parent word
    names, of a stored state of that level (or, at level end 0, a discarded initial state with NO_PARENT)."""
    _skip_without_reference(name)
    from store_audit import NO_PARENT, expected_violation
    a, st, found = _host_audit(all_models, name)
    want = expected_violation(a, found)
    assert want["level_end"] == level_end and want["level"] == level_end + 1 and want["kind"] == "invariant"
    rows, w = found["violators"], a.words
    assert len(rows) == found["violators_per_level_end"][level_end] > 0
    level = _level_of(st["widths"])
    inits = {tuple(int(x) for x in s) for s in a.init_states()}
    for r in rows:
        assert not a.in_model(r[:w]) and a.first_violated(r[:w]) == int(r[w + 1])
        pw = int(r[w])
        if level_end == 0:
            assert pw == NO_PARENT and tuple(int(x) for x in r[:w]) in inits
            continue
        idx, act = pw & 0xFFFFFFFFFF, pw >> 56
        assert level[idx] == level_end
        succ, acts = a.successors(st["states"][idx])
        assert any(np.array_equal(t, r[:w]) and int(x) == act for t, x in zip(succ, acts))
    # the pick is the smallest canonical fingerprint among them
    assert want["fingerprint"] == min(int(x) for x in a.fingerprints(rows[:, :w], True))


def test_audit_pick_chooses_between_stored_and_discarded_violators(all_models):
    """minibound_mixed: the first level end holds OneFull violators that are stored and NotOver violators that are
    discarded; the rule (smallest fingerprint) picks among both kinds."""
    a, st, found = _host_audit(all_models, "minibound_mixed")
    from store_audit import expected_violation
    want = expected_violation(a, found)
    rows, w = found["violators"], a.words
    inmodel = np.array([a.in_model(r[:w]) for r in rows])
    assert want["level"] == 3 and inmodel.any() and (~inmodel).any()
    names = lowered(all_models, "minibound_mixed").invariants
    assert {names[int(i)] for i in rows[inmodel, w + 1]} == {"OneFull"}
    assert {names[int(i)] for i in rows[~inmodel, w + 1]} <= {"OneFull", "NotOver"}
    fps = a.fingerprints(rows[:, :w], True)
    assert want["fingerprint"] == int(fps.min())


def expected_orbit(a, found):
    """The counterexample the documented rule picks, as an orbit: (canonical words, fingerprint of the canonical form),
    computed from the violators alone -- whichever member of each orbit a store happens to hold."""
    from store_audit import fingerprint
    w = a.words
    rows = found["violators"]
    dead = rows[:, w + 1] == np.uint64((1 << 64) - 1)
    canon = a.canonicalize(rows[:, :w])
    fps = fingerprint(canon, a.state_bits)
    keys = [(0 if d else 1, int(f)) for d, f in zip(dead, fps)]
    best = min(range(len(rows)), key=lambda i: keys[i])
    return [int(x) for x in canon[best]], int(fps[best])


def test_symmetry_pick_is_an_orbit_whichever_member_is_stored(all_models):
    """minibound_sym: OneFull is first violated at level 3 by three orbits, each reached through three members, none of
    them canonical (First starts at Max).  The rule's pick (deadlocks first, then the smallest fingerprint of the
    canonical form) is the same orbit whichever members the store holds, and differs from a pick by the stored
    members' own fingerprints."""
    from store_audit import expected_violation
    picks, members = [], []
    for sites in (False, True):
        a, st, found = _host_audit(all_models, "minibound_sym", sites=sites)
        w = a.words
        rows = found["violators"]
        canon = {tuple(int(x) for x in c) for c in a.canonicalize(rows[:, :w])}
        assert len(canon) == 3 and found["violators_per_level_end"][2] == len(rows)
        want = expected_violation(a, found)
        orbit, fp = expected_orbit(a, found)
        assert want["level"] == 3 and want["fingerprint"] == fp
        assert [int(x) for x in a.canonicalize(np.asarray([want["words"]], dtype=np.uint64))[0]] == orbit
        picks.append((orbit, fp))
        members.append({tuple(int(x) for x in r[:w]) for r in rows})
    assert picks[0] == picks[1]
    # no stored violator is its orbit's canonical form: the fingerprint of the stored member is never the orbit's
    from store_audit import fingerprint
    a = audit_lib(all_models, "minibound_sym")
    stored = np.asarray(sorted(members[0] | members[1]), dtype=np.uint64)
    assert not (a.canonicalize(stored) == stored).all(axis=1).any()
    assert picks[0][1] not in {int(x) for x in fingerprint(stored, a.state_bits)}


@pytest.mark.parametrize("name", ["minibound_sym", "minibound"])
def test_sharded_stand_in_reports_the_rule_pick(name, all_models, tmp_path):
    """The host stand-in of a sharded rank (host_model.cpp hs_*) under the multi-rank driver, two ranks over gloo:
    the job's counterexample is the orbit the rule picks over the union of the violators."""
    from test_sharded_gloo import _run
    r = _run(name, 2, 5, tmp_path)
    _, _, found = _host_audit(all_models, name)
    a = audit_lib(all_models, name)
    _, fp = expected_orbit(a, found)
    assert r["violation"]["fingerprint"] == fp and r["trace_ok"] is True
