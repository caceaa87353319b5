"""The whole-store audit (tests/support/host_model.cpp, store_audit.py) on the CPU: it accepts a clean store written in
the engine's format by a level-ordered host BFS through the two-phase form, and rejects each kind of corruption with
the check that catches it.  The reference fingerprints are checked against their pure-int restatement."""
import os

import numpy as np
import pytest

from conftest import ROOT, needs_reference
from store_audit import AuditLib

AUDITED = ["kip320_n2", "asyncisr_v2", "kip320sym_n2"]


@pytest.fixture(scope="module")
def clean_stores():
    out = {}
    for name in AUDITED:
        a = AuditLib.for_registered(name)
        out[name] = (a, a.host_bfs(sites=True))     # the order coverage.json was made in
    return out


def _check(a, st, goldens, coverage_golden=None, deadlocks=None):
    from store_audit import compare
    found = a.check_store(st["states"], st["parents"], st["widths"], st["n_expanded"], check_deadlock=a.check_deadlock)
    g = goldens[a.name]
    stats = {"generated": g["generated"], "deadlocks": g["deadlocks"] if deadlocks is None else deadlocks,
             "out_of_model": found["out_of_model"]}
    cov = None
    if coverage_golden is not None:
        c = coverage_golden[a.name]
        parents = st["parents"]
        init = (parents & np.uint64(0xFFFFFFFFFFFF)) == np.uint64(0xFFFFFFFFFFFF)
        hist = np.bincount((parents[~init] >> np.uint64(56)).astype(np.int64), minlength=a.num_actions)
        cov = {"actions": [{"generated": c["per_action"][n], "distinct": int(hist[i])} for i, n in enumerate(c["actions"])],
               "sites": c["per_site"]}
    compare(a, found, stats=stats, coverage=cov, parents=st["parents"], violation=None, record=None, invariants=[])
    return found


@needs_reference
@pytest.mark.parametrize("name", AUDITED)
def test_audit_accepts_a_clean_store(name, clean_stores, goldens):
    import json
    a, st = clean_stores[name]
    g = goldens[name]
    assert st["widths"] == g["levels"] and len(st["states"]) == g["distinct"]
    cov = json.load(open(os.path.join(ROOT, "tests", "golden", "coverage.json")))
    found = _check(a, st, goldens, cov)
    assert found["generated"] == g["generated"] and found["deadlocks"] == g["deadlocks"]
    assert sum(found["violators_per_level_end"]) == 0


def _corrupt(st, how, a):
    states, parents, widths = st["states"].copy(), st["parents"].copy(), list(st["widths"])
    bounds = np.concatenate([[0], np.cumsum(widths)])
    l3 = int(bounds[2])                                   # first state of level 3
    if how == "parent_off_by_one":
        parents[l3] += np.uint64(1)
    elif how == "swapped_action_ids":
        # two states of level 3 reached by different actions exchange their action ids
        acts = parents[l3:bounds[3]] >> np.uint64(56)
        j = l3 + int(np.argmax(acts != acts[0]))
        assert acts[j - l3] != acts[0]
        lo = np.uint64(0x00FFFFFFFFFFFFFF)
        parents[l3], parents[j] = (parents[l3] & lo) | (acts[j - l3] << np.uint64(56)), (parents[j] & lo) | (acts[0] << np.uint64(56))
    elif how == "dropped_state":
        # the last state of the last level: nothing points at it, only closure can miss it
        states, parents = states[:-1], parents[:-1]
        widths[-1] -= 1
    elif how == "duplicated_state":
        states = np.concatenate([states, states[-1:]])
        parents = np.concatenate([parents, parents[-1:]])
        widths[-1] += 1
    elif how == "swapped_across_levels":
        i, j = l3, int(bounds[3])                        # first of level 3 <-> first of level 4
        states[[i, j]] = states[[j, i]]
        parents[[i, j]] = parents[[j, i]]
    return {"states": states, "parents": parents, "widths": widths, "n_expanded": st["n_expanded"]}


@needs_reference
@pytest.mark.parametrize("name", AUDITED)
@pytest.mark.parametrize("how,check", [("parent_off_by_one", "edges"), ("swapped_action_ids", "edges"),
                                       ("dropped_state", "closure"), ("duplicated_state", "uniqueness"),
                                       ("swapped_across_levels", "edges"), ("wrong_deadlock_count", "totals")])
def test_audit_rejects_a_corrupted_store(name, how, check, clean_stores, goldens):
    from store_audit import AuditError
    a, st = clean_stores[name]
    with pytest.raises(AuditError) as e:
        if how == "wrong_deadlock_count":
            _check(a, st, goldens, deadlocks=goldens[name]["deadlocks"] + 1)
        else:
            _check(a, _corrupt(st, how, a), goldens)
    assert str(e.value).startswith(check + ":"), str(e.value)


@needs_reference
def test_audit_finds_the_first_violating_level(goldens):
    """trunchw_n2 violates its invariants: the violators the audit lists start at the golden's first violation level,
    and the counterexample build_trace's rule picks there is an invariant violation of that level."""
    from store_audit import expected_violation
    a = AuditLib.for_registered("trunchw_n2")
    st = a.host_bfs()
    found = a.check_store(st["states"], st["parents"], st["widths"], st["n_expanded"], check_deadlock=False)
    first = min(l for l in goldens["trunchw_n2"]["first_violation_level"].values() if l)
    want = expected_violation(a, found)
    assert want["kind"] == "invariant" and want["level"] == first
    assert want["count"] == found["violators_per_level_end"][first - 1] and not any(found["violators_per_level_end"][: first - 1])
    assert want["fingerprint"] == min(int(x) for x in want["fps"])


@needs_reference
def test_audit_of_a_bounded_store(goldens):
    """A store that stops after a level end (its last level not expanded) passes; so does closure, level by level."""
    a = AuditLib.for_registered("kip320_n2")
    st = a.host_bfs(stop_after=500)
    assert st["n_expanded"] == len(st["widths"]) - 1
    assert st["widths"] == goldens["kip320_n2"]["levels"][: len(st["widths"])]
    a.check_store(st["states"], st["parents"], st["widths"], st["n_expanded"], check_deadlock=False)


def test_reference_fingerprints_numpy_equals_int():
    from store_audit import (bucket_of, bucket_of_int, fingerprint, fingerprint_int, key_of, key_of_int, owner_of,
                             owner_of_int)
    rng = np.random.default_rng(11)
    for w, bits in ((1, 54), (1, 64), (2, 100), (3, 136), (4, 250)):
        rows = rng.integers(0, 2**64, size=(3000, w), dtype=np.uint64, endpoint=False)
        rows[:5] = np.uint64(2**64 - 1)                 # all-ones words
        rows[5:10] = 0
        fp = fingerprint(rows, bits)
        keys = key_of(rows, fp)
        for i in range(len(rows)):
            words = [int(x) for x in rows[i]]
            f = fingerprint_int(words, bits)
            assert int(fp[i]) == f and (f != 0 or bits <= 63)
            assert tuple(int(x) for x in keys[i]) == key_of_int(words, f)
        mask = (1 << 20) - 1
        assert [int(x) for x in bucket_of(fp, mask)] == [bucket_of_int(int(x), mask) for x in fp]
        for world in (1, 2, 3, 8):
            assert [int(x) for x in owner_of(fp, world)] == [owner_of_int(int(x), world) for x in fp]

