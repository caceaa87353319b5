"""The per-invariant report of -continue runs, without a GPU: the lowering's violated_invariants() (invariants.h) against
the goldens and against first_violated_invariant, the >64-invariant fallback, and the CLI's error blocks."""
import os
import random

import pytest

from conftest import REFERENCE, ROOT, needs_reference
from hostmodel import HostModel, lower_model

DIRS = [REFERENCE, os.path.join(ROOT, "models"), os.path.join(ROOT, "tests", "specs")]


def _registry():
    from kafka_specification_b200.build import registry
    return registry()


def _lower(name):
    spec = _registry()[name]
    with open(os.path.join(ROOT, spec["cfg"])) as f:
        return lower_model(spec["module"], DIRS, f.read(), name=name)


ORACLE_A_MODELS = sorted(n for n, s in _registry().items() if s.get("oracle_a"))


@needs_reference
@pytest.mark.parametrize("name", ORACLE_A_MODELS)
def test_host_bfs_by_mask_gives_every_first_violation_level(name, goldens):
    """A host BFS of the lowered model that checks states through violated_invariants() finds each invariant's first
    violating level as the goldens record it (Oracle A's, and Oracle B's where it ran), constraint-discarded violators
    included; and on every checked state the mask agrees with first_violated_invariant."""
    m = _lower(name)
    rep = HostModel.from_lowered(m).invariant_report(m.invariants)
    assert rep.pop(None) == 0, "violated_invariants and first_violated_invariant disagree on a checked state"
    want = {i: l for i, l in goldens[name]["first_violation_level"].items() if l is not None}
    assert {i: r["level"] for i, r in rep.items()} == want
    for r in rep.values():
        assert 1 <= r["violators_first_level"] <= r["violators"]


@needs_reference
def test_two_invariants_at_one_level_and_a_discarded_only_violation(goldens):
    """minibound_mixed breaks NotOver and OneFull at level 3; asyncisr_bounded breaks VersionInBound only through
    successors its CONSTRAINT discards (the stored states never violate it)."""
    mixed = _lower("minibound_mixed")
    rep = HostModel.from_lowered(mixed).invariant_report(mixed.invariants)
    assert rep["NotOver"]["level"] == rep["OneFull"]["level"] == 3
    m = _lower("asyncisr_bounded")
    hm = HostModel.from_lowered(m)
    rep = hm.invariant_report(m.invariants)
    assert rep["VersionInBound"]["level"] == goldens["asyncisr_bounded"]["first_violation_level"]["VersionInBound"]
    r = hm.bfs()
    bit = 1 << m.invariants.index("VersionInBound")
    assert not any(hm.mask(s) & bit for s in r["states"])


# the walks of test_oracles_sampled.py, with Oracle A's verdict on every invariant of every state
WALKS = [("kip320_3x4_r4e3", 2, 45), ("trunchw_3x4_r3e3", 2, 40), ("firsttry_3x4_r3e3", 2, 40),
         ("kip320_with279_small", 2, 30), ("asyncisr_deep", 2, 45)]


@needs_reference
@pytest.mark.parametrize("name,walks,steps", WALKS)
def test_mask_on_random_walks_matches_oracle_a_and_first_violated(name, walks, steps):
    import tla_interp
    from kafka_specification_b200.frontend.cfg import parse_cfg
    from kafka_specification_b200.frontend.modules import load_root
    spec = _registry()[name]
    cfg_text = open(os.path.join(ROOT, spec["cfg"])).read()
    m = lower_model(spec["module"], DIRS, cfg_text, name=name)
    hm = HostModel.from_lowered(m)
    cfg = parse_cfg(cfg_text)
    it = tla_interp.Interp(load_root(spec["module"], DIRS), cfg)
    rng = random.Random(20260923 + len(name))
    inits = list(hm.init_states())
    for _ in range(walks):
        cur = inits[rng.randrange(len(inits))].copy()
        for _ in range(steps):
            st = m.decode_state(cur)
            mask = hm.mask(cur)
            want = sum(1 << i for i, inv in enumerate(cfg.invariants) if not it.eval_named_predicate(inv, st))
            assert mask == want, (name, m.state_text(cur))
            first = hm.first_violated(cur)
            assert first == ((mask & -mask).bit_length() - 1 if mask else -1)
            rows, _ = hm.successors(cur)
            nxt = [r for r in rows if hm.in_model(r)]
            if not nxt:
                break
            cur = nxt[rng.randrange(len(nxt))].copy()


@needs_reference
def test_more_than_64_invariants_lower_without_a_mask():
    """A cfg with 65 INVARIANT entries lowers and runs as before (model.h does not depend on invariants.h); its
    invariants.h says there is no mask, and the engine then reports no per-invariant results (KMC_E_BADARG)."""
    spec = _registry()["minibound_mixed"]
    cfg_text = open(os.path.join(ROOT, spec["cfg"])).read() + "\nINVARIANT\n" + "\n".join(["TypeOk"] * 65) + "\n"
    m = lower_model(spec["module"], DIRS, cfg_text, name="minibound_65")
    assert len(m.invariants) > 64
    assert "HAS_INVARIANT_MASK = false" in m.invariants_header
    assert "violated_invariants" not in m.header and "first_violated_invariant" in m.header
    small = _lower("minibound_mixed")
    assert "HAS_INVARIANT_MASK = true" in small.invariants_header
    assert small.meta() == _lower("minibound_mixed").meta() and "invariants_header" not in small.meta()


def _trace(n):
    return [{"action": None if i == 0 else {"name": f"A{i}", "module": "M"}, "text": f"/\\ x = {i}"} for i in range(n)]


def _report(name, index, level):
    return {"invariant": name, "index": index, "level": level, "trace": _trace(level)}


def test_cli_blocks_are_ordered_by_level_then_cfg_index():
    from kafka_specification_b200.tlc2 import EXIT_VIOLATION_SAFETY, error_messages
    reports = [_report("StrongIsr", 2, 13), _report("WeakIsr", 1, 12), _report("Aaa", 3, 12)]
    violation = {"kind": "invariant", "invariant": "WeakIsr", "level": 12, "trace_len": 12}
    blocks, code = error_messages(violation, _trace(12), reports)
    assert code == EXIT_VIOLATION_SAFETY
    heads = [t for k, t, _ in blocks if k == "inv_behavior"]
    assert heads == ["Error: Invariant WeakIsr is violated.", "Error: Invariant Aaa is violated.",
                     "Error: Invariant StrongIsr is violated."]
    kinds = [k for k, _, _ in blocks]
    assert kinds == (["inv_behavior", "behavior"] + ["state"] * 12) * 2 + ["inv_behavior", "behavior"] + ["state"] * 13
    assert [c for _, _, c in blocks] == [1 if k != "state" else 4 for k in kinds]
    # without reports (no -continue), the one block of the run's violation, as before
    one, code = error_messages(violation, _trace(12), [])
    assert one == blocks[:14] and code == EXIT_VIOLATION_SAFETY
    assert blocks[2][1] == "State 1: <Initial predicate>\n/\\ x = 0\n"
    assert blocks[3][1] == "State 2: <A1 of module M>\n/\\ x = 1\n"


def test_cli_initial_state_block_and_deadlock_first():
    from kafka_specification_b200.tlc2 import EXIT_OK, EXIT_VIOLATION_DEADLOCK, error_messages
    blocks, _ = error_messages(None, [], [_report("TypeOk", 0, 1)])
    assert [k for k, _, _ in blocks] == ["inv_initial", "state"]
    assert blocks[0][1] == "Error: Invariant TypeOk is violated by the initial state:"
    dead = {"kind": "deadlock", "invariant": None, "level": 4, "trace_len": 4}
    blocks, code = error_messages(dead, _trace(4), [_report("NotOver", 1, 3)])
    assert code == EXIT_VIOLATION_DEADLOCK
    assert [k for k, _, _ in blocks] == ["deadlock", "behavior"] + ["state"] * 4 + ["inv_behavior", "behavior"] + ["state"] * 3
    assert error_messages(None, [], []) == ([], EXIT_OK)
