"""Every generator form of the device form of Init, on the host (MiniDecode.tla).  The small cfgs against their host-table
twins (the multiset of solutions, and the whole host BFS level by level) and against Oracle A; the cfgs of 2^32 and
more candidates candidate by candidate, at 0, around 2^32, at the last index and at random indices, against a plain
mixed-radix decode written from the spec (init_forms.py); and a layout narrower than some solutions, which traps the
host BFS unless a filter rejects exactly those candidates first."""
import collections
import os
import random

import numpy as np
import pytest

from conftest import ROOT
from hostmodel import HostModel, lower_registered
from init_forms import LARGE, SPACE, boundary_indices, decode, solution_indices
from oracle_a_actions import init_states as oracle_a_init

from kafka_specification_b200.build import device_init_registry
from kafka_specification_b200.runtime import StateDecoder

SPECS = os.path.join(ROOT, "tests", "specs")
TWINS = [("minidecode_leaves", "minidecode_leaves_device"), ("minidecode_shapes", "minidecode_shapes_device")]
KMC_FAIL_LAYOUT = 1


def host(name) -> HostModel:
    return HostModel.from_lowered(lower_registered(name))


def texts(name, rows) -> collections.Counter:
    return collections.Counter(StateDecoder(lower_registered(name).meta()).texts(rows))


def test_forms_reach_the_generated_code():
    """What the cfgs are for, checked in the headers they lower to, so that a change of the spec or of the lowering
    cannot quietly drop a form."""
    leaves, shapes = lower_registered("minidecode_leaves_device"), lower_registered("minidecode_shapes_device")
    # the \E branch, the constant-FALSE branch, a branch of 1 candidate and one of fewer than 32
    assert [b["space"] for b in leaves.init["branches"]] == [576, 10, 1, 10]
    false_branch = leaves.header.split("init_candidate_1(")[1].split("\n}\n")[0]
    assert "return false;" in false_branch and "out.w" not in false_branch
    assert [b["space"] for b in shapes.init["branches"]] == [12960, 12960]
    for name in LARGE:
        m = lower_registered(name)
        assert m.init["device"] and [b["space"] for b in m.init["branches"]] == [SPACE[name]]
    # 64-bit digits above 2^32 candidates, 32-bit ones at exactly 2^32, a 64-bit SUBSET digit
    assert "ull" in lower_registered("minidecode_ranges").header
    assert "(unsigned)idx" in lower_registered("minidecode_edge").header
    assert "(uint64_t)(idx" in lower_registered("minidecode_subsets").header


@pytest.mark.parametrize("table,device", TWINS)
def test_small_forms_agree_with_the_host_table_and_oracle_a(table, device):
    mt, md = lower_registered(table), lower_registered(device)
    assert "device" not in mt.init and md.init["device"] and md.layout == mt.layout
    hd = host(device)
    assert sum(hd.init_space) == md.init["candidates"] <= 65536
    got = texts(device, hd.init_solutions())
    assert got == texts(table, np.array(mt.init_states, dtype=np.uint64))
    spec = device_init_registry()[table]
    with open(os.path.join(ROOT, spec["cfg"])) as f:
        assert set(oracle_a_init("MiniDecode", f.read(), [SPECS])) == set(got)


@pytest.mark.parametrize("table,device", TWINS)
def test_host_bfs_of_the_device_form_is_the_table_forms(table, device):
    """The host BFS seeded from init_candidate() and the one seeded from the table: totals, levels, each level's states."""
    ht, hd = host(table), host(device)
    rt, rd = ht.bfs(), hd.bfs()
    assert rd["complete"] and rd["fail"] == 0 and len(rd["widths"]) > 1
    for k in ("generated", "deadlocks", "widths", "n_expanded", "action_generated", "first_invariant"):
        assert rd[k] == rt[k], k
    first = 0
    for w in rt["widths"]:
        a, b = (sorted(map(tuple, r["states"][first:first + w].tolist())) for r in (rt, rd))
        assert a == b
        first += w


@pytest.mark.parametrize("name", LARGE)
def test_pointwise_decode_at_the_boundaries(name):
    """init_candidate() of the large cfgs against init_forms.decode at the indices where a 32-bit index or digit would
    wrap, at the last index and at 300 random ones (a fixed seed)."""
    hm = host(name)
    assert hm.init_space == [SPACE[name]]
    dec = StateDecoder(lower_registered(name).meta())
    rng = random.Random(20261018)
    idxs = boundary_indices(name) + [rng.randrange(SPACE[name]) for _ in range(300)]
    idxs += [rng.choice(solution_indices(name)) for _ in range(300)]
    # solutions in the top half of the 32-bit range and (above 2^32 candidates) past it
    assert any(i >= 1 << 31 and decode(name, i) for i in idxs)
    assert SPACE[name] <= 1 << 32 or any(i >= 1 << 32 and decode(name, i) for i in idxs)
    for i in idxs:
        status, words = hm.init_candidate(0, i)
        want = decode(name, i)
        got = dec.text([int(x) for x in words]) if status == "solution" else None
        assert status != "trapped" and got == want, f"{name} candidate {i}: {got!r} != {want!r}"


@pytest.mark.parametrize("name", LARGE)
def test_closed_form_solutions_are_distinct_solutions(name):
    hm = host(name)
    rows = []
    for i in solution_indices(name):
        status, words = hm.init_candidate(0, i)
        assert status == "solution", i
        rows.append(tuple(int(x) for x in words))
    assert len(set(rows)) == len(rows) == {"minidecode_ranges": 65537 * 4, "minidecode_edge": 65536,
                                           "minidecode_subsets": 35}[name]


def test_a_layout_narrower_than_a_solution_traps_and_a_rejected_candidate_does_not():
    """Under LAYOUT NarrowOk (a \\in -2 .. 4), the solutions of Leaves with a = 9 trap; LeavesFit rejects exactly those
    candidates before packing, so nothing traps and its solutions are Leaves' others."""
    leaves, narrow, fit = host("minidecode_leaves_device"), host("minidecode_narrow"), host("minidecode_narrow_fit")
    assert narrow.init_space == fit.init_space == leaves.init_space
    dec = StateDecoder(lower_registered("minidecode_leaves_device").meta())
    trapped = 0
    for b, space in enumerate(leaves.init_space):
        for i in range(space):
            want, words = leaves.init_candidate(b, i)
            too_wide = want == "solution" and dec.decode([int(x) for x in words])["a"] > 4
            trapped += too_wide
            assert narrow.init_candidate(b, i)[0] == ("trapped" if too_wide else want)
            assert fit.init_candidate(b, i)[0] == ("rejected" if too_wide else want)
    assert trapped > 0
    r = narrow.bfs()
    assert r["fail"] == KMC_FAIL_LAYOUT and not r["complete"] and r["widths"] == []
    with pytest.raises(RuntimeError, match="traps the layout"):
        narrow.init_solutions()
    r = fit.bfs()
    assert r["complete"] and r["fail"] == 0
    assert texts("minidecode_narrow_fit", fit.init_solutions()) == collections.Counter(
        {t: c for t, c in texts("minidecode_leaves_device", leaves.init_solutions()).items()
         if int(t.split("\n")[0].split(" = ")[1]) <= 4})
