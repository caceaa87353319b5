"""MiniWide (tests/specs/MiniWide.tla) on the CPU: its cfgs pack to the widths and set-key forms that test_zz_wide_states.py
runs on the GPU, and the lowered model compiled for the host agrees with Oracle A and with the closed form there.

    miniwide_one64     W = 1, all 64 bits used: the engine hashes the one-word key (no bijection)
    miniwide_two128    W = 2, can pack to all-ones: the engine keys the set by the 128-bit fingerprint
    miniwide_w5/6/7    W = 5, 6, 7 (the expand kernel's tile holds SPT = 2, 1, 1 states per thread)
    miniwide_w6_sym    W = 6 under SYMMETRY
    *_large            levels of 10^5 states and more; checked against the closed form and the host BFS only
A state that packs into more than 7 words is refused by the lowering (MiniWide_w8.cfg)."""
import os

import pytest

from conftest import ROOT
from golden.make_golden import closed_form, state_digest
from hostmodel import HostModel, lower_registered, run_host
from kafka_specification_b200.build import registry, tla_search_dirs
from kafka_specification_b200.frontend.cfg import parse_cfg
from kafka_specification_b200.lower.model import lower_model
from kafka_specification_b200.lower.svals import LowerError
from store_audit import host_audit

REGISTRY = registry()
# name: (words, state bits, can pack to all-ones)
SHAPES = {"miniwide_one64": (1, 64, True), "miniwide_two128": (2, 128, True), "miniwide_w5": (5, 306, True),
          "miniwide_w6": (6, 357, False), "miniwide_w7": (7, 408, False), "miniwide_w6_sym": (6, 357, False),
          "miniwide_w5_large": (5, 306, True), "miniwide_w6_large": (6, 357, False),
          "miniwide_w7_large": (7, 408, False)}
SMALL = ["miniwide_one64", "miniwide_two128", "miniwide_w5", "miniwide_w6", "miniwide_w7"]
LARGE = ["miniwide_w5_large", "miniwide_w6_large", "miniwide_w7_large"]


def cfg_of(name):
    return parse_cfg(open(os.path.join(ROOT, REGISTRY[name]["cfg"])).read())


def test_every_miniwide_cfg_is_listed():
    assert sorted(n for n, s in REGISTRY.items() if s["module"] == "MiniWide") == sorted(SHAPES)
    assert all(REGISTRY[n].get("large") for n in LARGE)


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_cfg_lowers_to_its_width(name):
    """A spec or layout change that narrows these cfgs would silently take the GPU tests off the paths they are for."""
    words, bits, all_ones = SHAPES[name]
    m = lower_registered(name)
    assert (m.words, m.state_bits, m.lowerer.layout.all_ones_possible) == (words, bits, all_ones)
    hm = HostModel.from_lowered(m)
    assert (hm.words, hm.state_bits, hm.all_ones_possible) == (words, bits, all_ones)


def test_eight_words_are_refused_by_the_lowering():
    with open(os.path.join(ROOT, "tests", "specs", "MiniWide_w8.cfg")) as f:
        text = f.read()
    with pytest.raises(LowerError, match=r"packs into 8 64-bit words .* at most 7 words"):
        lower_model("MiniWide", tla_search_dirs(), text, name="miniwide_w8")


@pytest.mark.parametrize("name", ["miniwide_one64", "miniwide_two128"])
def test_golden_is_oracle_a(name, goldens):
    """The committed golden is what Oracle A computes now (the two small enough to interpret in a second)."""
    import tla_interp
    text = open(os.path.join(ROOT, REGISTRY[name]["cfg"])).read()
    a = tla_interp.run_bfs("MiniWide", tla_search_dirs(), text + "\nCHECK_DEADLOCK FALSE\n", collect_states=True,
                           stop_on_violation=False)
    g = goldens[name]
    for k in ("distinct", "generated", "depth", "levels", "deadlocks", "out_of_model", "first_violation_level"):
        assert g[k] == a[k], k
    assert g["state_digest"] == state_digest(a["states"])


@pytest.mark.parametrize("name", SMALL)
def test_golden_is_the_closed_form(name, goldens):
    g, cf = goldens[name], closed_form("MiniWide", cfg_of(name))
    assert "oracle_a" in g["sources"] and "closed_form" in g["sources"]
    for k in ("distinct", "generated", "depth", "levels", "deadlocks", "out_of_model", "first_violation_level"):
        assert g[k] == cf[k], k


@pytest.mark.parametrize("items", [False, True])
@pytest.mark.parametrize("name", SMALL + ["miniwide_w6_sym"])
def test_host_bfs_is_oracle_a_state_for_state(name, items, goldens):
    """Through expand() and through the two-phase form the expand kernel runs: Oracle A's counts and, without SYMMETRY,
    its set of states (the golden's digest)."""
    g = goldens[name]
    m = lower_registered(name)
    r = run_host(m, dump=True, items=items)
    assert r["complete"] and not r["fail"]
    assert (r["distinct"], r["generated"], r["depth"], r["levels"], r["deadlocks"]) == (
        g["distinct"], g["generated"], g["depth"], g["levels"], g["deadlocks"])
    assert r["first_violation_level"] == g["first_violation_level"]
    if name != "miniwide_w6_sym":
        assert state_digest([m.state_text(row) for row in r["states"]]) == g["state_digest"]


@pytest.mark.parametrize("name", SMALL + LARGE)
def test_host_bfs_and_audit_are_the_closed_form(name):
    """Widths, generated, deadlocks and out_of_model of the host BFS's store (recomputed by the audit from the stored
    states), and the per-invariant report, against the closed form."""
    cf = closed_form("MiniWide", cfg_of(name))
    a, st, found = host_audit(name, sites=False)
    assert st["widths"] == cf["levels"] and len(st["states"]) == cf["distinct"]
    assert (found["generated"], found["deadlocks"], found["out_of_model"]) == (
        cf["generated"], cf["deadlocks"], cf["out_of_model"])
    assert found["violators_per_level_end"][cf["first_violation_level"]["FewFull"] - 1] == cf["violators_first_level"]["FewFull"]
    m = lower_registered(name)
    rep = a.invariant_report(m.invariants)
    assert rep.pop(None) == 0
    assert list(rep) == ["FewFull"]
    assert rep["FewFull"]["level"] == cf["first_violation_level"]["FewFull"]
    assert rep["FewFull"]["violators_first_level"] == cf["violators_first_level"]["FewFull"]
