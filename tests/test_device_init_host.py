"""The device form of Init on the host: init_candidate() of the lowered header, compiled for the host (hostmodel.py) and
looped over every candidate of every branch, gives the same multiset of initial states as the host form's table and the
same set as Oracle A; and every Init the device form cannot decode is refused with a LowerError that names the
conjunct."""
import collections
import json
import os

import numpy as np
import pytest

from conftest import ROOT, needs_reference
from hostmodel import HostModel, lower_registered
from oracle_a_actions import init_states as oracle_a_init

from kafka_specification_b200.build import device_init_registry, tla_search_dirs
from kafka_specification_b200.lower.init_device import INIT_DEVICE_THRESHOLD, MAX_BRANCH_CANDIDATES
from kafka_specification_b200.lower.model import lower_model
from kafka_specification_b200.lower.svals import LowerError

SPECS = os.path.join(ROOT, "tests", "specs")
TWINS = [("miniinit", "miniinit_device"), ("miniinit_viol", "miniinit_viol_device"), ("miniinit_sym", "miniinit_sym_device")]


def registry():
    return device_init_registry()


@needs_reference
def test_generated_headers_match_their_digests():
    """Every device-Init test model's header and model.json, byte for byte, against device_init_header_digests.json."""
    from golden.make_header_digests import header_digests
    with open(os.path.join(ROOT, "tests", "golden", "device_init_header_digests.json")) as f:
        golden = json.load(f)
    assert set(golden) == set(registry())
    changed = [name for name, spec in registry().items() if header_digests(name, spec) != golden[name]]
    assert not changed, f"generated code changed for {changed}: rerun tests/golden/make_device_init_digests.py"


def device_solutions(m):
    """(solutions as a (n, W) array, candidates) of the device-form model m, from its header compiled for the host."""
    hm = HostModel.from_lowered(m)
    return hm.init_solutions(), sum(hm.init_space)


def texts(m, rows) -> collections.Counter:
    return collections.Counter(m.state_text([int(x) for x in r]) for r in rows)


@pytest.mark.parametrize("host,device", TWINS)
def test_twin_inits_agree_with_the_host_table_and_oracle_a(host, device):
    mh, md = lower_registered(host), lower_registered(device)
    assert "device" not in mh.init and mh.init_states            # 5,761 candidates: the table, without the hint
    assert md.init["device"] and md.init_states == [] and md.init["candidates"] == 1 + sum(
        b["space"] for b in md.init["branches"][:-1])
    assert md.layout == mh.layout
    rows, cand = device_solutions(md)
    assert cand == md.init["candidates"]
    table = np.array(mh.init_states, dtype=np.uint64)
    assert texts(md, rows) == texts(mh, table)
    # the alternatives of Init and the values of its \E overlap: states are generated more than once
    assert len(rows) > len(set(map(tuple, rows.tolist())))
    spec = registry()[host]
    oracle = oracle_a_init("MiniInit", open(os.path.join(ROOT, spec["cfg"])).read(), [SPECS])
    assert set(oracle) == set(texts(md, rows))


def test_twin_headers_differ_only_in_init():
    """The hint changes Init and nothing else: the same Next, invariants, constraints and symmetry."""
    mh, md = lower_registered("miniinit_sym"), lower_registered("miniinit_sym_device")
    cut = "/* successor enumeration:"
    assert mh.header.split(cut)[1] == md.header.split(cut)[1]
    assert mh.invariants_header.split("\n", 1)[1] == md.invariants_header.split("\n", 1)[1]
    assert mh.digest != md.digest                                  # a checkpoint of one is refused by the other
    assert md.meta()["init"]["device"] and "device" not in mh.meta()["init"]


@needs_reference
def test_type_init_tiny_agrees_with_the_host_form_and_oracle_a():
    md = lower_registered("frl_typeinit_tiny")
    assert md.init["candidates"] == 19683
    rows, cand = device_solutions(md)
    assert cand == 19683 and len(rows) == 343
    spec = registry()["frl_typeinit_tiny"]
    cfg_text = open(os.path.join(ROOT, spec["cfg"])).read()
    host_text = cfg_text.replace("\\* kspec: INIT DEVICE\n", "")
    assert host_text != cfg_text
    mh = lower_model("MCFrlTypeInit", tla_search_dirs(), host_text, name="frl_typeinit_tiny_host")
    assert "device" not in mh.init
    assert texts(md, rows) == texts(mh, np.array(mh.init_states, dtype=np.uint64))
    assert oracle_a_init("MCFrlTypeInit", cfg_text, tla_search_dirs()) == texts(md, rows)


@needs_reference
def test_type_init_3x4x2_is_the_closed_form():
    """FiniteReplicatedLog's TypeOk is inductive: its solutions are the 29,791 reachable states of frl_3x4x2."""
    from golden.make_golden import state_digest
    md = lower_registered("frl_typeinit_3x4x2")
    assert md.init["device"] and md.init["candidates"] == 66430125 > INIT_DEVICE_THRESHOLD   # no hint in the cfg
    rows, cand = device_solutions(md)
    assert cand == 66430125 and len(rows) == 29791 == len(set(map(tuple, rows.tolist())))
    goldens = json.load(open(os.path.join(ROOT, "tests", "golden", "goldens.json")))
    assert state_digest([md.state_text([int(x) for x in r]) for r in rows]) == goldens["frl_3x4x2"]["state_digest"]


@needs_reference
def test_type_init_3x4x3_candidate_count():
    md = lower_registered("frl_typeinit_3x4x3")
    assert md.init["candidates"] == 1280 ** 3 == 2097152000
    assert "INIT_SPACE[INIT_BRANCHES] = {2097152000ull}" in md.header


REFUSE_TLA = """---- MODULE Refuse ----
EXTENDS Integers
VARIABLES x, y
TypeOk == x \\in 0 .. 2 /\\ y \\in 0 .. 2
Next == UNCHANGED <<x, y>>
FromNat == x \\in Nat /\\ y = 0
FromInt == x \\in Int /\\ y = 0
OnState == x \\in 0 .. 2 /\\ y \\in 0 .. x
OnBound == \\E k \\in 0 .. 2 : x \\in 0 .. k /\\ y = 0
ReadEarly == y > 0 /\\ x \\in 0 .. 2 /\\ y \\in 0 .. 2
Huge == x \\in 0 .. 2 /\\ y = 0 /\\ \\E f \\in [1 .. 13 -> 0 .. 9] : f[1] = x
Overlap == x \\in 0 .. 2 /\\ y = 0 /\\ \\E r \\in [a : 0 .. 1] \\union [a : 1 .. 2] : r.a = x
====
"""


@pytest.mark.parametrize("init,message", [
    ("FromNat", r"'x \\in Nat': a generator over Nat is unbounded"),
    ("FromInt", r"'x \\in Int': a generator over Int is unbounded"),
    ("OnState", r"'y \\in 0 \.\. x': its generator set depends on a state variable"),
    ("OnBound", r"its generator set depends on a bound variable"),
    ("ReadEarly", r"'y > 0': variable y' read before it is assigned"),
    ("Huge", "an Init branch has 30,000,000,000,000 candidates, more than the device form enumerates "
             f"\\({MAX_BRANCH_CANDIDATES:,}\\)"),
    ("Overlap", r"a union of sets of the same kind \(rec:a\) may overlap"),
])
def test_device_form_refusals(init, message, tmp_path):
    (tmp_path / "Refuse.tla").write_text(REFUSE_TLA)
    cfg = f"\\* kspec: INIT DEVICE\nINIT {init}\nNEXT Next\nINVARIANT TypeOk\n"
    with pytest.raises(LowerError, match=message):
        lower_model("Refuse", [str(tmp_path)], cfg)
