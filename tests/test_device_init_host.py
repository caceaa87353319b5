"""The device form of Init on the host: init_candidate() of the lowered header, compiled with g++ and looped over every
candidate of every branch, gives the same multiset of initial states as the host form's table and the same set as
Oracle A; and every Init the device form cannot decode is refused with a LowerError that names the conjunct."""
import collections
import ctypes
import functools
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, needs_reference

from kafka_specification_b200.build import device_init_registry, tla_search_dirs
from kafka_specification_b200.lower.init_device import INIT_DEVICE_THRESHOLD, MAX_BRANCH_CANDIDATES
from kafka_specification_b200.lower.model import lower_model
from kafka_specification_b200.lower.svals import LowerError

SPECS = os.path.join(ROOT, "tests", "specs")
TWINS = [("miniinit", "miniinit_device"), ("miniinit_viol", "miniinit_viol_device"), ("miniinit_sym", "miniinit_sym_device")]



def registry():
    return device_init_registry()


@functools.lru_cache(maxsize=None)
def lower_registered(name):
    """A model of tests/specs/MODELS_device_init.json lowered as build() lowers it."""
    spec = registry()[name]
    with open(os.path.join(ROOT, spec["cfg"])) as f:
        return lower_model(spec["module"], tla_search_dirs(), f.read(), name=name)


@needs_reference
def test_generated_headers_match_their_digests():
    """Every device-Init test model's header and model.json, byte for byte, against device_init_header_digests.json."""
    from golden.make_header_digests import header_digests
    with open(os.path.join(ROOT, "tests", "golden", "device_init_header_digests.json")) as f:
        golden = json.load(f)
    assert set(golden) == set(registry())
    changed = [name for name, spec in registry().items() if header_digests(name, spec) != golden[name]]
    assert not changed, f"generated code changed for {changed}: rerun tests/golden/make_device_init_digests.py"


DRIVER = r"""
#include <stdint.h>
#include KMC_MODEL_HEADER
using namespace kmc_model;
// every candidate of every branch: the solutions' words (up to cap of them), the number of solutions, the candidates
extern "C" uint64_t enumerate_init(uint64_t* out, uint64_t cap, uint64_t* candidates, unsigned* fail_out) {
  uint64_t n = 0, c = 0;
  for (int b = 0; b < INIT_BRANCHES; ++b)
    for (uint64_t i = 0; i < INIT_SPACE[b]; ++i, ++c) {
      State s;
      unsigned fail = 0;
      if (init_candidate(b, i, s, fail)) {
        if (n < cap)
          for (int k = 0; k < W; ++k) out[n * W + k] = s.w[k];
        ++n;
      }
      if (fail) *fail_out = fail;
    }
  *candidates = c;
  return n;
}
"""


def device_solutions(m, tmp_path, cap=1 << 20):
    """(solutions as a (n, W) array, candidates) of the device-form model m, from its header compiled for the host."""
    hdr, src, so = tmp_path / f"{m.name}.h", tmp_path / "driver.cpp", tmp_path / f"{m.name}.so"
    hdr.write_text(m.header)
    src.write_text(DRIVER)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", f'-DKMC_MODEL_HEADER="{hdr}"', str(src), "-o", str(so)])
    lib = ctypes.CDLL(str(so))
    lib.enumerate_init.restype = ctypes.c_uint64
    out = np.zeros((cap, m.words), dtype=np.uint64)
    cand, fail = ctypes.c_uint64(), ctypes.c_uint(0)
    n = lib.enumerate_init(out.ctypes.data_as(ctypes.c_void_p), cap, ctypes.byref(cand), ctypes.byref(fail))
    assert fail.value == 0 and n <= cap
    return out[:n], cand.value


def texts(m, rows) -> collections.Counter:
    return collections.Counter(m.state_text([int(x) for x in r]) for r in rows)


def oracle_a_init(module, cfg_text, dirs) -> collections.Counter:
    import tla_interp
    from kafka_specification_b200.frontend.cfg import parse_cfg
    from kafka_specification_b200.frontend.modules import load_root
    from kafka_specification_b200.frontend.values import fmt
    cfg = parse_cfg(cfg_text)
    root = load_root(module, dirs)
    it = tla_interp.Interp(root, cfg)
    init_e, _ = tla_interp.resolve_init_next(root, cfg)
    return collections.Counter("\n".join(f"/\\ {v} = {fmt(st[v])}" for v in it.variables) for st in it.init_states(init_e))


@pytest.mark.parametrize("host,device", TWINS)
def test_twin_inits_agree_with_the_host_table_and_oracle_a(host, device, tmp_path):
    mh, md = lower_registered(host), lower_registered(device)
    assert "device" not in mh.init and mh.init_states            # 5,761 candidates: the table, without the hint
    assert md.init["device"] and md.init_states == [] and md.init["candidates"] == 1 + sum(
        b["space"] for b in md.init["branches"][:-1])
    assert md.layout == mh.layout
    rows, cand = device_solutions(md, tmp_path)
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
def test_type_init_tiny_agrees_with_the_host_form_and_oracle_a(tmp_path):
    md = lower_registered("frl_typeinit_tiny")
    assert md.init["candidates"] == 19683
    rows, cand = device_solutions(md, tmp_path)
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
def test_type_init_3x4x2_is_the_closed_form(tmp_path):
    """FiniteReplicatedLog's TypeOk is inductive: its solutions are the 29,791 reachable states of frl_3x4x2."""
    from golden.make_golden import state_digest
    md = lower_registered("frl_typeinit_3x4x2")
    assert md.init["device"] and md.init["candidates"] == 66430125 > INIT_DEVICE_THRESHOLD   # no hint in the cfg
    rows, cand = device_solutions(md, tmp_path)
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
