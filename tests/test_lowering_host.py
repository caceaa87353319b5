"""The AOT lowering, compiled for the HOST by the test harness, against the goldens.

This exercises exactly the header the CUDA engine includes (same expand / invariant / constraint
code, same packed layout) on a machine without a GPU.  The harness (tests/support/host_model.cpp)
is test infrastructure: no product path runs on the CPU.
"""
import os

import numpy as np
import pytest

from conftest import REFERENCE, ROOT, needs_reference
from golden.make_golden import state_digest
from hostmodel import lower_model, run_host

DIRS = [REFERENCE, os.path.join(ROOT, "models")]

SMALL = ["idsequence", "frl_tiny", "frl_3x4x2", "kip320_n2", "trunchw_n2", "kip101_n2", "kip279_n2", "firsttry_n2",
         "asyncisr_v2", "asyncisr_small", "kip320sym_n2"]
MEDIUM = ["kip320_small", "trunchw_small", "kip101_small", "kip279_small", "firsttry_small", "kip320sym_small",
          "kip320_with279_small", "asyncisr_w3"]
if os.environ.get("KSPEC_SLOW_TESTS") == "1":
    MEDIUM.append("frl_3x4x3")       # 28 M successors on the sequential host harness: 2 more minutes (digest verified once, round 2)


def _lower(registry, name):
    spec = registry[name]
    return lower_model(spec["module"], DIRS, open(os.path.join(ROOT, spec["cfg"])).read(), name=name)


@needs_reference
@pytest.mark.parametrize("name", SMALL)
def test_lowered_model_matches_golden_state_for_state(name, goldens, registry):
    g = goldens[name]
    m = _lower(registry, name)
    assert not m.warnings
    r = run_host(m, dump=True, max_states=200000)
    assert r["fail"] == 0 and r["complete"]
    for k in ("distinct", "generated", "depth", "levels", "deadlocks"):
        assert r[k] == g[k], k
    assert r["max_fanout_seen"] <= m.max_fanout
    if "state_digest" in g:
        texts = [m.state_text(row) for row in r["states"]]
        assert len(set(texts)) == g["distinct"]
        assert state_digest(texts) == g["state_digest"]
    # first violated invariant (cfg order) appears at the level the oracles report
    levels = {i: l for i, l in g["first_violation_level"].items() if l is not None and i in m.invariants}
    if levels:
        assert r["first_violated_level"] == min(levels.values())
    else:
        assert r["first_violated"] is None


@needs_reference
@pytest.mark.parametrize("name", MEDIUM)
def test_lowered_model_matches_golden_counts(name, goldens, registry):
    """The 3-replica models (10^5..10^6 states): counts against the golden and -- where Oracle A, the interpreter of the
    unchanged .tla text, has been run over the model (hours of Python, tests/golden/run_oracle_a.py) -- the reachable
    state SET, decoded to TLC text, against its order-independent digest."""
    from kafka_specification_b200.runtime import StateDecoder
    g = goldens[name]
    m = _lower(registry, name)
    want_digest = "state_digest" in g
    r = run_host(m, max_states=3_000_000, dump=want_digest)
    for k in ("distinct", "generated", "depth", "levels", "deadlocks"):
        assert r[k] == g[k], k
    if want_digest:
        assert "oracle_a" in g["sources"]
        texts = StateDecoder(m.meta()).texts(np.array(r["states"], dtype=np.uint64))
        assert len(texts) == g["distinct"] and state_digest(texts) == g["state_digest"]


@needs_reference
def test_layout_roundtrip_and_init(registry):
    m = _lower(registry, "kip320_small")
    lay = m.lowerer.layout
    assert m.words == lay.words and len(m.init_states) == 1
    st = m.decode_state(m.init_states[0])
    assert lay.py_pack(st) == m.init_states[0]
    # the runtime decoder (model.json only) agrees with the lowering's own decoder
    from kafka_specification_b200.runtime import StateDecoder
    dec = StateDecoder(m.meta())
    r = run_host(m, dump=True, max_states=5000)
    for row in r["states"][:500]:
        assert dec.decode(row) == m.decode_state(row)
        assert lay.py_pack(m.decode_state(row)) == [int(x) for x in row]


@needs_reference
def test_pinning_preserves_tlc_multiplicity(registry):
    """Kip279.tla:47-51 and Kip320.tla:82-83 generate the same successor twice; 'generated' counts both."""
    import kso
    for name, model in (("kip279_n2", "kip279"), ("kip320_n2", "kip320")):
        m = _lower(registry, name)
        assert run_host(m)["generated"] == kso.run(model, [2, 2, 2, 2], max_states=100000)["generated"]


@needs_reference
def test_layout_overflow_is_trapped():
    """A layout too narrow for a reachable value must trap (KMC_FAIL_LAYOUT), never wrap."""
    cfg = """CONSTANTS Replicas = {r1, r2} LogSize = 2 MaxRecords = 2 MaxLeaderEpoch = 2
INIT Init NEXT Next INVARIANT TypeOk CHECK_DEADLOCK FALSE
\\* kspec: CAPACITY leaderAndIsrRequests = 1
"""
    m = lower_model("Kip320", DIRS, cfg, name="kip320_narrow")
    r = run_host(m)
    assert r["fail"] == 1 and not r["complete"]


@needs_reference
def test_unbounded_layout_is_rejected():
    from kafka_specification_b200.lower.svals import LowerError
    cfg = """CONSTANTS Replicas = {r1, r2} Leader = r1 MaxOffset = 1
INIT Init NEXT Next INVARIANT ValidHighWatermark CHECK_DEADLOCK FALSE"""
    with pytest.raises(LowerError):
        lower_model("AsyncIsr", DIRS, cfg)       # TypeOk uses Nat (AsyncIsr.tla:42-55): needs a LAYOUT operator


@needs_reference
def test_false_assume_is_rejected():
    from kafka_specification_b200.lower.svals import LowerError
    with pytest.raises(LowerError):              # AsyncIsr.tla:27-29: MaxOffset > 0
        lower_model("MCAsyncIsr", DIRS, open(os.path.join(ROOT, "models", "MCAsyncIsr.cfg")).read().replace(
            "MaxOffset = 2", "MaxOffset = 0"))


@needs_reference
@pytest.mark.parametrize("name", ["frl_tiny", "kip320_n2", "kip279_n2", "firsttry_n2", "asyncisr_v2", "kip320_small"])
def test_two_phase_item_form_equals_expand(name, goldens, registry):
    """item_guard/item_body (what the CUDA expand kernel runs) enumerate exactly expand()'s successors."""
    g = goldens[name]
    m = _lower(registry, name)
    r = run_host(m, max_states=3_000_000, items=True)
    for k in ("distinct", "generated", "depth", "levels", "deadlocks"):
        assert r[k] == g[k], k


@needs_reference
def test_symmetry_reduction_counts_orbits(goldens, registry):
    """SYMMETRY Permutations(Replicas): the set holds one representative per orbit; the orbit count
    lies between |states| / n! and |states|, and every count equals both oracles'."""
    full, sym = goldens["kip320_small"], goldens["kip320sym_small"]
    assert full["distinct"] / 6 <= sym["distinct"] < full["distinct"]
    assert sym["depth"] == full["depth"]
    m = _lower(registry, "kip320sym_small")
    r = run_host(m, max_states=1_000_000)
    assert (r["distinct"], r["generated"], r["levels"]) == (sym["distinct"], sym["generated"], sym["levels"])
