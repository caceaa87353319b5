"""GPU tests written after this round's GPU budget was spent: they have CPU-side evidence only (the lowered models
agree with Oracle A / Oracle B on the host, tests/test_generic_frontend.py and the goldens' `sources`) and no GPU
verdict yet.  The file name and tests/conftest.py make them run LAST, so that -x cannot let them hide the
verdicts of the parity tests proper."""
import functools

import pytest

import gpu_runs
from gpu_runs import VIOLATING_MODELS

pytestmark = pytest.mark.gpu

checker = functools.partial(gpu_runs.checker, table_log2=24)


@pytest.mark.parametrize("name", ["miniqueue", "minimsgs", "miniwindow"])
def test_zz_sequence_models_match_oracle_a(name, goldens):
    """Sequences / tuples / RECURSIVE / \\X (SURVEY 8f row 4): counts, widths and the decoded state set against Oracle A."""
    from golden.make_golden import state_digest
    g = goldens[name]
    with checker(name, cont=True, table_log2=16) as ck:
        r = ck.run()
        texts = [ck.decoder.text(row) for row in ck.copy_states(0, r.distinct)]
    assert r.complete and r.violation is None
    assert (r.distinct, r.generated, r.depth, r.deadlocks, r.levels) == (
        g["distinct"], g["generated"], g["depth"], g["deadlocks"], g["levels"])
    assert state_digest(texts) == g["state_digest"]


@pytest.mark.parametrize("name", ["firsttry_3x4_r3e3", "kip279_3x4_r3e3", "kip101_3x4_r3e3", "trunchw_3x4_r3e3"])
def test_zz_protocol_variants_at_headline_bounds(name, goldens):
    """SURVEY 8(d) row 3: the four earlier protocol variants at the bounds of config #3 (3 brokers, LogSize 4,
    MaxRecords 3, MaxLeaderEpoch 3), searched past their violations: 1.7..2.9e8 states each, counts, per-level widths
    and first-violation level against the Oracle B golden (which the CPU BFS over the lowered model reproduces)."""
    g = goldens[name]
    with checker(name, cont=True, table_log2=30, max_states=g["distinct"] + (1 << 22)) as ck:
        r = ck.run()
        assert ck.info.exact == 1
    assert r.complete
    assert (r.distinct, r.generated, r.depth, r.deadlocks) == (g["distinct"], g["generated"], g["depth"], g["deadlocks"])
    assert r.levels == g["levels"]
    first = min(l for l in g["first_violation_level"].values() if l)
    assert r.violation is not None and r.violation["kind"] == "invariant" and r.violation["level"] == first


@pytest.mark.parametrize("name", VIOLATING_MODELS)
def test_zz_three_replica_state_sets_match_oracle_a(name, goldens):
    """The 3-replica models whose StrongIsr violations the reference describes: the whole reachable state set
    (1.4..2.0e6 states), decoded to TLC text, against the digest Oracle A -- the interpreter of the unchanged .tla
    text -- produced in hours of Python (tests/golden/run_oracle_a.py, merge_oracle_a.py).  Skipped for a model whose
    Oracle A run has not been merged into the goldens."""
    from golden.make_golden import state_digest
    g = goldens[name]
    if "state_digest" not in g:
        pytest.skip("no Oracle A digest merged for this model")
    with checker(name, cont=True) as ck:
        r = ck.run()
        texts = ck.decoder.texts(ck.copy_states(0, r.distinct))
    assert r.distinct == g["distinct"] and len(set(texts)) == g["distinct"]
    assert state_digest(texts) == g["state_digest"]


def test_zz_cli_runs_a_sequences_spec_end_to_end():
    """.tla with module Sequences + .cfg in, TLC's summary out (lowering + nvcc + GPU run inside the CLI)."""
    import os
    import subprocess
    import sys
    from conftest import ROOT
    specs = os.path.join(ROOT, "tests", "specs")
    p = subprocess.run([sys.executable, "-m", "kafka_specification_b200.tlc2", "-config", os.path.join(specs, "MiniQueue.cfg"),
                        "-deadlock", os.path.join(specs, "MiniQueue")], cwd=ROOT, capture_output=True, text=True, timeout=600)
    out = p.stdout + p.stderr
    assert p.returncode == 0, out
    assert "Model checking completed. No error has been found." in out
    assert "729 states generated, 160 distinct states found, 0 states left on queue." in out
    assert "The depth of the complete state graph search is 6." in out
