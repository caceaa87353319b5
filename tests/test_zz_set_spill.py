"""set_spill: the fingerprint set's keys move to host memory whenever its HBM table fills, and the run goes on.

Every run here uses a table far smaller than the state space, so that the keys move to host memory ten times or more,
also in the middle of a level, and every state appended since the last filter whose key was found in an earlier epoch
is removed again.  The results must be those of a run with a table large enough: the goldens, the audit of the whole
store (unique identities, valid parent edges, closure, recomputed coverage, the counterexample pick rule), and, for the
runs that stop at a violation, the same violation and per-invariant reports as a default run.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import REFERENCE, ROOT, needs_reference
from gpu_runs import audited_run, checker, report_summary

pytestmark = pytest.mark.gpu

BADARG, STORE_FULL = -1, -5


def max_fanout(name):
    with open(os.path.join(ROOT, "build", "models", name, "model.json")) as f:
        return json.load(f)["max_fanout"]


def spill_run(name, table_log2, max_states, **opts):
    """One set_spill run and the audit of its store; returns (RunResult, audit report)."""
    r, rep = audited_run(name, set_spill=True, table_log2=table_log2, max_states=max_states, **opts)
    st = r.stats
    # each key reaches host memory once, and what is left in the table stays below its load limit
    assert st["set_host_keys"] <= r.distinct and r.distinct - st["set_host_keys"] <= st["table_slots"] // 2
    assert st["set_link_bytes"] >= st["set_host_keys"] * st["slot_bytes"]
    return r, rep


def assert_golden(r, g):
    assert r.complete and r.queue == 0
    assert (r.distinct, r.generated, r.depth, r.levels) == (g["distinct"], g["generated"], g["depth"], g["levels"])


# (model, table_log2, slot bytes): 8-byte fingerprints, 16-byte exact keys, 128-bit fingerprints, SYMMETRY
MODELS = [("frl_3x4x3", 17, 8), ("kip320_small", 16, 16), ("asyncisr_w3", 16, 16), ("kip320sym_small", 14, 16)]


@pytest.mark.parametrize("name,table_log2,slot_bytes", MODELS)
def test_golden_and_audit_through_many_flushes(name, table_log2, slot_bytes, goldens):
    g = goldens[name]
    r, rep = spill_run(name, table_log2, g["distinct"] + (1 << table_log2))
    assert_golden(r, g)
    assert rep["widths"] == g["levels"]
    st = r.stats
    assert st["slot_bytes"] == slot_bytes and st["table_slots"] == 1 << table_log2
    # a flush happens only at a chunk boundary; more flushes than levels means some came in the middle of a level
    assert st["set_flushes"] >= 10 and st["set_flushes"] > r.depth
    assert st["set_filtered"] > 0 and st["gpu_ms_set_spill"] > 0


# the stopped runs hold ~34,000 states: a 2^12-slot table; the complete ones ~2 million: 2^15
@pytest.mark.parametrize("cont,table_log2", [(False, 12), (True, 15)])
@pytest.mark.parametrize("name", ["trunchw_small", "firsttry_small"])
def test_violations_are_those_of_a_default_run(name, cont, table_log2, goldens):
    g = goldens[name]
    with checker(name, cont=cont, table_log2=24) as ck:
        want = ck.run()
    r, rep = spill_run(name, table_log2, g["distinct"] + (1 << table_log2), cont=cont)
    assert r.stats["set_flushes"] >= 10
    assert (r.complete, r.levels, r.distinct) == (want.complete, want.levels, want.distinct)
    v, w = r.violation, want.violation
    assert (v["kind"], v["invariant"], v["level"], v["trace_len"], v["fingerprint"]) == \
           (w["kind"], w["invariant"], w["level"], w["trace_len"], w["fingerprint"])
    assert r.trace[-1]["words"] == want.trace[-1]["words"]
    assert rep["violation"]["fingerprint"] == v["fingerprint"] and rep["violation"]["level"] == v["level"]
    assert report_summary(r.invariant_violations) == report_summary(want.invariant_violations)
    if cont:
        assert_golden(r, g)


@pytest.mark.parametrize("cont", [False, True])
def test_constraint_discarded_violators(cont, goldens):
    """asyncisr_bounded: the first violators are successors a CONSTRAINT discards (never stored, never in the set)."""
    g = goldens["asyncisr_bounded"]
    table_log2 = 8
    assert (1 << table_log2) // 2 >= max_fanout("asyncisr_bounded")
    with checker("asyncisr_bounded", cont=cont, table_log2=16) as ck:
        want = ck.run()
    r, rep = spill_run("asyncisr_bounded", table_log2, g["distinct"] + 4096, cont=cont)
    assert r.violation == want.violation and r.violation["level"] == 6
    assert r.stats["out_of_model"] == want.stats["out_of_model"] == rep["found"]["out_of_model"]
    assert report_summary(r.invariant_violations) == report_summary(want.invariant_violations)
    if cont:
        assert_golden(r, g)
        assert r.stats["out_of_model"] == g["out_of_model"] and r.stats["set_flushes"] >= 10


def test_with_a_spilling_store_ring(goldens):
    g = goldens["kip320_small"]
    ring = 1 << 19
    r, rep = spill_run("kip320_small", 16, ring, spill=True, cont=True)
    assert_golden(r, g)
    assert r.stats["max_states"] == ring < r.distinct and r.stats["set_flushes"] >= 10


def test_recover_into_a_table_smaller_than_the_checkpoint(tmp_path, goldens):
    g = goldens["kip320_small"]
    d = str(tmp_path)
    with checker("kip320_small", table_log2=22, checkpoint_dir=d, stop_after_states=200_000) as ck:
        a = ck.run()
    assert not a.complete and a.distinct >= 200_000
    # 2^16 slots take 2^15 keys per epoch: the rebuild alone flushes several times
    r, _ = spill_run("kip320_small", 16, g["distinct"] + (1 << 16), recover=d)
    assert_golden(r, g)
    assert r.stats["set_flushes"] >= a.distinct // (1 << 15)


@pytest.mark.parametrize("opts", [{}, {"spill": True, "max_states": 1 << 15}])
def test_store_overflow_after_a_flush_is_reported(opts):
    """A store smaller than the state space ends in KMC_E_STORE_FULL, as without set_spill, also when keys are already in
    host memory: 2^16 slots flush from about 24,600 keys on, and the store (2^15 states: the default for 2^16 slots, or
    a 2^15-state ring) overflows after that, while level 10 or 11 is built."""
    with checker("kip320_small", set_spill=True, table_log2=16, **opts) as ck:
        r = ck.run(raise_on_error=False)
        assert ck.last_rc == STORE_FULL, ck.error_text(ck.last_rc)
    assert not r.complete and r.stats["set_flushes"] >= 1 and r.stats["max_states"] == 1 << 15


def test_refusals():
    from kafka_specification_b200.runtime import KmcError
    with pytest.raises(KmcError) as e:
        checker("kip320_n2", set_spill=True, world=2, rank=0)
    assert e.value.code == BADARG
    # a table whose half cannot hold one state's successors
    with pytest.raises(KmcError) as e:
        checker("kip320_n2", set_spill=True, table_log2=4)
    assert e.value.code == BADARG
    fps = np.arange(1, 11, dtype=np.uint64)
    seen = np.zeros(10, dtype=np.uint8)
    with checker("kip320_n2", set_spill=True, table_log2=16) as ck:
        assert ck.lib.kmc_fpset_put(ck.ctx, fps.ctypes.data, 10, seen.ctypes.data) == BADARG
        assert ck.lib.kmc_fpset_contains(ck.ctx, fps.ctypes.data, 10, seen.ctypes.data) == BADARG
        assert ck.lib.kmc_shard_begin(ck.ctx) == BADARG
        assert ck.lib.kmc_shard_expand(ck.ctx, 0, 1) == BADARG
        r = ck.run()                       # the context itself still runs
        assert r.complete and r.distinct == 5973
    # without the option, the same calls work
    with checker("kip320_n2", table_log2=16) as ck:
        assert ck.lib.kmc_fpset_put(ck.ctx, fps.ctypes.data, 10, seen.ctypes.data) == 0


def test_headline_at_scale(goldens):
    """Kip320 R4E3 (340 million states) through 2^27 slots: 2^26 keys per epoch, several flushes in mid-level."""
    g = goldens["kip320_3x4_r4e3"]
    with checker("kip320_3x4_r4e3", table_log2=27, max_states=350_000_000, set_spill=True) as ck:
        r = ck.run()
    assert_golden(r, g)
    assert (r.distinct, r.generated, r.depth) == (340_433_359, 1_025_370_772, 42)
    assert r.stats["set_flushes"] >= 4 and r.distinct - r.stats["set_host_keys"] <= 1 << 26


def test_asyncisr_deep_at_scale(goldens):
    g = goldens["asyncisr_deep"]
    with checker("asyncisr_deep", table_log2=27, max_states=300_000_000, set_spill=True) as ck:
        r = ck.run()
    assert_golden(r, g)
    assert r.stats["set_flushes"] >= 4


def _summary_lines(out):
    keep = ("states generated", "depth of the complete", "Model checking completed", "Error:")
    return [l for l in out.splitlines() if any(k in l for k in keep)]


@needs_reference
def test_cli_setspill_prints_what_a_large_table_prints():
    """5,973 states through 512 keys of room: the same summary lines and exit status as with 2^16 slots."""
    def run(*args):
        p = subprocess.run([sys.executable, "-m", "kafka_specification_b200.tlc2", *args, "-deadlock", "-config",
                            os.path.join(ROOT, "models", "Kip320_n2.cfg"), "-I", REFERENCE, os.path.join(ROOT, "models", "Kip320")],
                           cwd=ROOT, capture_output=True, text=True, timeout=900)
        return p.returncode, p.stdout + p.stderr
    rc_a, out_a = run("-fpbits", "10", "-maxstates", "8192", "-setspill")
    rc_b, out_b = run("-fpbits", "16")
    assert rc_a == rc_b == 0, out_a[-3000:]
    assert _summary_lines(out_a) == _summary_lines(out_b)
    assert "5973 distinct states found" in out_a
