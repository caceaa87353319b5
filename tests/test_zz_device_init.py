"""The device form of Init on the GPU (k_init): FiniteReplicatedLog's type as an Init gives exactly the closed form, and
each MiniInit cfg gives the same run from its host table and from k_init (counts, levels, states, violations, traces,
-continue reports, coverage), by default and under set_spill with flushes in the middle of level 1; a checkpointed
device-Init run recovers to the same counts; the command line reports level 1 as the initial states; one GPU only."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import REFERENCE, ROOT, needs_reference
from gpu_runs import checker, sorted_rows

from kafka_specification_b200.runtime import KmcError

pytestmark = pytest.mark.gpu
SPECS = os.path.join(ROOT, "tests", "specs")
TWINS = [("miniinit", "miniinit_device"), ("miniinit_viol", "miniinit_viol_device"), ("miniinit_sym", "miniinit_sym_device")]


def run_summary(name, **opts):
    """(summary of one run, the canonical forms of its stored states, sorted per level).  Under SYMMETRY the orbit
    member that is stored is whichever insert won, and its successors come from other emit sites than another
    member's: only the total over the sites is compared."""
    from hostmodel import HostModel
    hm = HostModel.for_built_model(name)
    with checker(name, **opts) as ck:
        r = ck.run()
        cov = ck.coverage()
        widths = r.levels or [r.distinct]
        levels, first = [], 0
        for w in widths:
            levels.append(sorted_rows(hm.canonicalize(ck.copy_states(first, w))))
            first += w
        s = {"distinct": r.distinct, "generated": r.generated, "deadlocks": r.deadlocks, "depth": r.depth,
             "out_of_model": r.stats["out_of_model"], "levels": r.levels, "complete": r.complete,
             "init_generated": r.init_generated,
             "violation": r.violation, "trace": r.trace, "reports": r.invariant_violations,
             "cov_init": cov["init"], "cov_sites": [sum(cov["sites"])] if hm.symmetry else cov["sites"],
             "cov_actions": [(a["name"], a["generated"]) for a in cov["actions"]],
             "cov_distinct": sum(a["distinct"] for a in cov["actions"])}
        return s, levels, r


def assert_same_runs(a, b):
    (sa, la, _), (sb, lb, _) = a, b
    assert sa == sb
    assert len(la) == len(lb)
    for x, y in zip(la, lb):
        assert np.array_equal(x, y)


@needs_reference
@pytest.mark.parametrize("name,candidates,init,generated", [
    ("frl_typeinit_tiny", 19683, 343, 3724),
    ("frl_typeinit_3x4x2", 66430125, 29791, 499720),
    ("frl_typeinit_3x4x3", 2097152000, 1771561, 30145819),
])
def test_type_init_is_the_closed_form(name, candidates, init, generated, goldens):
    """TypeOk is inductive: level 1 holds every reachable state and expanding it finds nothing new.  generated = the
    initial states + every state's successors (the table model's generated, less its one initial state)."""
    from golden.make_golden import state_digest
    base = {"frl_typeinit_tiny": "frl_tiny", "frl_typeinit_3x4x2": "frl_3x4x2", "frl_typeinit_3x4x3": "frl_3x4x3"}[name]
    g = goldens[base]
    assert generated == init + g["generated"] - 1 and init == g["distinct"]
    with checker(name, table_log2=23) as ck:
        r = ck.run()
        assert ck.info.num_init == 0 and ck.info.init_candidates == candidates
        assert r.init_candidates == candidates
        assert r.init_generated == r.distinct == init
        assert r.levels == [init] and r.depth == 1 and r.complete
        assert r.generated == generated
        assert r.stats["gpu_ms_init"] > 0
        texts = ck.decoder.texts(ck.copy_states(0, r.distinct))
    assert state_digest(texts) == g["state_digest"]


@pytest.mark.parametrize("host,device", TWINS)
def test_twins_give_the_same_run(host, device):
    a = run_summary(host, table_log2=20)
    b = run_summary(device, table_log2=20)
    assert a[2].init_candidates == 0 and b[2].init_candidates > 0
    assert a[2].init_generated == b[2].init_generated
    assert_same_runs(a, b)


@pytest.mark.parametrize("host,device", TWINS)
def test_twins_give_the_same_continue_run(host, device):
    assert_same_runs(run_summary(host, table_log2=20, cont=True), run_summary(device, table_log2=20, cont=True))


@pytest.mark.parametrize("host,device", TWINS)
def test_device_init_under_set_spill_flushes_inside_level_1(host, device):
    """A table of 1,024 slots flushes every 512 keys: level 1 alone holds more keys than that, so k_init's chunks end an
    epoch before level 1 does."""
    a = run_summary(host, table_log2=20)
    b = run_summary(device, table_log2=10, max_states=1 << 20, set_spill=True)
    assert (a[2].levels or [a[2].distinct])[0] > 512 and b[2].stats["set_flushes"] >= 1
    assert_same_runs(a, b)


def test_checkpoint_and_recover_a_device_init_run(tmp_path):
    ref = run_summary("miniinit_device", table_log2=20)[2]
    with checker("miniinit_device", table_log2=20, checkpoint_dir=str(tmp_path), checkpoint_minutes=0) as ck:
        ck.run()
    meta = open(tmp_path / "checkpoint.meta").read()
    assert f"init_generated {ref.init_generated}" in meta
    with checker("miniinit_device", table_log2=20, recover=str(tmp_path)) as ck:
        r = ck.run()
    assert (r.distinct, r.generated, r.deadlocks, r.init_generated, r.init_candidates) == \
           (ref.distinct, ref.generated, ref.deadlocks, ref.init_generated, ref.init_candidates)
    assert r.levels[-1] == ref.levels[-1]


@pytest.mark.parametrize("opts", [{"gpus": 2}, {"world": 2, "rank": 0}])
def test_device_init_runs_on_one_gpu(opts):
    with pytest.raises(KmcError, match="device Init.*one GPU"):
        checker("miniinit_device", **opts)


def run_cli(*args, timeout=900):
    p = subprocess.run([sys.executable, "-m", "kafka_specification_b200.tlc2", *args], cwd=ROOT,
                       capture_output=True, text=True, timeout=timeout)
    return p.returncode, p.stdout + p.stderr


@needs_reference
def test_cli_type_init_prints_level_1_as_the_initial_states():
    rc, out = run_cli("-config", os.path.join(SPECS, "MCFrlTypeInit_3x4x2.cfg"), "-I", REFERENCE,
                      os.path.join(SPECS, "MCFrlTypeInit"))
    assert rc == 0, out
    assert "Finished computing initial states: 29791 distinct states generated." in out
    assert "499720 states generated, 29791 distinct states found, 0 states left on queue." in out


def test_cli_device_init_violation_and_one_gpu():
    rc, out = run_cli("-config", os.path.join(SPECS, "MiniInit_viol_device.cfg"), os.path.join(SPECS, "MiniInit"))
    assert rc == 12, out
    assert "violated by the initial state" in out
    rc, out = run_cli("-workers", "2", "-config", os.path.join(SPECS, "MiniInit_device.cfg"), os.path.join(SPECS, "MiniInit"))
    assert rc == 1, out
    assert "device Init" in out and "one GPU" in out
