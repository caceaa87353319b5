"""Host paths of the single-rank engine: the shard building blocks on one GPU against kmc_run, reads of store ranges
that cross the host spill and the ring wrap, and recovery of a committed checkpoint.

tests/golden/checkpoint_kip320_n2/ is a bounded checkpoint of kip320_n2 (stop_after_states=2000: written at the end of
level 9, 2,033 states), kept to show that recover still reads the checkpoint format byte for byte."""
import functools
import json
import os

import numpy as np
import pytest

import gpu_runs
from conftest import ROOT
from gpu_runs import sorted_rows
from store_audit import copy_parents

pytestmark = pytest.mark.gpu

CHECKPOINT = os.path.join(ROOT, "tests", "golden", "checkpoint_kip320_n2")

checker = functools.partial(gpu_runs.checker, table_log2=22)


def sharded(name, cont=False):
    """One rank of the shard building blocks (world 1: no torch.distributed), driven by ShardedChecker."""
    from kafka_specification_b200.sharded import CudaShardEngine, ShardedChecker
    eng = CudaShardEngine(name, 0, 1, 0, table_log2=22)
    try:
        return ShardedChecker(eng, cont=cont).run(), eng.ck.coverage()
    finally:
        eng.close()


def coverage_sums(cov):
    return sum(a["generated"] for a in cov["actions"]), sum(a["distinct"] for a in cov["actions"])


def test_shard_building_blocks_match_kmc_run_and_golden(goldens):
    g = goldens["kip320_small"]
    with open(os.path.join(ROOT, "tests", "golden", "coverage.json")) as f:
        golden_cov = json.load(f)["kip320_small"]
    with checker("kip320_small", cont=True) as ck:
        a = ck.run()
        a_cov = ck.coverage()
    s, s_cov = sharded("kip320_small", cont=True)
    want = (g["distinct"], g["generated"], g["depth"], g["deadlocks"], g["levels"])
    assert (a.distinct, a.generated, a.depth, a.deadlocks, a.levels) == want
    assert (s.distinct, s.generated, s.depth, s.deadlocks, s.levels) == want
    assert s.complete and s.violation is None
    # generated per action is deterministic; distinct per action is not, its sum is (every non-initial state once)
    assert {x["name"]: x["generated"] for x in s_cov["actions"]} == golden_cov["per_action"]
    assert coverage_sums(s_cov) == coverage_sums(a_cov) == (g["generated"] - golden_cov["num_init"],
                                                            g["distinct"] - golden_cov["num_init"])
    assert s_cov["complete"] and s_cov["sites"] == a_cov["sites"]


def test_shard_building_blocks_stop_at_the_violation_kmc_run_finds():
    with checker("trunchw_small") as ck:
        a = ck.run()
    s, _ = sharded("trunchw_small")
    assert a.violation is not None and s.violation is not None and not s.complete
    assert s.violation["level"] == a.violation["level"]
    assert s.violation["trace_len"] == len(s.trace) == a.violation["trace_len"] == len(a.trace)


def test_spill_range_reads_across_the_host_spill_and_the_ring_wrap():
    """262,144 ring slots; the run stops after level 17, whose expansion spilled [0, 390,625) to the host and left the
    device window [390,625, 554,938), which wraps at 524,288.  One read of everything equals reads split across both
    boundaries, and every level holds the states of a run without spill."""
    ring = 1 << 18
    with checker("kip320_small", spill=True, max_states=ring, stop_after_states=500_000) as ck:
        r = ck.run()
        n = r.distinct
        base = sum(r.levels[:-1])              # the last expanded level starts the device window
        assert not r.complete and base < ring * 2 < n and n - base <= ring
        cuts = [0, base - 1000, base + 1000, 2 * ring - 1000, 2 * ring + 1000, n]
        states, parents = ck.copy_states(0, n), copy_parents(ck, 0, n)
        pieces = list(zip(cuts, cuts[1:]))
        assert np.array_equal(states, np.concatenate([ck.copy_states(a, b - a) for a, b in pieces]))
        assert np.array_equal(parents, np.concatenate([copy_parents(ck, a, b - a) for a, b in pieces]))
    with checker("kip320_small", stop_after_states=500_000) as ck:
        q = ck.run()
        plain = ck.copy_states(0, q.distinct)
    assert (q.distinct, q.levels, q.queue) == (n, r.levels, r.queue)
    bounds = np.concatenate([[0], np.cumsum(r.levels + [r.queue])])
    assert bounds[-1] == n
    for a, b in zip(bounds, bounds[1:]):
        assert np.array_equal(sorted_rows(states[a:b]), sorted_rows(plain[a:b]))


@pytest.mark.parametrize("spill", [False, True])
def test_recover_committed_checkpoint(spill, goldens):
    g = goldens["kip320_n2"]
    opts = {"spill": True, "max_states": 1 << 11, "table_log2": 16} if spill else {}
    with checker("kip320_n2", recover=CHECKPOINT, cont=True, **opts) as ck:
        r = ck.run()
        cov = ck.coverage()
    assert r.complete and r.violation is None
    assert (r.distinct, r.generated, r.depth, r.deadlocks, r.levels) == (
        g["distinct"], g["generated"], g["depth"], g["deadlocks"], g["levels"])
    with checker("kip320_n2", cont=True) as ck:
        ck.run()
        fresh = ck.coverage()
    assert cov["complete"] and cov["sites"] == fresh["sites"]
    assert coverage_sums(cov) == coverage_sums(fresh)
