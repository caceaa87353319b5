"""kmc_run inserts successors from inside the expand kernel (one launch per frontier chunk); the kmc_shard_* building
blocks keep the two-kernel pipeline (expand -> candidate buffer -> k_insert).  At world 1 both must find the same
BFS: counts, level widths, successors per emit site, the violation, and each level's set of states."""
import functools

import pytest

import gpu_runs
from gpu_runs import compare_runs

pytestmark = pytest.mark.gpu

SYMMETRIC = {"kip320sym_small"}   # the stored member of an orbit depends on which generator won the insert

fused_run = functools.partial(gpu_runs.fused_run, table_log2=24)
two_kernel_run = functools.partial(gpu_runs.two_kernel_run, table_log2=24)


@pytest.mark.parametrize("name,cont", [("kip320_small", True), ("kip320sym_small", True), ("asyncisr_w3", True),
                                       ("frl_3x4x3", True), ("trunchw_small", False), ("idsequence_deadlock", False)])
def test_fused_run_matches_two_kernel_pipeline(name, cont):
    fused = fused_run(name, cont=cont)
    if name == "trunchw_small":
        assert fused[0]["violation"]["kind"] == "invariant" and fused[0]["violation"]["level"] == 9
    if name == "idsequence_deadlock":
        assert fused[0]["violation"]["kind"] == "deadlock" and fused[0]["violation"]["trace_len"] == 6
    if name == "asyncisr_w3":
        assert fused[0]["out_of_model"] > 0
    assert fused[0]["levels"]
    compare_runs(fused, two_kernel_run(name, cont=cont), symmetric=name in SYMMETRIC)


def test_fused_run_with_a_spilling_ring_matches_two_kernel_pipeline():
    """262,144 ring slots for 737,794 states: the fused kernel appends to a ring that wraps while it expands."""
    fused = fused_run("kip320_small", cont=True, spill=True, max_states=1 << 18)
    assert fused[0]["levels"]
    compare_runs(fused, two_kernel_run("kip320_small", cont=True))


def test_fused_bounded_run_of_a_four_word_model_matches_two_kernel_pipeline():
    """kip320_5brokers: four words per state, 128-bit fingerprint keys, one state per thread of the expand tile."""
    kw = {"max_states": 1 << 21, "table_log2": 23}
    fused = fused_run("kip320_5brokers", stop_after_states=300_000, **kw)
    assert fused[0]["levels"]
    compare_runs(fused, two_kernel_run("kip320_5brokers", stop_after_states=300_000, **kw))
