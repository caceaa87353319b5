"""The fused insert on long probe chains: kip320_small (737,794 states) in a set of 2^20 slots, a load of 0.70, so
many rows walk several buckets before their CAS while the expansion goes on.  The fused run must find the same BFS as
the two-kernel pipeline: counts, level widths, successors per emit site and each level's set of states."""
import pytest

from gpu_runs import compare_runs, fused_run, two_kernel_run

pytestmark = pytest.mark.gpu


def test_fused_run_on_a_loaded_set_matches_two_kernel_pipeline():
    # the store gets its own size: by default it holds half as many states as the set has slots, fewer than 737,794
    kw = {"table_log2": 20, "max_states": 1 << 20}
    fused = fused_run("kip320_small", cont=True, **kw)
    assert fused[0]["distinct"] == 737_794 and fused[0]["levels"]
    compare_runs(fused, two_kernel_run("kip320_small", cont=True, **kw))
