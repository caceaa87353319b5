"""N > 1 path on CPU: the fingerprint-sharded driver (kafka_specification_b200/sharded.py) with
torch.distributed/gloo, world_size 2 and 3, over a host stand-in for the per-rank engine."""
import pytest

from gloo_runs import gloo_run


@pytest.mark.parametrize("name,world,chunk", [("kip320_n2", 2, 97), ("asyncisr_v2", 2, 50), ("frl_tiny", 3, 7),
                                              ("kip320_n2", 1, 1000)])
def test_sharded_bfs_matches_golden(name, world, chunk, tmp_path, goldens):
    g = goldens[name]
    r = gloo_run(name, world, chunk, tmp_path)
    assert (r["distinct"], r["generated"], r["depth"], r["deadlocks"]) == (
        g["distinct"], g["generated"], g["depth"], g["deadlocks"])
    assert r["levels"] == g["levels"] and r["complete"] and r["violation"] is None
    assert sum(r["per_rank"]) == g["distinct"] and len(r["per_rank"]) == world
    if world > 1:
        assert all(n > 0 for n in r["per_rank"])          # the fingerprint partition spreads the states
        assert r["exchanged_rows"] > 0


def test_sharded_bfs_stops_on_violation(tmp_path, goldens):
    g = goldens["trunchw_n2"]
    r = gloo_run("trunchw_n2", 2, 200, tmp_path)
    first = min(l for l in g["first_violation_level"].values() if l)
    assert r["violation"] is not None and not r["complete"]
    assert r["depth"] == first - 1                          # levels fully expanded before the violating one
    # the error trace is walked across ranks through the parent words: shortest, and a real behaviour
    assert r["violation"]["level"] == first and r["trace_len"] == first and r["trace_ok"] is True
    assert len(r["trace_ranks"]) == 2                       # it does hop between the two ranks' stores
    r = gloo_run("trunchw_n2", 2, 200, tmp_path, extra=("cont",))
    assert (r["distinct"], r["generated"], r["depth"]) == (g["distinct"], g["generated"], g["depth"])


@pytest.mark.parametrize("name,world,chunk", [("kip320_n2", 2, 97), ("frl_tiny", 3, 7), ("asyncisr_v2", 2, 50)])
def test_device_sync_driver_loop_matches_golden(name, world, chunk, tmp_path, goldens):
    """The driver's side of the device-synchronised protocol (one board per level, rounds without collectives of its
    own), over a stand-in whose rounds exchange through gloo: same counts and widths for any world size."""
    g = goldens[name]
    r = gloo_run(name, world, chunk, tmp_path, extra=("board",))
    assert (r["distinct"], r["generated"], r["depth"], r["deadlocks"]) == (
        g["distinct"], g["generated"], g["depth"], g["deadlocks"])
    assert r["levels"] == g["levels"] and r["complete"] and r["violation"] is None
    assert sum(r["per_rank"]) == g["distinct"] and all(n > 0 for n in r["per_rank"])


def test_device_sync_driver_loop_stops_on_violation(tmp_path, goldens):
    g = goldens["trunchw_n2"]
    first = min(l for l in g["first_violation_level"].values() if l)
    r = gloo_run("trunchw_n2", 2, 200, tmp_path, extra=("board",))
    assert r["violation"] is not None and not r["complete"] and r["depth"] == first - 1
    assert r["violation"]["level"] == first and r["trace_len"] == first and r["trace_ok"] is True
    r = gloo_run("trunchw_n2", 2, 200, tmp_path, extra=("board", "cont"))
    assert (r["distinct"], r["generated"], r["depth"], r["levels"]) == (g["distinct"], g["generated"], g["depth"], g["levels"])
