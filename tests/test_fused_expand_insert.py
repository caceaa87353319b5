"""kmc_run inserts successors from inside the expand kernel (one launch per frontier chunk); the kmc_shard_* building
blocks keep the two-kernel pipeline (expand -> candidate buffer -> k_insert).  At world 1 both must find the same
BFS: counts, level widths, successors per emit site, the violation, and each level's set of states."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SYMMETRIC = {"kip320sym_small"}   # the stored member of an orbit depends on which generator won the insert


def _checker(name, **kw):
    from kafka_specification_b200.runtime import Checker
    kw.setdefault("table_log2", 24)
    return Checker(name, **kw)


def _sorted_levels(ck, levels, first=0):
    out = []
    for w in levels:
        rows = ck.copy_states(first, w)
        out.append(rows[np.lexsort(rows.T[::-1])])
        first += w
    return out


def _summary(ck, levels):
    st = ck.stats()
    return {"distinct": st["distinct"], "generated": st["generated"], "deadlocks": st["deadlocks"],
            "out_of_model": st["out_of_model"], "levels": levels, "violation": ck.violation(),
            "sites": ck.coverage()["sites"]}


def fused_run(name, **kw):
    with _checker(name, **kw) as ck:
        r = ck.run()
        assert r.stats["launches_insert"] == 1          # the initial states only
        return _summary(ck, r.levels), _sorted_levels(ck, r.levels)


def two_kernel_run(name, cont=False, stop_after_states=0, **kw):
    """The level loop of kmc_run, written with the shard building blocks at world 1: expand into the candidate
    buffer, k_insert of the rows it produced, end of level."""
    from kafka_specification_b200.runtime import ShardBuffers
    with _checker(name, cont=cont, **kw) as ck:
        lib, ctx = ck.lib, ck.ctx
        b = ShardBuffers()
        ck._check(lib.kmc_shard_buffers(ctx, ctypes.byref(b)))
        chunk = max(1, b.region_rows // min(ck.info.max_fanout, 32))
        counts = (ctypes.c_uint64 * 8)()
        first, count = ctypes.c_uint64(), ctypes.c_uint64()
        ck._check(lib.kmc_shard_begin(ctx))
        ck._check(lib.kmc_shard_seed_init(ctx))
        ck._check(lib.kmc_shard_counts(ctx, counts))
        ck._check(lib.kmc_shard_insert(ctx, b.cand, counts[0], None))
        ck._check(lib.kmc_shard_level_done(ctx, ctypes.byref(first), ctypes.byref(count)))
        levels = []
        while count.value and (cont or ck.violation() is None):
            levels.append(count.value)
            end = first.value + count.value
            for off in range(first.value, end, chunk):
                ck._check(lib.kmc_shard_reset_cand(ctx))
                ck._check(lib.kmc_shard_expand(ctx, off, min(chunk, end - off)))
                ck._check(lib.kmc_shard_counts(ctx, counts))
                ck._check(lib.kmc_shard_insert(ctx, b.cand, counts[0], None))
            ck._check(lib.kmc_shard_level_done(ctx, ctypes.byref(first), ctypes.byref(count)))
            if stop_after_states and first.value + count.value >= stop_after_states:
                break
        return _summary(ck, levels), _sorted_levels(ck, levels)


def _compare(name, fused, ref):
    (a, sets_a), (b, sets_b) = fused, ref
    assert a["levels"] == b["levels"] and len(a["levels"]) > 0
    for k in ("distinct", "generated", "deadlocks", "out_of_model", "violation"):
        assert a[k] == b[k], k
    if name not in SYMMETRIC:
        assert a["sites"] == b["sites"]
        for depth, (x, y) in enumerate(zip(sets_a, sets_b)):
            assert np.array_equal(x, y), f"level {depth}"


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
    _compare(name, fused, two_kernel_run(name, cont=cont))


def test_fused_run_with_a_spilling_ring_matches_two_kernel_pipeline():
    """262,144 ring slots for 737,794 states: the fused kernel appends to a ring that wraps while it expands."""
    fused = fused_run("kip320_small", cont=True, spill=True, max_states=1 << 18)
    _compare("kip320_small", fused, two_kernel_run("kip320_small", cont=True))


def test_fused_bounded_run_of_a_four_word_model_matches_two_kernel_pipeline():
    """kip320_5brokers: four words per state, 128-bit fingerprint keys, one state per thread of the expand tile."""
    kw = {"max_states": 1 << 21, "table_log2": 23}
    fused = fused_run("kip320_5brokers", stop_after_states=300_000, **kw)
    _compare("kip320_5brokers", fused, two_kernel_run("kip320_5brokers", stop_after_states=300_000, **kw))
