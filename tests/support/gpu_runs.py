"""Test support: GPU runs of registered models and the checks that several test modules share.

``checker(name, **opts)`` is a Checker with exactly the options the caller passes; each test module binds its own
default set size (``functools.partial(gpu_runs.checker, table_log2=...)``), because probe counts, spill rings and
load-dependent assertions depend on it.  The other helpers take the same options.
"""
from __future__ import annotations

import ctypes

import numpy as np

# every parity model: counts, widths and coverage against the goldens
ALL_MODELS = ["idsequence", "frl_tiny", "frl_3x4x2", "frl_3x4x3", "kip320_n2", "trunchw_n2", "kip101_n2", "kip279_n2",
              "firsttry_n2", "kip320_small", "trunchw_small", "kip101_small", "kip279_small", "firsttry_small",
              "asyncisr_v2", "asyncisr_small", "kip320sym_n2", "kip320sym_small", "minilock", "kip320_with279_small",
              "asyncisr_w3"]
# the models whose whole decoded state set has an Oracle A digest in the goldens
DIGEST_MODELS = ["minilock", "idsequence", "frl_tiny", "kip320_n2", "trunchw_n2", "kip101_n2", "kip279_n2", "firsttry_n2",
                 "asyncisr_v2", "asyncisr_small", "kip320_small", "frl_3x4x2", "frl_3x4x3"]
# the 3-replica protocol variants that the reference says break StrongIsr
VIOLATING_MODELS = ["trunchw_small", "kip101_small", "kip279_small", "firsttry_small", "kip320_with279_small"]
# the test-only models (tests/specs) whose violations come from states a CONSTRAINT discards
CONSTRAINT_MODELS = ["minibound", "minibound_mixed", "minibound_init", "minibound_allout", "minibound_nodead",
                     "minibound_sym", "asyncisr_bounded"]


def checker(name, **opts):
    from kafka_specification_b200.runtime import Checker
    return Checker(name, **opts)


def sorted_rows(rows: np.ndarray) -> np.ndarray:
    """Packed states in lexicographic order of their words (first word most significant)."""
    return rows[np.lexsort(rows.T[::-1])] if len(rows) else rows


def sorted_levels(ck, levels: list[int], first: int = 0) -> list[np.ndarray]:
    """The stored states of each level, each level sorted."""
    out = []
    for w in levels:
        out.append(sorted_rows(ck.copy_states(first, w)))
        first += w
    return out


def _summary(ck, levels):
    st = ck.stats()
    return {"distinct": st["distinct"], "generated": st["generated"], "deadlocks": st["deadlocks"],
            "out_of_model": st["out_of_model"], "levels": levels, "violation": ck.violation(),
            "sites": ck.coverage()["sites"]}


def fused_run(name, **opts):
    """kmc_run, which inserts successors from inside the expand kernel: (summary, each level's sorted states)."""
    with checker(name, **opts) as ck:
        r = ck.run()
        assert r.stats["launches_insert"] == 1          # the initial states only
        return _summary(ck, r.levels), sorted_levels(ck, r.levels)


def shard_levels(ck, cont=False, stop_after_states=0) -> list[int]:
    """The level loop of kmc_run, written with the shard building blocks at world 1 on an open Checker: expand into the
    candidate buffer, k_insert of the rows it produced, end of level.  Returns the widths of the levels it expanded."""
    from kafka_specification_b200.runtime import ShardBuffers
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
    return levels


def two_kernel_run(name, cont=False, stop_after_states=0, **opts):
    """The kmc_shard_* pipeline at world 1 (shard_levels): (summary, each level's sorted states), as fused_run."""
    with checker(name, cont=cont, **opts) as ck:
        levels = shard_levels(ck, cont, stop_after_states)
        return _summary(ck, levels), sorted_levels(ck, levels)


def compare_runs(fused, ref, symmetric=False):
    """Two runs of one model find the same BFS: level widths, totals and violation; without SYMMETRY also the successors
    per emit site and each level's set of states (under SYMMETRY the stored member of an orbit is the one whose insert
    won)."""
    (a, sets_a), (b, sets_b) = fused, ref
    assert a["levels"] == b["levels"]
    for k in ("distinct", "generated", "deadlocks", "out_of_model", "violation"):
        assert a[k] == b[k], k
    if not symmetric:
        assert a["sites"] == b["sites"]
        for depth, (x, y) in enumerate(zip(sets_a, sets_b)):
            assert np.array_equal(x, y), f"level {depth}"


def audited_run(name, details=False, init_rows=None, **opts):
    """One kmc_run and the audit of its whole store (store_audit.audit_checker): (RunResult, audit report).  The report
    holds the run's violation record ("record"); with `details` also its coverage and the TLC text of every stored
    state ("coverage", "texts").  A "check_deadlock" option goes to the audit as well; `init_rows` are the generated
    initial states of a device Init too large for the audit to enumerate."""
    from store_audit import audit_checker
    with checker(name, **opts) as ck:
        r = ck.run()
        # the initial states only (none when recovering, none from k_init): the successors are inserted by the expand
        # kernel
        assert r.stats["launches_insert"] == (0 if "recover" in opts or ck.info.init_candidates else 1)
        rep = audit_checker(ck, r.levels, r.distinct, check_deadlock=opts.get("check_deadlock"), init_rows=init_rows)
        if details:
            rep["coverage"] = ck.coverage()
            rep["texts"] = [ck.decoder.text(row) for row in ck.copy_states(0, r.distinct)]
    assert sum(rep["widths"]) == r.distinct
    return r, rep


def report_summary(reports, words=True):
    """What a run reports per invariant.  (The states before the last one are not part of it: a state's parent is the
    generator whose insert won, which may differ from run to run, as for kmc_violation's trace; under SYMMETRY
    neither is the last one, so pass words=False: the pick is an orbit, and the member stored is the one whose insert
    won.)"""
    return [(r["invariant"], r["level"], r["violators_first_level"], r["violators"], r["fingerprint"], r["trace_len"],
             r["trace"][-1]["words"] if r["trace"] and words else None) for r in reports]


def assert_oracle_b_trace(name, trace, decoder, invariants):
    """Every step of an error trace of a Kafka model, re-checked against ORACLE B (the hand-written C restatement of the
    spec, independent of the front end and of the lowering): the first state is its Init, each state is among the
    successors its Next enumerates for the previous one, the last state violates one of `invariants` there too and no
    earlier state does.  (Round 1 validated the steps with the lowered header itself, which a lowering bug would
    pass.)"""
    import kso
    from kafka_specification_b200.build import registry
    model, params = registry()[name]["kso"]
    states = [decoder.decode(t["words"]) for t in trace]
    replicas = sorted(states[0]["replicaLog"].domain(), key=str)
    recs = [kso.kstate_from_tla(st, replicas) for st in states]
    assert recs[0] == kso.init_state(model, params), "trace does not start in the oracle's initial state"
    for i, (a, b) in enumerate(zip(recs, recs[1:])):
        assert b in kso.successors(model, params, a), f"trace step {i + 1} -> {i + 2} is not a successor under Oracle B"
    assert kso.violated(model, params, recs[-1], invariants), "last trace state violates nothing under Oracle B"
    for a in recs[:-1]:
        assert not kso.violated(model, params, a, invariants), "an earlier trace state already violates"
