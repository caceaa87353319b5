"""Lowered integer arithmetic past 32 bits on the GPU: nvcc's code for the MiniArith models (tests/specs/MiniArith.tla),
whose arithmetic overflows `int` wherever the lowering does not widen it, against Oracle A computed live.

For every MiniArith model: a full -continue run whose counts, levels, first violation levels and state digest are
Oracle A's; the store audited against the lowered Next compiled for the host; and the transitions kmc_edges enumerates
against the host's successors."""
import collections
import functools
import os

import numpy as np
import pytest

import gpu_runs
import tla_interp
from conftest import ROOT
from golden.make_golden import state_digest
from store_audit import AuditLib, audit_checker

from kafka_specification_b200.build import arith_registry

pytestmark = pytest.mark.gpu

checker = functools.partial(gpu_runs.checker, table_log2=20)
MODELS = sorted(arith_registry())


@functools.lru_cache(maxsize=None)
def oracle_a(name: str) -> dict:
    spec = arith_registry()[name]
    cfg_text = open(os.path.join(ROOT, spec["cfg"])).read()
    return tla_interp.run_bfs(spec["module"], [os.path.join(ROOT, "tests", "specs")], cfg_text,
                              stop_on_violation=False, collect_states=True)


@pytest.mark.parametrize("name", MODELS)
def test_run_is_oracle_a(name):
    ref = oracle_a(name)
    with checker(name, cont=True) as ck:
        r = ck.run()
        assert r.complete
        got = {"distinct": r.distinct, "generated": r.generated, "depth": r.depth, "levels": r.levels,
               "deadlocks": r.deadlocks,
               "first_violation_level": {inv: None for inv in ck.meta["invariants"]}}
        for rep in r.invariant_violations:
            got["first_violation_level"][rep["invariant"]] = rep["level"]
        assert got == {k: ref[k] for k in got}
        texts = ck.decoder.texts(ck.copy_states(0, r.distinct))
        assert sorted(texts) == ref["states"]
        assert state_digest(texts) == state_digest(ref["states"])
        audit_checker(ck, r.levels, r.distinct)


@pytest.mark.parametrize("name", MODELS)
def test_edges_match_the_host_model(name):
    a = AuditLib.for_built_model(name)
    with checker(name, cont=True) as ck:
        r = ck.run()
        st = ck.stats()
        n = st["distinct"] - st["queue"]
        e = ck.edges(0, n)
        states = ck.copy_states(0, n)
    assert r.complete and n == r.distinct
    want = collections.Counter()
    src_fps = a.fingerprints(states, a.symmetry)
    for i, s in enumerate(states):
        succ, act = a.successors(s)
        for fp, ac in zip(a.fingerprints(succ, a.symmetry).tolist(), act.tolist()):
            want[(i, int(src_fps[i]), int(fp), int(ac))] += 1
    cols = np.stack([e["src"], e["src_fp"], e["dst_fp"], e["action"].astype(np.uint64)], axis=1)
    assert collections.Counter(map(tuple, cols.tolist())) == want
    assert len(e) == st["generated"] - st["init_generated"]
