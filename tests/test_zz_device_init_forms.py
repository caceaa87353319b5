"""The device form of Init on the GPU (k_init), every run audited.  Each device-Init model (but frl_typeinit_3x4x3, whose
2.1 * 10^9 candidates and 1.77 * 10^6 solutions test_zz_device_init.py checks against the closed form's digest) runs
three times -- with the default chunks, with a small candidate buffer of an odd number of rows (many k_init launches
whose ends fall mid-warp, one of them across candidate 2^32), and under set_spill with a table small enough to flush
inside level 1 -- and each run's whole store goes through the audit (store_audit.py), seeded from the host's own
enumeration of the candidates or, above 2^32 candidates, from the closed form (init_forms.py); the three runs must store
the same states.  Then k_init's error exits: a solution wider than the layout, a full store, a full table."""
import json
import os

import numpy as np
import pytest

from conftest import ROOT
from gpu_runs import audited_run, checker, sorted_rows
from hostmodel import HostModel
from init_forms import LARGE, SPACE, decode, solution_indices

from kafka_specification_b200.build import device_init_registry
from kafka_specification_b200.runtime import KmcError, StateDecoder

pytestmark = pytest.mark.gpu

SMALL = ["frl_typeinit_tiny", "frl_typeinit_3x4x2", "miniinit_device", "miniinit_viol_device", "miniinit_sym_device",
         "minidecode_leaves_device", "minidecode_shapes_device", "minidecode_narrow_fit"]
CLOSED_FORM_ELSEWHERE = ["frl_typeinit_3x4x3"]
ERROR_ONLY = ["minidecode_narrow"]                   # every run of it stops with a layout overflow
CHUNK_ROWS = {"small": 999, "large": 123_456_791}    # odd: the chunks start at every residue mod 32
SPILL_LOG2 = {"minidecode_ranges": 19, "minidecode_edge": 17, "minidecode_subsets": 28}


def meta(name) -> dict:
    with open(os.path.join(ROOT, "build", "models", name, "model.json")) as f:
        return json.load(f)


def closed_form_rows(hm: HostModel, name: str) -> np.ndarray:
    """The solutions of a large model, packed by init_candidate() at the closed form's indices (the host tests check
    init_candidate() against a decode written from the spec at the indices that matter)."""
    rows = []
    for i in solution_indices(name):
        status, words = hm.init_candidate(0, i)
        assert status == "solution", (name, i)
        rows.append(words)
    return np.array(rows, dtype=np.uint64)


def test_every_device_init_model_is_run_here():
    device = {n for n, spec in device_init_registry().items() if meta(n)["init"].get("device")}
    assert device == set(SMALL + LARGE + CLOSED_FORM_ELSEWHERE + ERROR_ONLY)


def run_three_ways(name):
    """The default run, the run in small chunks and the set_spill run of one model, each audited: [(RunResult, report)]."""
    hm = HostModel.for_built_model(name)
    large = name in LARGE
    init_rows = closed_form_rows(hm, name) if large else None
    base = {"cont": True, "table_log2": 20}
    rows = CHUNK_ROWS["large" if large else "small"]
    if large:
        lg = SPILL_LOG2[name]
        # the chunk that holds candidate 2^32 starts mid-warp, so that candidates on both sides of 2^32 share a warp
        k = (1 << 32) // rows
        assert k * rows < 1 << 32 < min((k + 1) * rows, SPACE[name] + 1) and ((1 << 32) - k * rows) % 32
    else:
        lg = max(7, (hm.bfs()["widths"][0] - 1).bit_length())   # half the table holds fewer keys than level 1
    runs = []
    for opts in (base, {**base, "cand_bytes": rows * (hm.words + 1) * 8},
                 {"cont": True, "set_spill": True, "table_log2": lg, "max_states": 1 << 22}):
        r, rep = audited_run(name, init_rows=init_rows, **opts)
        runs.append((r, rep))
        assert r.complete and r.init_candidates == sum(hm.init_space)
        if opts.get("set_spill") and r.levels[0] > 1 << (lg - 1):
            assert r.stats["set_flushes"] >= 1
    return hm, runs


def level_sets(rep) -> list:
    out, first = [], 0
    for w in rep["widths"]:
        out.append(sorted_rows(rep["states"][first:first + w]))
        first += w
    return out


@pytest.mark.parametrize("name", SMALL + LARGE)
def test_device_init_runs_are_audited(name):
    hm, runs = run_three_ways(name)
    r0, rep0 = runs[0]
    if name in LARGE:
        sols = solution_indices(name)
        assert r0.init_generated == r0.levels[0] == len(sols)
        want = {decode(name, i) for i in sols}
        assert set(StateDecoder(meta(name)).texts(rep0["states"][: r0.levels[0]])) == want
    else:
        host = hm.bfs()
        assert host["complete"]
        assert (r0.distinct, r0.generated, r0.deadlocks) == (len(host["parents"]), host["generated"], host["deadlocks"])
        assert rep0["widths"] == host["widths"]
        assert r0.init_generated == len(hm.init_solutions())
    summary0 = (r0.distinct, r0.generated, r0.deadlocks, r0.levels, r0.init_generated, r0.init_candidates)
    for r, rep in runs[1:]:
        assert (r.distinct, r.generated, r.deadlocks, r.levels, r.init_generated, r.init_candidates) == summary0
        if not hm.symmetry:                  # under SYMMETRY the member of an orbit stored is whichever insert won
            for a, b in zip(level_sets(rep0), level_sets(rep)):
                assert np.array_equal(a, b)


def test_a_solution_wider_than_the_layout_stops_the_run():
    """minidecode_narrow's layout has a \\in -2 .. 4 and Leaves generates a = 9: KMC_E_LAYOUT_OVERFLOW from k_init, a
    trap in the host BFS; minidecode_narrow_fit, with a filter that rejects those candidates, runs clean (and is
    audited above)."""
    assert HostModel.for_built_model("minidecode_narrow").bfs()["fail"] == 1
    with checker("minidecode_narrow", table_log2=16) as ck:
        with pytest.raises(KmcError, match="LAYOUT_OVERFLOW") as e:
            ck.run()
        assert e.value.code == -6
    with checker("minidecode_narrow_fit", table_log2=16) as ck:
        r = ck.run()
        assert r.complete and r.levels[0] == HostModel.for_built_model("minidecode_narrow_fit").bfs()["widths"][0]


@pytest.mark.parametrize("opts,error,code", [
    ({"max_states": 1000, "table_log2": 16}, "STORE_FULL", -5),       # level 1 alone has 2,268 states
    ({"max_states": 1 << 16, "table_log2": 8}, "TABLE_FULL", -4),     # 256 slots, no set_spill
])
def test_a_full_store_or_table_inside_level_1(opts, error, code):
    with checker("minidecode_shapes_device", **opts) as ck:
        with pytest.raises(KmcError, match=error) as e:
            ck.run()
        assert e.value.code == code and not ck.stats()["complete"]
    with checker("minidecode_shapes_device", table_log2=16) as ck:
        r = ck.run()
        assert r.complete and r.levels == [2268, 1134]
