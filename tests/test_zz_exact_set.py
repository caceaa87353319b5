"""exact_set: the fingerprint set keyed by the packed state itself, on every model whose key is otherwise hashed.

MiniWide reaches every hashed key form: one full 64-bit word (16-byte slots), two words that can pack to all-ones
(32-byte slots) and five to seven words (64-byte slots).  Every run here must give what the closed form, the goldens
and a default run of the same model give -- counts, levels, stored states, counterexamples, per-invariant reports,
coverage, -dump files -- and its whole store must pass the audit against the lowered Next compiled for the host.  The
last test builds MiniWide with fingerprints cut to 10 bits: the default set then loses states, the exact one does not.
"""
import os
import subprocess

import numpy as np
import pytest

import gpu_runs
from conftest import ROOT
from golden.make_golden import closed_form
from gpu_runs import report_summary, sorted_levels
from kafka_specification_b200 import build as B
from kafka_specification_b200.frontend.cfg import parse_cfg
from store_audit import VIOL_RING, AuditLib, audit_checker

pytestmark = pytest.mark.gpu

BADARG = -1
# (model, words, exact_set slot bytes, table_log2)
SMALL = [("miniwide_one64", 1, 16, 16), ("miniwide_two128", 2, 32, 16), ("miniwide_w5", 5, 64, 16),
         ("miniwide_w6", 6, 64, 16), ("miniwide_w7", 7, 64, 16)]
LARGE = [("miniwide_w5_large", 5, 64, 21), ("miniwide_w6_large", 6, 64, 21), ("miniwide_w7_large", 7, 64, 21)]
SMALL_NAMES = [n for n, _, _, _ in SMALL]

checker = gpu_runs.checker


def expected(name):
    cfg = parse_cfg(open(os.path.join(ROOT, B.registry()[name]["cfg"])).read())
    return closed_form("MiniWide", cfg)


def coverage_counts(cov):
    """What a run's coverage must reproduce: generated per action and per emit site, and distinct in total (which
    generator of a new state won its insert, and so distinct per action, may differ between two runs)."""
    return ([a["generated"] for a in cov["actions"]], cov["sites"], cov["init"]["distinct"],
            sum(a["distinct"] for a in cov["actions"]))


def one_run(name, audit=False, **opts):
    """One kmc_run: its result, each level's sorted states (the queue last), coverage, model info and (`audit`) the
    audit report of its whole store."""
    with checker(name, **opts) as ck:
        r = ck.run()
        widths = list(r.levels) + ([r.distinct - sum(r.levels)] if r.distinct > sum(r.levels) else [])
        out = {"r": r, "sets": sorted_levels(ck, widths), "coverage": coverage_counts(ck.coverage()),
               "info": (ck.info.words, ck.info.exact)}
        if audit:
            out["audit"] = audit_checker(ck, r.levels, r.distinct)
    return out


def reports(r, symmetric=False):
    """The per-invariant reports, without the pick where the first level has more violators than the ring keeps (and,
    under SYMMETRY, without the counterexample's words: the stored member of its orbit is whichever insert won)."""
    out = []
    for rep, full in zip(report_summary(r.invariant_violations, words=not symmetric), r.invariant_violations):
        out.append(rep[:4] + (None, rep[5], None) if full["violators_first_level"] > VIOL_RING else rep)
    return out


def assert_same_search(x, y, symmetric=False):
    """Two runs of one model found the same states, violation and reports."""
    a, b = x["r"], y["r"]
    assert (a.complete, a.distinct, a.generated, a.depth, a.levels, a.deadlocks, a.stats["out_of_model"]) == \
           (b.complete, b.distinct, b.generated, b.depth, b.levels, b.deadlocks, b.stats["out_of_model"])
    if symmetric:
        # which member of an orbit is stored, and so expanded, is whichever insert won: per site only the totals agree
        assert x["coverage"][0] == y["coverage"][0] and x["coverage"][2:] == y["coverage"][2:]
        assert sum(x["coverage"][1]) == sum(y["coverage"][1])
    else:
        assert x["coverage"] == y["coverage"]
        assert len(x["sets"]) == len(y["sets"])
        for depth, (p, q) in enumerate(zip(x["sets"], y["sets"])):
            assert np.array_equal(p, q), f"level {depth + 1}"
    va, vb = a.violation, b.violation
    assert (va is None) == (vb is None)
    # more violators at the first violating level than the ring keeps: the pick is one of them, not a fixed one
    crowded = any(v["violators_first_level"] > VIOL_RING for v in a.invariant_violations)
    if va is not None and crowded:
        assert {k: v for k, v in va.items() if k != "fingerprint"} == {k: v for k, v in vb.items() if k != "fingerprint"}
    elif va is not None:
        assert va == vb
        if not symmetric:
            assert a.trace[-1]["words"] == b.trace[-1]["words"]
    assert reports(a, symmetric) == reports(b, symmetric)


def assert_closed_form(r, want):
    assert r.complete and r.queue == 0
    assert (r.distinct, r.generated, r.depth, r.levels, r.deadlocks, r.stats["out_of_model"]) == (
        want["distinct"], want["generated"], want["depth"], want["levels"], want["deadlocks"], want["out_of_model"])


@pytest.mark.parametrize("name,words,slot_bytes,table_log2", SMALL + LARGE)
def test_closed_form_audit_and_a_default_run(name, words, slot_bytes, table_log2):
    x = one_run(name, audit=True, exact_set=True, cont=True, table_log2=table_log2)
    assert x["info"] == (words, 1) and x["r"].stats["slot_bytes"] == slot_bytes
    assert x["r"].stats["table_slots"] == 1 << table_log2
    assert_closed_form(x["r"], expected(name))
    d = one_run(name, cont=True, table_log2=table_log2)
    assert d["info"] == (words, 0)
    assert_same_search(x, d)


@pytest.mark.parametrize("name", SMALL_NAMES + ["miniwide_w6_sym"])
def test_stopped_at_the_first_violation_as_a_default_run(name):
    x = one_run(name, audit=True, exact_set=True, table_log2=16)
    assert not x["r"].complete and x["r"].violation["invariant"] == "FewFull"
    assert_same_search(x, one_run(name, table_log2=16), symmetric=name.endswith("_sym"))


def test_symmetry_orbits_at_six_words(goldens):
    g = goldens["miniwide_w6_sym"]
    x = one_run("miniwide_w6_sym", audit=True, exact_set=True, cont=True, table_log2=16)
    r = x["r"]
    assert x["info"] == (6, 1) and r.stats["slot_bytes"] == 64
    assert (r.distinct, r.generated, r.depth, r.levels) == (g["distinct"], g["generated"], g["depth"], g["levels"])
    assert_same_search(x, one_run("miniwide_w6_sym", cont=True, table_log2=16), symmetric=True)


@pytest.mark.parametrize("name,table_log2,max_states,words", [
    ("asyncisr_deep", 30, 300_000_000, 3),                  # config #5: 190 bits
    ("kip320sym_5brokers_r1e2", 23, 0, 3),                 # five brokers under SYMMETRY: 3,087,863 orbits
])
def test_large_models_equal_their_goldens(name, table_log2, max_states, words, goldens):
    g = goldens[name]
    opts = {"max_states": max_states} if max_states else {}
    with checker(name, exact_set=True, table_log2=table_log2, **opts) as ck:
        r = ck.run()
        assert ck.info.exact == 1 and ck.info.words == words and r.stats["slot_bytes"] == 32
    assert r.complete and r.violation is None
    assert (r.distinct, r.generated, r.depth, r.levels) == (g["distinct"], g["generated"], g["depth"], g["levels"])


@pytest.mark.parametrize("name,table_log2", [("miniwide_one64", 4), ("miniwide_two128", 4), ("miniwide_w5", 6),
                                             ("miniwide_w6", 6), ("miniwide_w7", 6), ("miniwide_w6_sym", 6)])
def test_set_spill_through_many_flushes(name, table_log2, goldens):
    """The state words move to host memory whenever half the table is used, also in the middle of a level: the results
    are those of a default run with a large table."""
    g = goldens[name]
    x = one_run(name, audit=True, exact_set=True, set_spill=True, cont=True, table_log2=table_log2,
                max_states=g["distinct"] + 4096)
    st = x["r"].stats
    assert x["info"][1] == 1 and st["table_slots"] == 1 << table_log2
    assert st["set_host_keys"] <= x["r"].distinct and x["r"].distinct - st["set_host_keys"] <= st["table_slots"] // 2
    assert st["set_link_bytes"] >= st["set_host_keys"] * 8 * x["info"][0]
    if name == "miniwide_one64":
        assert st["set_flushes"] >= 1
    else:
        assert st["set_flushes"] >= 5 and st["set_flushes"] > x["r"].depth and st["set_filtered"] > 0
    assert_same_search(x, one_run(name, cont=True, table_log2=16), symmetric=name.endswith("_sym"))


@pytest.mark.parametrize("name,ring", [("miniwide_w5_large", 1 << 17), ("miniwide_w7_large", 1 << 19)])
def test_spilling_store_ring(name, ring):
    x = one_run(name, audit=True, exact_set=True, spill=True, cont=True, max_states=ring, table_log2=21)
    assert x["r"].stats["max_states"] == ring < x["r"].distinct
    assert_closed_form(x["r"], expected(name))
    assert_same_search(x, one_run(name, cont=True, table_log2=21))


@pytest.mark.parametrize("name", SMALL_NAMES + ["miniwide_w6_sym"])
def test_checkpoint_and_recover_into_a_smaller_table(name, tmp_path, goldens):
    """Stopped with a checkpoint after level 2, recovered into a table of the smallest power of two above twice the state
    count: the rebuild inserts every checkpointed state into the exact set."""
    g = goldens[name]
    d = str(tmp_path)
    with checker(name, exact_set=True, table_log2=16, checkpoint_dir=d, stop_after_states=sum(g["levels"][:2]) + 1,
                 cont=True) as ck:
        a = ck.run()
    assert not a.complete and a.levels == g["levels"][:2]
    small = max(5, int(g["distinct"]).bit_length() + 1)
    x = one_run(name, audit=True, exact_set=True, recover=d, cont=True, table_log2=small, max_states=g["distinct"] + 4096)
    assert x["r"].stats["table_slots"] == 1 << small < 1 << 16
    r = x["r"]
    assert r.complete and (r.distinct, r.generated, r.depth, r.levels) == (g["distinct"], g["generated"], g["depth"],
                                                                          g["levels"])
    # the same again with set_spill, which flushes during the rebuild itself
    y = one_run(name, exact_set=True, recover=d, cont=True, set_spill=True, table_log2=max(4, small - 4),
                max_states=g["distinct"] + 4096)
    assert y["r"].distinct == g["distinct"] and y["r"].levels == g["levels"]


@pytest.mark.parametrize("name", ["miniwide_one64", "miniwide_two128", "miniwide_w5", "miniwide_w7"])
def test_dump_files_are_byte_identical(name, tmp_path):
    files = {}
    for exact in (False, True):
        with checker(name, exact_set=exact, cont=True, table_log2=16) as ck:
            ck.run()
            for kind in ("states", "dot"):
                path = str(tmp_path / f"{kind}_{exact}")
                if kind == "states":
                    ck.dump_states(path)
                else:
                    ck.dump_dot(path, actionlabels=True, colorize=True)
                files[(kind, exact)] = open(path, "rb").read()
    assert files[("states", True)] == files[("states", False)] and len(files[("states", True)]) > 0
    assert files[("dot", True)] == files[("dot", False)] and len(files[("dot", True)]) > 0


def test_a_model_with_an_exact_key_is_unchanged(goldens):
    g = goldens["kip320_small"]
    with checker("kip320_small", exact_set=True, table_log2=22) as ck:
        r = ck.run()
        assert ck.info.exact == 1 and r.stats["slot_bytes"] == 16
        fps = np.arange(1, 11, dtype=np.uint64)
        seen = np.zeros(10, dtype=np.uint8)
        # the option did nothing here, so neither does it refuse the set's own calls
        assert ck.lib.kmc_fpset_contains(ck.ctx, fps.ctypes.data, 10, seen.ctypes.data) == 0
    assert (r.distinct, r.generated, r.depth, r.levels) == (g["distinct"], g["generated"], g["depth"], g["levels"])


def test_refusals():
    from kafka_specification_b200.runtime import KmcError
    import torch
    with pytest.raises(KmcError) as e:
        checker("miniwide_w5", exact_set=True, world=2, rank=0)
    assert e.value.code == BADARG and "exact_set runs on one GPU" in str(e.value)
    if torch.cuda.device_count() >= 2:
        with pytest.raises(KmcError) as e:
            checker("miniwide_w5", exact_set=True, gpus=2)
        assert e.value.code == BADARG and "exact_set runs on one GPU" in str(e.value)
    fps = np.arange(1, 11, dtype=np.uint64)
    seen = np.zeros(10, dtype=np.uint8)
    with checker("miniwide_w5", exact_set=True, table_log2=16) as ck:
        assert ck.lib.kmc_fpset_put(ck.ctx, fps.ctypes.data, 10, seen.ctypes.data) == BADARG
        assert "a 64-bit fingerprint is not a key" in ck.error_text(BADARG)
        assert ck.lib.kmc_fpset_contains(ck.ctx, fps.ctypes.data, 10, seen.ctypes.data) == BADARG
        assert ck.lib.kmc_shard_begin(ck.ctx) == BADARG
        assert "exact_set runs on one GPU" in ck.error_text(BADARG)
        assert ck.lib.kmc_shard_expand(ck.ctx, 0, 1) == BADARG
        r = ck.run()                       # the context itself still runs, to the first violation
        assert r.violation["invariant"] == "FewFull" and r.violation["level"] == 4
    with checker("miniwide_w5", table_log2=16) as ck:
        assert ck.lib.kmc_fpset_put(ck.ctx, fps.ctypes.data, 10, seen.ctypes.data) == 0


# ---------------------------------------------------------------------------------------------- exactness, observed
FP_BITS = 10


@pytest.fixture(scope="module")
def narrow_fp_lib(tmp_path_factory):
    """miniwide_w5 compiled with fingerprints of FP_BITS bits and a 128-bit key of no more (KMC_TEST_FP_BITS), with the
    nvcc command of the default build; the default build itself is untouched."""
    out = str(tmp_path_factory.mktemp("narrow_fp") / "libkmc_miniwide_w5_fp10.so")
    cmd = B._nvcc_cmd(os.path.join(B.model_dir("miniwide_w5"), "model.h"), out)
    cmd.insert(1, f"-DKMC_TEST_FP_BITS={FP_BITS}")
    subprocess.check_call(cmd)
    return out


def store_audit(name, ck, r):
    """The audit of the whole store (Init, edges, unique states, closure, totals) without the counterexample check,
    whose fingerprints the audit computes at full width."""
    a = AuditLib.for_built_model(name)
    states = ck.copy_states(0, r.distinct)
    parents = np.empty(r.distinct, dtype=np.uint64)
    ck._check(ck.lib.kmc_copy_parents(ck.ctx, 0, r.distinct, parents.ctypes.data))
    found = a.check_store(states, parents, r.levels, len(r.levels), check_deadlock=a.check_deadlock)
    for k in ("generated", "deadlocks", "out_of_model"):
        assert r.stats[k] == found[k], k


def test_narrow_fingerprints_lose_states_only_without_exact_set(narrow_fp_lib):
    want = expected("miniwide_w5")
    with checker("miniwide_w5", model_lib=narrow_fp_lib, cont=True, table_log2=16) as ck:
        lossy = ck.run()
        assert ck.info.exact == 0
    assert lossy.distinct < want["distinct"]
    with checker("miniwide_w5", model_lib=narrow_fp_lib, exact_set=True, cont=True, table_log2=16) as ck:
        r = ck.run()
        assert ck.info.exact == 1
        assert_closed_form(r, want)
        store_audit("miniwide_w5", ck, r)
    with checker("miniwide_w5", model_lib=narrow_fp_lib, exact_set=True, set_spill=True, cont=True, table_log2=8,
                 max_states=want["distinct"] + 4096) as ck:
        r = ck.run()
        assert r.stats["set_flushes"] >= 5
        assert_closed_form(r, want)
        store_audit("miniwide_w5", ck, r)
