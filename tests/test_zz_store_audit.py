"""Whole-store audits of GPU runs: every stored state, parent word and counterexample against the lowered Next compiled
for the host (tests/support/host_model.cpp, store_audit.py).  The totals and digests of the other GPU tests cannot see
an off-by-one tile offset, a scatter round labelling pairs with the wrong tile slot, a chunk or ring offset error, or
two actions of equal fan-out swapping ids: each of these keeps every count and corrupts traces and coverage.  The
audit checks, for each state, that its parent word names a state of the previous level whose Next produces exactly
this state under that action, that level 1 is Init, that the identities are unique and that the store is closed under
Next level by level; it recomputes the run's totals and coverage from the stored states, and the counterexample from
every violator the engine records.

Also here: the fingerprint set alone (kmc_fpset_*) with 8-byte and 16-byte slots, at the edges of its probe sequence.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from test_gpu_parity import ALL_MODELS

pytestmark = pytest.mark.gpu

CHECKPOINT = os.path.join(ROOT, "tests", "golden", "checkpoint_kip320_n2")


def checker(name, **kw):
    from kafka_specification_b200.runtime import Checker
    kw.setdefault("table_log2", 22)
    return Checker(name, **kw)


def audit_run(name, check_deadlock=None, **opts):
    """One kmc_run, then the audit of its whole store; returns (RunResult, audit report)."""
    from store_audit import audit_checker
    if check_deadlock is not None:
        opts["check_deadlock"] = check_deadlock
    with checker(name, **opts) as ck:
        r = ck.run()
        rep = audit_checker(ck, r.levels, r.distinct, check_deadlock=check_deadlock)
    assert sum(rep["widths"]) == r.distinct
    return r, rep


@pytest.mark.parametrize("name", ALL_MODELS)
def test_store_audit_full_run(name, goldens):
    r, rep = audit_run(name, cont=True, table_log2=24)
    g = goldens[name]
    assert r.complete and rep["widths"] == g["levels"] and rep["found"]["generated"] == g["generated"]


@pytest.mark.parametrize("name", ["trunchw_small", "kip101_small", "kip279_small", "firsttry_small", "kip320_with279_small"])
def test_store_audit_stop_at_first_violation(name, goldens):
    r, rep = audit_run(name)
    first = min(l for l in goldens[name]["first_violation_level"].values() if l)
    assert not r.complete and rep["violation"]["level"] == r.violation["level"] == first
    assert r.queue > 0 and len(rep["widths"]) == len(r.levels) + 1


def test_store_audit_deadlock():
    r, rep = audit_run("idsequence_deadlock")
    assert r.violation["kind"] == rep["violation"]["kind"] == "deadlock" and r.violation["level"] == 6
    # with deadlocks unchecked the deadlocked state is counted but not reported
    r, rep = audit_run("idsequence_deadlock", check_deadlock=False)
    assert r.violation is None and rep["found"]["deadlocks"] == r.deadlocks == 1


def test_store_audit_initial_state_violation():
    r, rep = audit_run("leaderinisr_init")
    assert r.violation["level"] == rep["violation"]["level"] == 1 and rep["violation"]["level_end"] == 0


def test_store_audit_many_chunks(goldens):
    r, rep = audit_run("kip320_small", cont=True, cand_bytes=8 << 20)
    assert r.stats["launches_expand"] > 2 * goldens["kip320_small"]["depth"]


@pytest.mark.parametrize("name,ring,cont", [("kip320_small", 1 << 18, True), ("trunchw_small", 1 << 15, False)])
def test_store_audit_spill(name, ring, cont):
    r, rep = audit_run(name, spill=True, max_states=ring, cont=cont)
    assert r.stats["max_states"] == ring < r.distinct


@pytest.mark.parametrize("spill", [False, True])
def test_store_audit_bounded_run_and_recover(tmp_path, spill):
    opts = {"spill": True, "max_states": 1 << 18} if spill else {}
    d = str(tmp_path)
    a, _ = audit_run("kip320_small", checkpoint_dir=d, stop_after_states=200_000, **opts)
    assert not a.complete and a.queue > 0
    b, _ = audit_run("kip320_small", recover=d, cont=True, **opts)
    assert b.complete


@pytest.mark.parametrize("spill", [False, True])
def test_store_audit_committed_checkpoint(spill):
    opts = {"spill": True, "max_states": 1 << 11, "table_log2": 16} if spill else {}
    r, _ = audit_run("kip320_n2", recover=CHECKPOINT, cont=True, **opts)
    assert r.complete


@pytest.mark.parametrize("name,cont", [("kip320_small", True), ("trunchw_small", False)])
def test_store_audit_shard_building_blocks(name, cont):
    """CudaShardEngine (world 1) + ShardedChecker: the same audit over eng.ck."""
    from kafka_specification_b200.sharded import CudaShardEngine, ShardedChecker
    from store_audit import audit_checker
    eng = CudaShardEngine(name, 0, 1, 0, table_log2=22)
    try:
        res = ShardedChecker(eng, cont=cont).run()
        rep = audit_checker(eng.ck, res.levels, res.distinct)
    finally:
        eng.close()
    assert res.complete == cont
    if not cont:
        assert rep["violation"]["level"] == res.violation["level"]


def test_store_audit_four_words_bounded(goldens):
    """kip320_5brokers: 4 words per state, 259 emit sites in 5 site groups, one state per thread of the expand tile,
    no golden: the bounded run's levels equal the host BFS's, and the audit needs no golden."""
    from store_audit import AuditLib
    a = AuditLib.for_built_model("kip320_5brokers")
    host = a.host_bfs(stop_after=800_000)
    assert a.words == 4 and a.num_sites == 259
    r, rep = audit_run("kip320_5brokers", stop_after_states=800_000, max_states=1 << 21)
    assert rep["widths"] == host["widths"] and len(r.levels) == host["n_expanded"]
    assert (r.distinct, sum(r.levels)) == (809_721, 184_786)


def test_store_audit_three_words_with_symmetry(goldens):
    """kip320sym_5brokers_r1e2: 3 words, 120 permutations per identity.  A full run takes minutes of host auditing, so
    by default only its first 300,000 states are audited."""
    slow = os.environ.get("KSPEC_SLOW_TESTS") == "1"
    opts = {} if slow else {"stop_after_states": 300_000}
    r, rep = audit_run("kip320sym_5brokers_r1e2", table_log2=24, max_states=4_000_000, cont=True, **opts)
    if slow:
        g = goldens["kip320sym_5brokers_r1e2"]
        assert r.complete and rep["widths"] == g["levels"]


def test_store_audit_two_gpu_union(tmp_path):
    """Two ranks (torchrun): the union of both stores passes the audit with cross-rank parent words, every state sits
    on the rank its canonical fingerprint maps to, and the job's counterexample is the rule's pick over both rings."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from store_audit import AuditLib, compare, owner_of
    a = AuditLib.for_built_model("trunchw_small")
    invariants = json.load(open(os.path.join(ROOT, "build", "models", "trunchw_small", "model.json")))["invariants"]
    for cont, port in ((True, 29561), (False, 29562)):
        out = tmp_path / ("cont" if cont else "stop")
        out.mkdir()
        p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                            "--master-addr", "127.0.0.1", "--master-port", str(port),
                            os.path.join(ROOT, "tests", "support", "store_dump_worker.py"), "trunchw_small", str(out)]
                           + (["cont"] if cont else []), capture_output=True, text=True, timeout=900)
        assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
        res = json.load(open(out / "result.json"))
        ranks = [np.load(out / f"rank{r}.npz") for r in range(2)]
        metas = [json.loads(str(d["meta"])) for d in ranks]
        states = np.concatenate([d["states"] for d in ranks])
        parents = np.concatenate([d["parents"] for d in ranks])
        n_levels = len(res["levels"]) + (0 if res["complete"] else 1)
        rank_widths = []
        for d in ranks:
            c = [int(x) for x in d["level_counts"]] + [0] * n_levels
            rank_widths.append(c[:n_levels])
            assert sum(c) == len(d["states"])
        found = a.check_store(states, parents, None, len(res["levels"]), check_deadlock=a.check_deadlock,
                              rank_widths=rank_widths)
        fp = a.fingerprints(states, True)
        where = np.repeat([0, 1], [len(d["states"]) for d in ranks])
        assert np.array_equal(owner_of(fp, 2), where.astype(np.uint64)), "placement: a state is not on its owner rank"
        stats = {k: sum(m["stats"][k] for m in metas) for k in ("generated", "deadlocks", "out_of_model")}
        cov = {"actions": [{"generated": sum(m["coverage"]["actions"][i]["generated"] for m in metas),
                            "distinct": sum(m["coverage"]["actions"][i]["distinct"] for m in metas)}
                           for i in range(a.num_actions)],
               "sites": [sum(m["coverage"]["sites"][i] for m in metas) for i in range(a.num_sites)]}
        # the job's pick (deadlocks first, then the smallest fingerprint over both ranks' picks) is the rule's pick
        # over the union of the violators
        want = compare(a, found, stats=stats, coverage=cov, parents=parents, violation=res["violation"], record=None,
                       invariants=invariants)
        assert want is not None and res["violation"]["level"] == want["level"]


# ------------------------------------------------------------------------------------------- the fingerprint set alone
FPSET_MODELS = [("idsequence", 8), ("kip320_small", 16)]    # one-word states: 8-byte slots; two words: 16-byte slots


def _bucket_slots(slot_bytes):
    return 32 // slot_bytes                                  # one 32-byte sector per bucket


def _slot_bytes(ck):
    return 8 if ck.words == 1 else 16


@pytest.mark.parametrize("name,slot_bytes", FPSET_MODELS)
def test_fpset_one_key_many_threads(name, slot_bytes):
    """10^6 concurrent puts of 1,000 keys, each 1,000 times, shuffled: exactly one put per key reports it new."""
    rng = np.random.default_rng(3)
    keys = rng.integers(1, 2**64 - 1, size=1000, dtype=np.uint64)
    assert len(np.unique(keys)) == 1000
    batch = np.repeat(keys, 1000)
    rng.shuffle(batch)
    with checker(name, table_log2=16) as ck:
        assert _slot_bytes(ck) == slot_bytes
        seen = ck.fpset_put(batch)
        new_per_key = np.bincount(np.searchsorted(np.sort(keys), batch[~seen]), minlength=1000)
        assert (new_per_key == 1).all(), f"keys inserted more than once: {int((new_per_key > 1).sum())}"
        assert ck.fpset_size() == 1000
        assert ck.fpset_contains(keys).all()


@pytest.mark.parametrize("name,slot_bytes", FPSET_MODELS)
def test_fpset_probe_sequence_wraps_past_the_last_bucket(name, slot_bytes):
    from store_audit import bucket_of
    with checker(name, table_log2=10) as ck:
        assert _slot_bytes(ck) == slot_bytes
        mask = 1024 // _bucket_slots(slot_bytes) - 1
        rng = np.random.default_rng(5)
        cand = rng.integers(2, 2**64 - 1, size=400_000, dtype=np.uint64)
        last = cand[bucket_of(cand, mask) == np.uint64(mask)][: 3 * _bucket_slots(slot_bytes)]
        first = cand[bucket_of(cand, mask) == 0][: _bucket_slots(slot_bytes)]
        assert len(last) == 3 * _bucket_slots(slot_bytes) and len(first) == _bucket_slots(slot_bytes)
        assert not ck.fpset_put(last).any()              # three buckets' worth: two of them past the end, in 0 and 1
        assert ck.fpset_contains(last).all()
        assert not ck.fpset_put(first).any()             # bucket 0's own keys still find room, further on
        assert ck.fpset_put(np.concatenate([last, first])).all() and ck.fpset_contains(first).all()
        assert ck.fpset_size() == len(last) + len(first)


@pytest.mark.parametrize("name,slot_bytes", FPSET_MODELS)
def test_fpset_full_table(name, slot_bytes):
    """2^10 slots take exactly 2^10 keys; the next insert is KMC_E_TABLE_FULL and every stored key is still found."""
    rng = np.random.default_rng(9)
    keys = np.unique(rng.integers(2, 2**64 - 1, size=1100, dtype=np.uint64))[:1025]
    with checker(name, table_log2=10) as ck:
        assert _slot_bytes(ck) == slot_bytes
        for part in np.array_split(keys[:1024], 4):
            assert not ck.fpset_put(part).any()
        assert ck.fpset_size() == 1024
        extra = np.ascontiguousarray(keys[1024:])
        seen = np.zeros(1, dtype=np.uint8)
        assert ck.lib.kmc_fpset_put(ck.ctx, extra.ctypes.data, 1, seen.ctypes.data) == -4
        assert ck.fpset_size() == 1024
        # the failure stays latched in the context, so the raw call reports it again; its answers are still filled in
        out = np.zeros(1024, dtype=np.uint8)
        rc = ck.lib.kmc_fpset_contains(ck.ctx, keys[:1024].ctypes.data, 1024, out.ctypes.data)
        assert rc in (0, -4) and out.all()


@pytest.mark.parametrize("name,slot_bytes", FPSET_MODELS)
def test_fpset_fingerprint_zero_is_stored_as_one(name, slot_bytes):
    with checker(name, table_log2=12) as ck:
        assert not ck.fpset_put(np.array([0], dtype=np.uint64)).any()
        assert ck.fpset_contains(np.array([1], dtype=np.uint64)).all()
        assert ck.fpset_put(np.array([1, 0], dtype=np.uint64)).all()
        assert ck.fpset_size() == 1
