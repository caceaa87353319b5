"""Parity tests proper: the CUDA path, through the C ABI, against the goldens and the C oracle.

Run on an H100:  python -m pytest tests -m gpu -x -q
Nothing here reads the .tla sources: models are prebuilt (build/models/*), goldens are committed
(tests/golden/goldens.json), Oracle B compiles from oracle/ with gcc.
"""
import functools
import os

import numpy as np
import pytest

import gpu_runs
from conftest import ROOT
from gpu_runs import ALL_MODELS, DIGEST_MODELS, VIOLATING_MODELS, assert_oracle_b_trace

pytestmark = pytest.mark.gpu

checker = functools.partial(gpu_runs.checker, table_log2=24)


@pytest.mark.parametrize("name", ALL_MODELS)
def test_full_bfs_matches_golden(name, goldens):
    """distinct / generated / depth / per-level widths / deadlocks bit-exact; search runs on past violations."""
    g = goldens[name]
    with checker(name, cont=True) as ck:
        r = ck.run()
    assert r.complete
    assert (r.distinct, r.generated, r.depth, r.deadlocks) == (g["distinct"], g["generated"], g["depth"], g["deadlocks"])
    assert r.levels == g["levels"]
    assert r.queue == 0
    inv_levels = {i: l for i, l in g["first_violation_level"].items() if l is not None}
    if inv_levels:
        assert r.violation is not None and r.violation["kind"] == "invariant"
        assert r.violation["level"] == min(inv_levels.values())
        assert inv_levels[r.violation["invariant"]] == r.violation["level"]
        assert r.violation["trace_len"] == r.violation["level"]       # BFS counterexamples are shortest
    else:
        assert r.violation is None


@pytest.mark.parametrize("name", DIGEST_MODELS)
def test_state_set_matches_oracle_a_digest(name, goldens):
    """Every reachable state, decoded to TLC text, matches the interpreter's set (order-independent digest)."""
    from golden.make_golden import state_digest
    g = goldens[name]
    with checker(name, cont=True) as ck:
        r = ck.run()
        states = ck.copy_states(0, r.distinct)
        texts = ck.decoder.texts(states)             # vectorised: one decode per distinct value of each variable
        assert texts[:50] == [ck.decoder.text(row) for row in states[:50]]
    assert len(set(texts)) == g["distinct"]
    assert state_digest(texts) == g["state_digest"]


@pytest.mark.parametrize("name,params", [("kip320_small", ("kip320", [3, 2, 2, 2])),
                                         ("firsttry_small", ("firsttry", [3, 2, 2, 2])),
                                         ("frl_3x4x3", ("frl", [3, 4, 3]))])
def test_against_oracle_b_live(name, params):
    """The hand-written C restatement, run on the box's host cores, agrees with the GPU."""
    import kso
    ref = kso.run(params[0], params[1], max_states=4_000_000)
    with checker(name, cont=True) as ck:
        r = ck.run()
    assert (r.distinct, r.generated, r.depth, r.deadlocks, r.levels) == (
        ref["distinct"], ref["generated"], ref["depth"], ref["deadlocks"], ref["levels"])


def test_stop_at_first_violation_and_trace():
    """Default (no -continue): stop at the first violating level; the trace is a valid behaviour."""
    with checker("trunchw_small") as ck:
        r = ck.run()
        assert not r.complete and r.violation["kind"] == "invariant"
        assert r.violation["invariant"] in ("WeakIsr", "StrongIsr") and r.violation["level"] == 9
        assert len(r.trace) == 9 and r.trace[0]["action"] is None
        assert_oracle_b_trace("trunchw_small", r.trace, ck.decoder, ck.meta["invariants"])
        assert r.queue > 0


def test_init_state_violation():
    with checker("leaderinisr_init") as ck:
        r = ck.run()
    assert r.violation == {"kind": "invariant", "invariant": "LeaderInIsr", "level": 1, "trace_len": 1,
                           "fingerprint": r.violation["fingerprint"]}
    assert "quorumState = [isr |-> {r1, r2, r3}, leader |-> \"NONE\", leaderEpoch |-> -1]" in r.trace[0]["text"]


def test_deadlock_detection_and_override():
    with checker("idsequence_deadlock") as ck:
        r = ck.run()
        assert r.violation["kind"] == "deadlock" and r.violation["level"] == 6 and len(r.trace) == 6
        assert [t["state"]["nextId"] for t in r.trace] == [0, 1, 2, 3, 4, 5]
    with checker("idsequence_deadlock", check_deadlock=False) as ck:       # TLC's -deadlock switch
        r = ck.run()
        assert r.violation is None and r.complete and r.distinct == 6


def test_rerun_is_deterministic_and_reusable():
    with checker("kip279_small") as ck:
        a = ck.run()
        b = ck.run()
    assert a.violation == b.violation                                 # min-fingerprint counterexample
    assert [t["words"] for t in a.trace][-1] == [t["words"] for t in b.trace][-1]
    assert (a.distinct, a.generated) == (b.distinct, b.generated)


def test_table_full_and_store_full_are_reported():
    from kafka_specification_b200.runtime import KmcError
    with checker("kip320_small", table_log2=12, max_states=1 << 20) as ck:
        with pytest.raises(KmcError) as e:
            ck.run()
        assert e.value.code == -4
    with checker("kip320_small", table_log2=22, max_states=1000) as ck:
        with pytest.raises(KmcError) as e:
            ck.run()
        assert e.value.code == -5


def test_chunked_frontier_gives_identical_results(goldens):
    """A tiny candidate buffer forces many expand/insert chunks per level."""
    g = goldens["kip320_small"]
    with checker("kip320_small", cand_bytes=8 << 20) as ck:
        r = ck.run()
    assert (r.distinct, r.generated, r.depth, r.levels) == (g["distinct"], g["generated"], g["depth"], g["levels"])
    assert r.stats["launches_expand"] > 2 * g["depth"]


def test_fpset_put_contains_size():
    """TLC's FPSet contract: put() returns true iff the fingerprint was already present."""
    rng = np.random.default_rng(7)
    fps = rng.integers(1, 2**63, size=200_000, dtype=np.uint64)
    with checker("idsequence", table_log2=20) as ck:
        first = ck.fpset_put(fps[:100_000])
        assert not first.any() or first.sum() == len(fps[:100_000]) - len(np.unique(fps[:100_000]))
        again = ck.fpset_put(fps[:100_000])
        assert again.all()
        assert ck.fpset_contains(fps[:100_000]).all()
        fresh = fps[100_000:]
        fresh = fresh[~np.isin(fresh, fps[:100_000])]
        assert not ck.fpset_contains(fresh).any()
        assert ck.fpset_size() == len(np.unique(fps[:100_000]))
        # duplicates inside one batch: exactly one of each pair is "new"
        dup = np.concatenate([fresh[:1000], fresh[:1000]])
        seen = ck.fpset_put(dup)
        assert seen.sum() == 1000


def test_probe_count_matches_generated(goldens):
    """Hash-probe accounting used by the roofline: at load <= 0.5 about one 32 B bucket per candidate."""
    with checker("kip320_small", table_log2=24) as ck:
        r = ck.run()
    assert r.generated <= r.stats["probes"] <= 1.05 * r.generated


@pytest.mark.parametrize("name", VIOLATING_MODELS)
def test_error_traces_are_behaviours_under_oracle_b(name, goldens):
    """Default run (stop at the first violation) of every protocol variant the reference says is broken:
    shortest counterexample, each step validated by Oracle B."""
    g = goldens[name]
    first = min(l for l in g["first_violation_level"].values() if l)
    with checker(name) as ck:
        r = ck.run()
        assert not r.complete and r.violation["kind"] == "invariant" and r.violation["level"] == first
        assert len(r.trace) == first and r.trace[0]["action"] is None
        assert all(t["action"] is not None for t in r.trace[1:])
        assert_oracle_b_trace(name, r.trace, ck.decoder, ck.meta["invariants"])


def test_kip320_needs_its_epoch_check_as_the_reference_says(goldens):
    """Kip320.tla:126-133: replacing FencedBecomeFollowerAndTruncate with BecomeFollowerTruncateKip279 breaks
    StrongIsr; with the action as written (kip320_small) all invariants hold."""
    g = goldens["kip320_with279_small"]
    assert g["first_violation_level"]["StrongIsr"] is not None
    with checker("kip320_with279_small", cont=True) as ck:
        r = ck.run()
    assert (r.distinct, r.generated, r.depth, r.levels) == (g["distinct"], g["generated"], g["depth"], g["levels"])
    assert r.violation is not None and r.violation["level"] == g["first_violation_level"]["StrongIsr"]
    with checker("kip320_small", cont=True) as ck:
        assert ck.run().violation is None


def test_exactness_of_the_set_by_state_width():
    """<= 63 bits: bijective 64-bit fingerprint; two words: the packed state itself is the 128-bit key (exact);
    wider (asyncisr_w3: three words): 128-bit fingerprint."""
    for name, exact, slot in (("frl_3x4x3", 1, 8), ("kip320_small", 1, 16), ("asyncisr_small", 1, 16), ("asyncisr_w3", 0, 16)):
        with checker(name, cont=True) as ck:
            r = ck.run()
            assert (ck.info.exact, r.stats["slot_bytes"]) == (exact, slot), name


def test_config4_five_brokers_with_symmetry_matches_oracle_b_golden(goldens):
    """BASELINE config #4 (Kip320, 5 brokers, LogSize 5) as an instance that completes: SYMMETRY over the 5 replicas
    (120 permutations), MaxRecords 1, MaxLeaderEpoch 2: 3,087,863 orbits, counts and per-level widths against Oracle B."""
    g = goldens["kip320sym_5brokers_r1e2"]
    with checker("kip320sym_5brokers_r1e2", table_log2=24, max_states=4_000_000) as ck:
        r = ck.run()
    assert r.complete and r.violation is None
    assert (r.distinct, r.generated, r.depth, r.deadlocks, r.levels) == (
        g["distinct"], g["generated"], g["depth"], g["deadlocks"], g["levels"])


def test_config5_asyncisr_deep_matches_oracle_b_golden(goldens):
    """BASELINE config #5 (AsyncIsr, deep bounds): 294 M states of 190 bits -- 128-bit fingerprints in 16-byte slots
    (collision probability ~ n^2 / 2^129) -- against the Oracle B golden."""
    g = goldens["asyncisr_deep"]
    with checker("asyncisr_deep", table_log2=30, max_states=300_000_000) as ck:
        r = ck.run()
        assert ck.info.exact == 0 and r.stats["slot_bytes"] == 16
    assert r.complete and r.violation is None
    assert (r.distinct, r.generated, r.depth, r.deadlocks, r.levels) == (
        g["distinct"], g["generated"], g["depth"], g["deadlocks"], g["levels"])


@pytest.mark.parametrize("name,opts", [("kip320_3x4_r4e2", {"table_log2": 26, "max_states": 20_000_000}),
                                       ("kip320_3x4_r3e3", {"table_log2": 28, "max_states": 70_000_000}),
                                       ("kip320sym_3x4_r4e3", {"table_log2": 28, "max_states": 60_000_000})])
def test_headline_sizes_match_oracle_b_golden(name, opts, goldens):
    """Full-size runs (10^7..10^8 states): counts and per-level widths against the committed Oracle B golden."""
    g = goldens[name]
    with checker(name, **opts) as ck:
        r = ck.run()
    assert r.complete and r.violation is None
    assert (r.distinct, r.generated, r.depth, r.deadlocks) == (g["distinct"], g["generated"], g["depth"], g["deadlocks"])
    assert r.levels == g["levels"]


def test_spill_store_smaller_than_the_state_space(goldens):
    """spill: the device store is a ring over the live window (the level being expanded + the one being built);
    older levels move to host memory.  262,144 slots for 737,794 states: identical counts and widths."""
    g = goldens["kip320_small"]
    with checker("kip320_small", spill=True, max_states=1 << 18, cont=True) as ck:
        r = ck.run()
        assert r.stats["max_states"] == 1 << 18
        # every state is still addressable (host spill + device ring) and decodes to a distinct value
        rows = ck.copy_states(0, 5000)
        assert len({tuple(int(x) for x in row) for row in rows}) == 5000
    assert r.complete and (r.distinct, r.generated, r.depth, r.deadlocks, r.levels) == (
        g["distinct"], g["generated"], g["depth"], g["deadlocks"], g["levels"])
    # without spill the same store is too small
    from kafka_specification_b200.runtime import KmcError
    with checker("kip320_small", max_states=1 << 18) as ck:
        with pytest.raises(KmcError) as e:
            ck.run()
        assert e.value.code == -5


def test_error_trace_through_spilled_levels(goldens):
    """The parent links of a counterexample reach back into levels that were spilled to the host."""
    g = goldens["trunchw_small"]
    first = min(l for l in g["first_violation_level"].values() if l)
    # 32,768 ring slots: the level being expanded when the violation shows (8,937 states) and the one being built
    # (17,187) fit together, the 34,012 states up to there do not -- the trace walks into the host spill
    with checker("trunchw_small", spill=True, max_states=1 << 15) as ck:
        r = ck.run()
        assert not r.complete and r.violation["level"] == first and len(r.trace) == first
        assert_oracle_b_trace("trunchw_small", r.trace, ck.decoder, ck.meta["invariants"])


def test_checkpoint_and_recover(tmp_path, goldens):
    """-checkpoint / -recover: a run that stops (here: bounded) leaves a checkpoint at a level boundary; a new context
    recovers it (the set is rebuilt from the stored states) and finishes with the golden's counts and widths."""
    g = goldens["kip320_small"]
    d = str(tmp_path)
    with checker("kip320_small", checkpoint_dir=d, stop_after_states=200_000) as ck:
        a = ck.run()
    assert not a.complete and a.queue > 0
    assert os.path.exists(os.path.join(d, "checkpoint.meta")) and os.path.exists(os.path.join(d, "checkpoint.bin"))
    for extra in ({}, {"spill": True, "max_states": 1 << 18}):
        with checker("kip320_small", recover=d, cont=True, **extra) as ck:
            b = ck.run()
        assert b.complete and (b.distinct, b.generated, b.depth, b.deadlocks, b.levels) == (
            g["distinct"], g["generated"], g["depth"], g["deadlocks"], g["levels"])
    # a checkpoint of another model is refused
    from kafka_specification_b200.runtime import KmcError
    with checker("kip279_small", recover=d) as ck:
        with pytest.raises(KmcError) as e:
            ck.run()
        assert e.value.code == -7


def test_bounded_run_stops_cleanly():
    """stop_after_states: a bounded throughput run ends at a level boundary with the queue reported."""
    with checker("kip320_small", stop_after_states=100_000) as ck:
        r = ck.run()
    assert not r.complete and r.violation is None and r.queue > 0
    assert r.distinct >= 100_000 and sum(r.levels) + r.queue == r.distinct


def test_two_gpu_sharded_run_matches_golden(goldens):
    """Fingerprint-sharded BFS over NCCL on 2 GPUs (skipped on a single-GPU box)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import json
    import subprocess
    import sys
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                          "--master-addr", "127.0.0.1", "--master-port", "29533", os.path.join(ROOT, "bench.py"),
                          "--gpus", "2", "--steps", "1", "--warmup", "3", "--model", "kip320_3x4_r4e2"],
                         capture_output=True, text=True, timeout=600)
    line = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert line, out.stdout + out.stderr
    r = json.loads(line[-1])
    g = goldens["kip320_3x4_r4e2"]
    assert r["config"]["distinct"] == g["distinct"] and r["config"]["generated"] == g["generated"]
    assert sum(r["config"]["per_rank_distinct"]) == g["distinct"]


def test_candidate_overflow_is_an_error_not_a_wrong_answer():
    """Chunks are sized for a realistic fan-out; if a model exceeds it the run fails loudly (KMC_E_CAND_FULL)."""
    from kafka_specification_b200.runtime import KmcError
    with checker("frl_3x4x2", cand_bytes=1 << 20, fanout_bound=1) as ck:
        with pytest.raises(KmcError) as e:
            ck.run()
        assert e.value.code == -10
    with checker("frl_3x4x2", cand_bytes=1 << 20, fanout_bound=32) as ck:
        assert ck.run().distinct == 29791


def test_scatter_rounds_when_a_tile_enables_more_pairs_than_the_list_holds(goldens):
    """FiniteReplicatedLog enables ~16 successors per state: a 4096-state tile overflows the 12288-entry pair
    list of the expand kernel, which then works through the site segments in several scatter rounds."""
    g = goldens["frl_3x4x3"]
    with checker("frl_3x4x3", cont=True) as ck:
        r = ck.run()
    assert (r.distinct, r.generated, r.levels) == (g["distinct"], g["generated"], g["levels"])
    assert r.generated / r.distinct > 12


def _torchrun(script_args, port):
    import json
    import subprocess
    import sys
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                          "--master-addr", "127.0.0.1", "--master-port", str(port)] + script_args,
                         capture_output=True, text=True, timeout=600)
    line = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert line, out.stdout[-2000:] + out.stderr[-2000:]
    return json.loads(line[-1])


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
def test_two_gpu_violation_and_cross_rank_trace(mode, goldens):
    """2 ranks: stop at the first violating level, agree on one offending state, and walk its parent
    links across the two GPUs' stores back to the initial state (both exchange paths)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    g = goldens["trunchw_small"]
    first = min(l for l in g["first_violation_level"].values() if l)
    r = _torchrun([os.path.join(ROOT, "tools", "sharded_check.py"), "trunchw_small", mode], 29541 if mode == "p2p" else 29542)
    assert r["p2p"] == (mode == "p2p")
    assert not r["complete"] and r["violation"]["kind"] == "invariant" and r["violation"]["level"] == first
    assert r["depth"] == first - 1 and r["levels"] == g["levels"][: first - 1]
    assert len(r["trace"]) == first and r["trace"][0]["action"] is None
    assert len({t["rank"] for t in r["trace"]}) == 2
    with checker("trunchw_small") as ck:
        trace = [{"words": t["words"]} for t in r["trace"]]
        assert_oracle_b_trace("trunchw_small", trace, ck.decoder, ck.meta["invariants"])
    # and the full search past the violation still matches the golden
    r = _torchrun([os.path.join(ROOT, "tools", "sharded_check.py"), "trunchw_small", mode, "cont"], 29543 if mode == "p2p" else 29544)
    assert (r["distinct"], r["generated"], r["depth"], r["levels"]) == (g["distinct"], g["generated"], g["depth"], g["levels"])
