"""TLC's -dump on the GPU: the transitions kmc_edges enumerates, the state and dot files, and the tlc2 command line.

The edges of every expanded stored state are checked against the lowered Next compiled for the host
(tests/support/host_model.cpp): for each source, the host's successors that the CONSTRAINT keeps, fingerprinted by set
identity, must be exactly the GPU's, as a multiset.  The pass must leave the run as it was, and spilled levels must
give the same edges as a run that keeps its whole store on the device.
"""
import collections
import functools
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import gpu_runs
from conftest import REFERENCE, ROOT, needs_reference
from golden.make_golden import state_digest
from store_audit import AuditLib, copy_parents

pytestmark = pytest.mark.gpu

checker = functools.partial(gpu_runs.checker, table_log2=22)
EDGE_MODELS = ["idsequence", "frl_tiny", "kip320_n2", "kip279_n2", "kip320sym_n2", "minibound", "miniinit_device"]


def expanded(ck) -> int:
    st = ck.stats()
    return st["distinct"] - st["queue"]


def edge_multiset(e, with_src=True) -> collections.Counter:
    cols = [e["src"]] if with_src else []
    cols += [e["src_fp"], e["dst_fp"], e["action"].astype(np.uint64)]
    return collections.Counter(map(tuple, np.stack(cols, axis=1).tolist()))


def host_edges(a: AuditLib, states: np.ndarray) -> collections.Counter:
    """(src, src_fp, dst_fp, action) of every successor the host's Next generates and the CONSTRAINT keeps."""
    src_fps = a.fingerprints(states, a.symmetry)
    out = collections.Counter()
    for i, s in enumerate(states):
        succ, act = a.successors(s)
        keep = np.array([a.in_model(t) for t in succ], dtype=bool)
        if not keep.any():
            continue
        for fp, ac in zip(a.fingerprints(succ[keep], a.symmetry).tolist(), act[keep].tolist()):
            out[(i, int(src_fps[i]), int(fp), int(ac))] += 1
    return out


@pytest.mark.parametrize("name", EDGE_MODELS)
def test_edges_match_the_host_model(name):
    a = AuditLib.for_built_model(name)
    with checker(name, cont=True) as ck:          # (minibound violates an invariant: every level is expanded)
        r = ck.run()
        assert r.complete
        n = expanded(ck)
        e = ck.edges(0, n)
        states = ck.copy_states(0, n)
        st = ck.stats()
        fps = ck.fingerprints(0, n)
    assert edge_multiset(e) == host_edges(a, states)
    # out_of_model also counts the initial states a CONSTRAINT discards
    init_out = sum(not a.in_model(s) for s in a.init_solutions())
    assert len(e) + st["out_of_model"] - init_out == st["generated"] - st["init_generated"]
    # the fingerprints of the stored states are the edges' source ids
    assert np.array_equal(fps, a.fingerprints(states, a.symmetry))
    assert set(e["src_fp"].tolist()) <= set(fps.tolist())


@pytest.mark.parametrize("stop", [0, 5000])
def test_edge_count_is_generated_less_init(stop):
    opts = {"stop_after_states": stop} if stop else {}
    with checker("kip320_small", **opts) as ck:
        r = ck.run()
        assert r.complete == (stop == 0) and (r.queue > 0) == (stop > 0)
        st = ck.stats()
        e = ck.edges(0, expanded(ck), chunk=3001)
    assert len(e) + st["out_of_model"] == st["generated"] - st["init_generated"]


def run_state(ck) -> dict:
    st = ck.stats()
    return {"stats": st, "coverage": ck.coverage(), "violation": ck.violation(), "reports": ck.invariant_reports(),
            "levels": ck.level_widths(), "states": ck.copy_states(0, st["distinct"]).tobytes(),
            "parents": copy_parents(ck, 0, st["distinct"]).tobytes()}


def test_the_pass_changes_nothing():
    # a -continue run that violates invariants: stats, coverage, the violation, the reports and the store stay
    with checker("trunchw_small", cont=True) as ck:
        ck.run()
        before = run_state(ck)
        assert before["violation"] and before["reports"]
        e = ck.edges(0, ck.stats()["distinct"])
        assert len(e) > 0
        after = run_state(ck)
    assert before == after


def test_spilled_levels_give_the_same_edges():
    with checker("kip320_small") as ck:
        ck.run()
        ref = edge_multiset(ck.edges(0, expanded(ck)), with_src=False)
    # a ring of 2^18 states (a third of the state space): the first levels are on the host when the last ones are
    # expanded
    with checker("kip320_small", spill=True, max_states=1 << 18) as ck:
        r = ck.run()
        assert r.complete and ck.stats()["max_states"] == 1 << 18
        spilled = edge_multiset(ck.edges(0, expanded(ck)), with_src=False)
    assert spilled == ref


def dump_texts(path) -> list[str]:
    blocks = open(path).read().split("\n\n")
    assert blocks[-1] == ""
    out = []
    for k, b in enumerate(blocks[:-1]):
        head, _, text = b.partition("\n")
        assert head == f"State {k + 1}:"
        out.append(text)
    return out


@pytest.mark.parametrize("name", ["kip320_small", "trunchw_small"])
def test_state_dump_has_oracle_a_digest(name, goldens, tmp_path):
    with checker(name, cont=True) as ck:
        r = ck.run()
        t = ck.dump_states(str(tmp_path / "s.dump"))
    texts = dump_texts(tmp_path / "s.dump")
    assert len(texts) == r.distinct == t["states"] == goldens[name]["distinct"]
    assert state_digest(texts) == goldens[name]["state_digest"]


def test_state_dump_is_identical_across_spill_and_set_spill(tmp_path):
    files = []
    runs = [{}, {"spill": True, "max_states": 1 << 18}, {"set_spill": True, "table_log2": 18, "max_states": 1 << 20}]
    for i, opts in enumerate(runs):
        with checker("kip320_small", **opts) as ck:
            r = ck.run()
            assert r.complete
            if opts.get("set_spill"):
                assert ck.stats()["set_flushes"] > 0
            ck.dump_states(str(tmp_path / f"{i}.dump"))
        files.append(open(tmp_path / f"{i}.dump", "rb").read())
    assert files[0] == files[1] == files[2]


def test_symmetric_dump_holds_the_same_orbits(tmp_path):
    a = AuditLib.for_built_model("kip320sym_small")
    orbits = []
    for i, opts in enumerate([{}, {"spill": True, "max_states": 1 << 16}]):
        with checker("kip320sym_small", **opts) as ck:
            r = ck.run()
            rows = ck.copy_states(0, r.distinct)
            ck.dump_states(str(tmp_path / f"{i}.dump"))
            texts = dump_texts(tmp_path / f"{i}.dump")
            assert sorted(texts) == sorted(ck.decoder.texts(rows))
            orbits.append(set(a.fingerprints(rows, True).tolist()))
    assert orbits[0] == orbits[1] and len(orbits[0]) == r.distinct


def test_edges_refused_on_a_world_2_context():
    from kafka_specification_b200.runtime import KmcError
    with checker("kip320_n2", world=2, rank=0, cand_bytes=1 << 24) as ck:
        with pytest.raises(KmcError) as e:
            ck.edges(0, 1)
    assert e.value.code == -1 and "one-GPU" in str(e.value)


def run_cli(*args):
    p = subprocess.run([sys.executable, "-m", "kafka_specification_b200.tlc2", *args], cwd=ROOT, capture_output=True,
                       text=True, timeout=900)
    return p.returncode, p.stdout + p.stderr


@needs_reference
def test_cli_dot_dump_of_idsequence(tmp_path):
    rc, out = run_cli("-dump", "dot,actionlabels,colorize", str(tmp_path / "graph"), "-config",
                      os.path.join(ROOT, "models", "IdSequence.cfg"), os.path.join(REFERENCE, "IdSequence"))
    assert rc == 0, out
    got = open(tmp_path / "graph.dot").read()
    want = open(os.path.join(ROOT, "tests", "golden", "idsequence.dot")).read()
    assert got == want
    assert len(re.findall(r"^-?\d+ \[label=", got, re.M)) == 6 and len(re.findall(" -> ", got)) == 5


def test_cli_state_dump_after_a_violation(tmp_path):
    specs = os.path.join(ROOT, "tests", "specs")
    spec = tmp_path / "MiniLock.tla"
    spec.write_text(open(os.path.join(specs, "MiniLock.tla")).read().replace(
        "HolderNotWaiting ==", "NeverTwo == Cardinality(waiting) < 2\nHolderNotWaiting =="))
    cfg = tmp_path / "MiniLock.cfg"
    cfg.write_text(open(os.path.join(specs, "MiniLock.cfg")).read().replace(
        "INVARIANTS TypeOk Bounded HolderNotWaiting", "INVARIANTS TypeOk NeverTwo"))
    rc, out = run_cli("-config", str(cfg), "-dump", str(tmp_path / "states"), str(spec))
    assert rc == 12 and "Error: Invariant NeverTwo is violated." in out, out
    m = re.search(r"(\d+) distinct states found", out)
    texts = dump_texts(tmp_path / "states.dump")
    assert len(texts) == int(m.group(1)) > 0
