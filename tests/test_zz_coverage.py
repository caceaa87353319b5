"""Coverage (TLC -coverage): per-site and per-action generated counts from K1, per-action distinct counts from K2.

CPU: the lowering's site -> action map, the committed coverage goldens, the labelled Oracle A against the host
harness, the CLI's report format.  GPU: every parity model's counts against the goldens, the sums, the parent
words, stopped / recovered / multi-GPU runs, and the CLI end to end.
"""
import functools
import json
import os
import re
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest

import gpu_runs
from conftest import ROOT, needs_reference
from gpu_runs import ALL_MODELS
from store_audit import NO_PARENT, copy_parents

GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def coverage_golden():
    with open(os.path.join(GOLDEN, "coverage.json")) as f:
        return json.load(f)


def by_action(per_site, site_action, names):
    out = Counter({n: 0 for n in names})
    for count, a in zip(per_site, site_action):
        if a >= 0:
            out[names[a]] += count
    return dict(out)


# ---------------------------------------------------------------------------------------------------------- CPU
@needs_reference
def test_every_model_lowers_with_site_actions_matching_the_emit_labels(registry):
    """SITE_ACTION[i] is the label of site i's sink.emit, model.json agrees with the header, and the digest that
    checkpoints are checked against is the one the models had before coverage existed."""
    from hostmodel import lower_registered
    digests = json.load(open(os.path.join(GOLDEN, "body_digests.json")))
    for name in registry:
        m = lower_registered(name)
        assert m.digest == digests[name], name
        n = int(re.search(r"static constexpr int NUM_SITES = (\d+);", m.header).group(1))
        table = re.search(r"SITE_ACTION\[[^\]]*\] = \{([^}]*)\};", m.header).group(1)
        site_action = [int(x) for x in table.split(",")][:n]
        bodies = re.split(r"KMC_HD void site_body\(SiteTag<\d+>", m.header)[1:]
        assert len(bodies) == n == len(m.sites), name
        for i, body in enumerate(bodies):
            labels = set(re.findall(r"sink\.emit\(n, (\d+)\);", body.split("\n}\n")[0]))
            assert labels == {str(site_action[i])}, (name, i, labels)
        assert [s["action"] for s in m.sites] == site_action
        assert all(0 <= a < len(m.actions) for a in site_action)
        meta = m.meta()
        assert meta["sites"] == m.sites and meta["actions"] == m.actions
        assert meta["init"]["name"] and meta["init"]["module"]


@needs_reference
def test_init_span_is_the_initial_predicate():
    from hostmodel import lower_registered
    m = lower_registered("minilock")
    src = open(os.path.join(ROOT, "tests", "specs", "MiniLock.tla")).read().split("\n")
    assert m.init["name"] == "Init" and m.init["module"] == "MiniLock"
    assert src[m.init["line"] - 1][m.init["col"] - 1:].startswith("Init")


@needs_reference
@pytest.mark.parametrize("name", ["kip320_n2", "trunchw_n2", "asyncisr_v2", "minilock"])
def test_oracle_a_action_labels_agree_with_the_lowering(name, registry, goldens):
    """TLC's rule (first operator below Next), applied by Oracle A to the .tla text, gives the same generated count
    per action as the lowered model's emit labels on the host."""
    from kafka_specification_b200.build import tla_search_dirs
    from hostmodel import lower_registered, run_host
    from oracle_a_actions import run_bfs_by_action
    spec = registry[name]
    cfg_text = open(os.path.join(ROOT, spec["cfg"])).read()
    a = run_bfs_by_action(spec["module"], tla_search_dirs(), cfg_text)
    h = run_host(lower_registered(name))
    assert a["generated"] == h["generated"] == goldens[name]["generated"]
    assert {k: v for k, v in h["per_action"].items() if v} == a["per_action"]


def test_coverage_golden_sums(coverage_golden, goldens):
    """Per action + initial states = generated of the model's golden; per site, summed by action = per action."""
    assert set(ALL_MODELS) <= set(coverage_golden)
    for name, c in coverage_golden.items():
        assert sum(c["per_action"].values()) + c["num_init"] == goldens[name]["generated"] == c["generated"], name
        assert by_action(c["per_site"], c["site_action"], c["actions"]) == c["per_action"], name
        assert c["per_action_source"] in ("oracle_a", "host_bfs") and c["per_site_source"] == "host_site_mask"


def test_coverage_golden_matches_the_built_models(coverage_golden):
    """The goldens' site -> action maps are those of the models build() lowered."""
    n = 0
    for name, c in coverage_golden.items():
        p = os.path.join(ROOT, "build", "models", name, "model.json")
        if not os.path.exists(p):
            continue
        meta = json.load(open(p))
        assert [s["action"] for s in meta["sites"]] == c["site_action"], name
        assert [a["name"] for a in meta["actions"]] == c["actions"], name
        n += 1
    if n == 0:
        pytest.skip("models not built")


STUB = {"init": {"name": "Init", "module": "MiniLock", "line": 19, "col": 1, "end_line": 23, "end_col": 19,
                 "distinct": 1, "generated": 1},
        "actions": [{"name": "Request", "module": "MiniLock", "location": {"line": 25, "col": 1, "end_line": 28, "end_col": 30},
                     "generated": 84, "distinct": 40},
                    {"name": "Never", "module": "MiniLock", "location": {}, "generated": 0, "distinct": 0}],
        "sites": [84, 0], "complete": True}


def test_cli_coverage_report_format(capsys):
    from kafka_specification_b200 import tlc2
    lines = tlc2.coverage_lines(STUB, "2026-01-02 03:04:05")
    assert [t for _, t in lines] == [
        "The coverage statistics at 2026-01-02 03:04:05",
        "<Init line 19, col 1 to line 23, col 19 of module MiniLock>: 1:1",
        "<Request line 25, col 1 to line 28, col 30 of module MiniLock>: 40:84",
        "<Never of module MiniLock>: 0:0",
        "End of statistics."]
    assert [k for k, _ in lines] == ["coverage_start", "coverage_init", "coverage_next", "coverage_next", "coverage_end"]
    tlc2._TOOL = True
    try:
        tlc2.print_coverage({**STUB, "complete": False})
    finally:
        tlc2._TOOL = False
    out = capsys.readouterr().out
    assert out.count("@!@!@STARTMSG") == out.count("@!@!@ENDMSG") == 6       # warning + 5 lines
    assert "@!@!@STARTMSG 2201:0 @!@!@\nThe coverage statistics at" in out
    assert "@!@!@STARTMSG 2772:0 @!@!@\n<Init line 19" in out and out.count("@!@!@STARTMSG 2773:0 @!@!@") == 2
    assert "@!@!@STARTMSG 2202:0 @!@!@\nEnd of statistics.\n@!@!@ENDMSG 2202 @!@!@" in out
    for code in re.findall(r"STARTMSG (\d+):", out):
        assert f"@!@!@ENDMSG {code} @!@!@" in out


# ---------------------------------------------------------------------------------------------------------- GPU
checker = functools.partial(gpu_runs.checker, table_log2=24)


def parents_histogram(ck, distinct):
    par = copy_parents(ck, 0, distinct)
    init = (par & np.uint64(NO_PARENT)) == np.uint64(NO_PARENT)
    acts = (par[~init] >> np.uint64(56)).astype(np.int64)
    names = [a["name"] for a in ck.meta["actions"]]
    return int(init.sum()), {n: int((acts == i).sum()) for i, n in enumerate(names)}


def assert_sums(ck, r, cov):
    """The run's own totals: generated per site sums to the successors, distinct per action + initial states to the
    distinct states, and distinct <= generated per action."""
    assert sum(cov["sites"]) == r.generated - len(ck.meta["init_states"])
    assert sum(a["generated"] for a in cov["actions"]) == sum(cov["sites"])
    assert sum(a["distinct"] for a in cov["actions"]) + cov["init"]["distinct"] == r.distinct
    for a in cov["actions"]:
        assert a["distinct"] <= a["generated"], a
    names = [a["name"] for a in ck.meta["actions"]]
    assert by_action(cov["sites"], [s["action"] for s in ck.meta["sites"]], names) == \
        {a["name"]: a["generated"] for a in cov["actions"]}
    assert ck.action_counts() == {a["name"]: a["generated"] for a in cov["actions"]}


@pytest.mark.gpu
@pytest.mark.parametrize("name", ALL_MODELS)
def test_gpu_coverage_matches_golden(name, coverage_golden, registry):
    g = coverage_golden[name]
    with checker(name, cont=True) as ck:
        r = ck.run()
        cov = ck.coverage()
        n_init, hist = parents_histogram(ck, r.distinct)
        assert_sums(ck, r, cov)
    assert r.complete and cov["complete"]
    if not registry[name].get("symmetry"):
        # under SYMMETRY the stored member of an orbit is the one whose insert won, and the members' successors are
        # spread differently over the (per-replica) sites; per action they are the same
        assert cov["sites"] == g["per_site"]
    assert {a["name"]: a["generated"] for a in cov["actions"]} == g["per_action"]
    assert {a["name"]: a["distinct"] for a in cov["actions"]} == hist
    assert cov["init"]["distinct"] == n_init and cov["init"]["generated"] == g["num_init"]


@pytest.mark.gpu
def test_gpu_coverage_headline_sums_and_determinism(registry):
    name = "kip320_3x4_r4e3"
    opts = {"table_log2": 30, "max_states": registry[name]["max_states"]}
    runs = []
    with checker(name, **opts) as ck:
        for _ in range(2):
            r = ck.run()
            cov = ck.coverage()
            assert r.complete
            assert_sums(ck, r, cov)
            runs.append(cov["sites"])
    assert runs[0] == runs[1]


@pytest.mark.gpu
def test_gpu_coverage_of_a_run_stopped_at_its_first_violation():
    with checker("trunchw_small") as ck:
        r = ck.run()
        assert not r.complete and r.violation is not None
        cov = ck.coverage()
        n_init, hist = parents_histogram(ck, r.distinct)
        assert_sums(ck, r, cov)
    assert {a["name"]: a["distinct"] for a in cov["actions"]} == hist and cov["init"]["distinct"] == n_init


@pytest.mark.gpu
def test_gpu_coverage_survives_checkpoint_and_recover(tmp_path, coverage_golden):
    """Spill + a bounded run that leaves a checkpoint, then recover: the per-site counts equal an uninterrupted run's.
    A checkpoint without the site_generated line (written before it existed) still recovers with the same counts
    and levels; its coverage is flagged incomplete."""
    g = coverage_golden["kip320_small"]
    d = str(tmp_path / "ck")
    os.makedirs(d)
    with checker("kip320_small", checkpoint_dir=d, stop_after_states=200_000, spill=True, max_states=1 << 18) as ck:
        a = ck.run()
        assert not a.complete and a.queue > 0
        assert_sums(ck, a, ck.coverage())
    meta = open(os.path.join(d, "checkpoint.meta")).read()
    assert meta.index("site_generated") < meta.index("widths")
    with checker("kip320_small", recover=d, cont=True, spill=True, max_states=1 << 18) as ck:
        b = ck.run()
        cov = ck.coverage()
        _, hist = parents_histogram(ck, b.distinct)
        assert_sums(ck, b, cov)
    assert b.complete and cov["complete"] and cov["sites"] == g["per_site"]
    assert {x["name"]: x["distinct"] for x in cov["actions"]} == hist
    old = str(tmp_path / "old")
    os.makedirs(old)
    with open(os.path.join(old, "checkpoint.meta"), "w") as f:
        f.write("".join(line for line in meta.splitlines(keepends=True) if not line.startswith("site_generated")))
    os.link(os.path.join(d, "checkpoint.bin"), os.path.join(old, "checkpoint.bin"))
    with checker("kip320_small", recover=old, cont=True) as ck:
        c = ck.run()
        cov_old = ck.coverage()
    assert (c.distinct, c.generated, c.depth, c.levels) == (b.distinct, b.generated, b.depth, b.levels)
    assert not cov_old["complete"]
    assert sum(cov_old["sites"]) < sum(g["per_site"])
    assert sum(x["distinct"] for x in cov_old["actions"]) + cov_old["init"]["distinct"] == c.distinct


@pytest.mark.gpu
def test_gpu_cli_coverage_on_minilock(coverage_golden):
    p = subprocess.run([sys.executable, "-m", "kafka_specification_b200.tlc2", "-coverage", "1", "-deadlock",
                        "-config", os.path.join(ROOT, "tests", "specs", "MiniLock.cfg"),
                        os.path.join(ROOT, "tests", "specs", "MiniLock")], cwd=ROOT, capture_output=True, text=True, timeout=600)
    out = p.stdout
    assert p.returncode == 0, out + p.stderr
    start, end = out.index("The coverage statistics at"), out.index("End of statistics.")
    rows = re.findall(r"^<(\w+) [^>]*>: (\d+):(\d+)$", out[start:end], flags=re.M)
    assert rows[0][0] == "Init"
    assert sum(int(x[2]) for x in rows) == 169 and sum(int(x[1]) for x in rows) == 76
    g = coverage_golden["minilock"]
    assert g["per_action_source"] == "oracle_a"
    assert {n: int(gen) for n, _, gen in rows[1:]} == g["per_action"]
    assert out.index("End of statistics.") < out.index("169 states generated")


@pytest.mark.gpu
def test_gpu_coverage_on_two_gpus(coverage_golden):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    g = coverage_golden["kip320_small"]
    with checker("kip320_small", cont=True, gpus=2) as ck:
        r = ck.run()
        cov = ck.coverage()
        assert_sums(ck, r, cov)
    assert {a["name"]: a["generated"] for a in cov["actions"]} == g["per_action"] and cov["sites"] == g["per_site"]
