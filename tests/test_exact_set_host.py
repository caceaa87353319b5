"""The exact_set option without a GPU: the tlc2 flag that turns it on, the summary line it prints, and its C-ABI text.

The command line is run with stand-ins for the build and for Checker, so that what reaches Checker and what the run
prints can be checked on a machine without a GPU.
"""
import os
import types

import pytest

from conftest import ROOT
from kafka_specification_b200 import tlc2

SPEC = os.path.join(ROOT, "tests", "specs", "MiniWide")


class FakeChecker:
    """Records its options and reports a complete run of 10 states; `info.exact` as kmc_model_info gives it."""
    created = []

    def __init__(self, name, **opts):
        self.opts = opts
        self.info = types.SimpleNamespace(exact=1 if opts.get("exact_set") else 0)
        self.last_rc = 0
        FakeChecker.created.append(self)

    def run(self, raise_on_error=True):
        return types.SimpleNamespace(stats={"gpu_ms_total": 1.0}, levels=[1, 9], violation=None, trace=[],
                                     invariant_violations=[], generated=20, distinct=10, queue=0, complete=True, depth=2)

    def close(self):
        pass


@pytest.fixture
def cli(monkeypatch):
    model = types.SimpleNamespace(warnings=[], init_states=[[0]], init={})
    monkeypatch.setattr(tlc2.B, "lower_to_dir", lambda module, cfg, name: model)
    monkeypatch.setattr(tlc2.B, "build_dispatcher", lambda *a, **k: None)
    monkeypatch.setattr(tlc2.B, "compile_model", lambda *a, **k: None)
    monkeypatch.setattr(tlc2, "Checker", FakeChecker)
    FakeChecker.created = []
    return FakeChecker


def collision_lines(out):
    return [l for l in out.splitlines() if "val = " in l]


def test_exactset_flag_reaches_checker_and_prints_an_exact_estimate(cli, capsys):
    assert tlc2.main(["-exactset", "-config", SPEC + "_w5.cfg", SPEC]) == tlc2.EXIT_OK
    assert cli.created[-1].opts.get("exact_set") is True
    assert collision_lines(capsys.readouterr().out) == [
        "  calculated (optimistic):  val = 0 (exact: the set key is the packed state)"]


def test_without_the_flag_nothing_changes(cli, capsys):
    assert tlc2.main(["-config", SPEC + "_w5.cfg", SPEC]) == tlc2.EXIT_OK
    assert "exact_set" not in cli.created[-1].opts
    (line,) = collision_lines(capsys.readouterr().out)
    assert "128-bit fingerprints" in line


def test_exactset_combines_with_the_other_extension_flags(cli):
    assert tlc2.main(["-exactset", "-setspill", "-spill", "-config", SPEC + "_w5.cfg", SPEC]) == tlc2.EXIT_OK
    opts = cli.created[-1].opts
    assert opts["exact_set"] is True and opts["set_spill"] is True and opts["spill"] is True


def test_tlc2_docstring_calls_it_an_extension():
    doc = tlc2.__doc__
    assert "[-exactset]" in doc and "``-exactset`` (an extension" in doc


def test_header_documents_the_option():
    text = open(os.path.join(ROOT, "include", "kspecmc.h")).read()
    opt = text[text.index('"exact_set":false'):]
    opt = opt[:opt.index(" * Unknown keys")]
    for phrase in ("packed state", "slot_bytes 16 at one word", "32 at two or three", "64 at four to seven",
                   '"set_spill"', '"gpus" > 1, world > 1, the kmc_shard_* calls', "kmc_fpset_*", "KMC_E_BADARG"):
        assert phrase in opt, phrase
    assert "KMC_E_SET_TIMEOUT = -12" in text
    from kafka_specification_b200.runtime import KMC_ERRORS
    assert KMC_ERRORS[-12] == "KMC_E_SET_TIMEOUT"
