"""Lowered integer arithmetic at and past 32 bits, on the host, against Oracle A (oracle/tla_interp.py) and Python's
exact integers.

The lowering computes in `int` where an expression's interval fits one and in `int64_t` where it does not; these tests
pin both sides of that choice: the MiniArith specs (tests/specs/MiniArith.tla), a seeded corpus of random expressions
over edge values, the refusal of an interval beyond 64-bit integers, and wide sets and ranges that must lower (or be
refused) without materialising them."""
import os
import random
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import tla_interp
from conftest import ROOT
from golden.make_golden import state_digest
from hostmodel import lower_registered, run_host

from kafka_specification_b200.build import arith_registry
from kafka_specification_b200.lower.model import lower_model
from kafka_specification_b200.lower.svals import LowerError
from kafka_specification_b200.runtime import StateDecoder

SPECS = os.path.join(ROOT, "tests", "specs")
MODELS = sorted(arith_registry())
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1


def oracle_a(module: str, dirs: list[str], cfg_text: str) -> dict:
    return tla_interp.run_bfs(module, dirs, cfg_text, stop_on_violation=False, collect_states=True)


def assert_agrees_with_oracle_a(m, ref: dict):
    """Both forms of the lowered Next (expand() and the two-phase form the GPU runs) against Oracle A's full run."""
    for items in (False, True):
        r = run_host(m, dump=True, items=items)
        assert r["fail"] == 0 and r["complete"]
        got = {k: r[k] for k in ("distinct", "generated", "depth", "levels", "deadlocks", "first_violation_level")}
        assert got == {k: ref[k] for k in got}, f"items={items}"
        texts = [m.state_text([int(w) for w in row]) for row in r["states"]]
        assert sorted(texts) == ref["states"], f"items={items}"
        assert state_digest(texts) == state_digest(ref["states"])
        assert StateDecoder(m.meta()).texts(np.asarray(r["states"], dtype=np.uint64)) == texts


@pytest.mark.parametrize("name", MODELS)
def test_miniarith_agrees_with_oracle_a(name):
    spec = arith_registry()[name]
    cfg_text = open(os.path.join(ROOT, spec["cfg"])).read()
    assert_agrees_with_oracle_a(lower_registered(name), oracle_a(spec["module"], [SPECS], cfg_text))


def test_miniarith_reaches_the_edges():
    """The specs do what they are there for: 64-bit fields and arithmetic, violations only past 32 bits, a device Init
    whose values cross 2^31."""
    m = lower_registered("miniarith_viol")
    assert "const uint64_t a" in m.header and "int64_t" in m.header
    assert {a["path"]: a["bits"] for a in m.layout["atoms"]}["z"] == 41
    assert run_host(m)["first_violation_level"] == {"Sane": None, "NoWrap": 2, "SumSmall": 3}
    md = lower_registered("miniarith_init_device")
    assert md.init["device"] and md.init["candidates"] == 21 * 2 * 2
    assert "(int64_t)" in md.header.split("init_candidate_0")[1].split("}")[0]


OVF_TLA = """---- MODULE Ovf ----
EXTENDS Integers
VARIABLES x, y
TypeOk == x \\in 0 .. 70000 /\\ y \\in 0 .. 6
Init == x = 0 /\\ y = 0
Step == /\\ x < 70000
        /\\ x' = IF x = 0 THEN 65000 ELSE x + 1
        /\\ y' = (x * x) % 7
Next == Step
====
"""
OVF_CFG = "INIT Init NEXT Next INVARIANTS TypeOk CHECK_DEADLOCK FALSE\n"


def test_square_past_32_bits_keeps_its_remainder(tmp_path):
    """x * x for x up to 70000 leaves `int`: (x * x) % 7 must be the exact remainder, not that of a wrapped product."""
    (tmp_path / "Ovf.tla").write_text(OVF_TLA)
    m = lower_model("Ovf", [str(tmp_path)], OVF_CFG)
    assert_agrees_with_oracle_a(m, oracle_a("Ovf", [str(tmp_path)], OVF_CFG))


# ---------------------------------------------------------------------------------------------------------------------
# a seeded corpus of random expressions

# the operands: variables with their layout ranges and the values they take, and constants at the edges
VARS = {
    "a": ((-8, 8), [-7, -1, 0, 5]),
    "b": ((-2147483650, 2147483650), [-2147483649, 2147483647, 2147483648]),
    "c": ((0, 1 << 40), [0, (1 << 40) - 1, 1 << 40]),
    "p": ((1, 1 << 31), [1, 3, 1 << 31]),                     # a divisor: always positive
}
CONSTS = [0, 1, -1, 2147483647, -2147483648, 2147483648, 4294967296, 65536, 65537, 3037000499]
DIVISORS = [1, 7, 65536, 2147483648]
CMPS = {"<": int.__lt__, "<=": int.__le__, ">": int.__gt__, ">=": int.__ge__, "=": int.__eq__, "#": int.__ne__}


def gen(rng: random.Random, depth: int):
    """A random expression tree of depth <= `depth`; the divisor of \\div and % is always provably positive."""
    if depth == 0 or rng.random() < 0.2:
        if rng.random() < 0.6:
            return ("var", rng.choice(sorted(VARS)))
        return ("num", rng.choice(CONSTS))
    op = rng.choice(["+", "-", "*", "neg", "\\div", "%", "if"])
    if op == "neg":
        return ("neg", gen(rng, depth - 1))
    if op in ("\\div", "%"):
        div = ("var", "p") if rng.random() < 0.5 else ("num", rng.choice(DIVISORS))
        return (op, gen(rng, depth - 1), div)
    if op == "if":
        return ("if", rng.choice(sorted(CMPS)), gen(rng, depth - 2 if depth > 1 else 0), gen(rng, 0),
                gen(rng, depth - 1), gen(rng, depth - 1))
    return (op, gen(rng, depth - 1), gen(rng, depth - 1))


def tla(e) -> str:
    k = e[0]
    if k == "var":
        return e[1]
    if k == "num":
        return f"({e[1]})" if e[1] < 0 else str(e[1])
    if k == "neg":
        return f"(-{tla(e[1])})"
    if k == "if":
        return f"(IF {tla(e[2])} {e[1]} {tla(e[3])} THEN {tla(e[4])} ELSE {tla(e[5])})"
    return f"({tla(e[1])} {k} {tla(e[2])})"


def value(e, env: dict) -> int:
    """The exact value, with TLA+'s floor \\div and % (Python's // and %)."""
    k = e[0]
    if k == "var":
        return env[e[1]]
    if k == "num":
        return e[1]
    if k == "neg":
        return -value(e[1], env)
    if k == "if":
        return value(e[4] if CMPS[e[1]](value(e[2], env), value(e[3], env)) else e[5], env)
    a, b = value(e[1], env), value(e[2], env)
    return {"+": a + b, "-": a - b, "*": a * b, "\\div": a // b if b else 0, "%": a % b if b else 0}[k]


def interval(e) -> tuple[int, int, bool]:
    """(lo, hi, ok) of e over its variables' layout ranges, by interval arithmetic with the lowering's intermediate
    values of \\div and % on a negative dividend; ok is False if any of them leaves int64."""
    k = e[0]
    if k == "var":
        return (*VARS[e[1]][0], True)
    if k == "num":
        return e[1], e[1], True
    if k == "neg":
        lo, hi, ok = interval(e[1])
        return -hi, -lo, ok and INT64_MIN <= -hi and -lo <= INT64_MAX
    if k == "if":
        oks = [interval(x)[2] for x in e[2:4]]
        (l1, h1, o1), (l2, h2, o2) = interval(e[4]), interval(e[5])
        return min(l1, l2), max(h1, h2), all(oks) and o1 and o2
    (al, ah, ao), (bl, bh, bo) = interval(e[1]), interval(e[2])
    if k == "+":
        lo, hi = al + bl, ah + bh
    elif k == "-":
        lo, hi = al - bh, ah - bl
    elif k == "*":
        c = [al * bl, al * bh, ah * bl, ah * bh]
        lo, hi = min(c), max(c)
    elif k == "\\div":
        c = [al // bl, al // bh, ah // bl, ah // bh]
        lo, hi = min(c), max(c)
        if al < 0:
            ao = ao and -al + bh - 1 <= INT64_MAX
    else:
        lo, hi = (0, min(bh - 1, ah)) if al >= 0 else (0, bh - 1)
        if al < 0:
            ao = ao and 2 * bh - 1 <= INT64_MAX
    return lo, hi, ao and bo and INT64_MIN <= lo and hi <= INT64_MAX


def envs():
    names = sorted(VARS)
    grid = np.array(np.meshgrid(*[VARS[n][1] for n in names], indexing="ij"), dtype=object).reshape(len(names), -1).T
    return [dict(zip(names, (int(v) for v in row))) for row in grid]


_rng = random.Random(20261019)
CORPUS = [gen(_rng, 3) for _ in range(360)]
R_BOUND = 1 << 62                 # the result field: -2^62 .. 2^62 - 1 (a 63-bit atom)

CORPUS_TLA = """---- MODULE Corpus ----
EXTENDS Integers
VARIABLES a, b, c, p, tag, r
Layout == /\\ a \\in -8 .. 8 /\\ b \\in -2147483650 .. 2147483650 /\\ c \\in 0 .. 1099511627776
          /\\ p \\in 1 .. 2147483648 /\\ tag \\in 0 .. {ntag} /\\ r \\in -4611686018427387904 .. 4611686018427387903
Init == /\\ a \\in {{-7, -1, 0, 5}} /\\ b \\in {{-2147483649, 2147483647, 2147483648}}
        /\\ c \\in {{0, 1099511627775, 1099511627776}} /\\ p \\in {{1, 3, 2147483648}} /\\ tag = 0 /\\ r = 0
{actions}
Next == {next}
====
"""


def corpus_spec(exprs: list) -> str:
    acts = [f"E{i} == tag = 0 /\\ tag' = {i + 1} /\\ r' = {tla(e)} /\\ UNCHANGED <<a, b, c, p>>"
            for i, e in enumerate(exprs)]
    return CORPUS_TLA.format(ntag=len(exprs), actions="\n".join(acts),
                             next=" \\/ ".join(f"E{i}" for i in range(len(exprs))))


CORPUS_CFG = "\\* kspec: LAYOUT Layout\nINIT Init\nNEXT Next\nCHECK_DEADLOCK FALSE\n"


def split_corpus():
    """(expressions to run, expressions beyond int64) of the corpus: those with every interval in int64 and every
    value within the result field run, those with an interval beyond int64 are refused."""
    run, refused = [], []
    for e in CORPUS:
        ok = interval(e)[2]
        if ok and all(-R_BOUND <= value(e, env) < R_BOUND for env in envs()):
            run.append(e)
        elif not ok:
            refused.append(e)
    return run, refused


def test_corpus_covers_both_sides():
    run, refused = split_corpus()
    assert len(run) >= 150 and len(refused) >= 20
    ops = {e[0] for e in run}
    assert ops >= {"+", "-", "*", "neg", "\\div", "%", "if"}
    # past 32 bits, in the values that are stored as well as in the intervals
    assert any(max(abs(value(e, env)) for env in envs()) >= 1 << 40 for e in run)


@pytest.mark.parametrize("part", range(3))
def test_corpus_values_agree_with_exact_integers(part, tmp_path):
    """Every expression as one action `r' = expr`: the values of r per action, on the lowered model (both forms of
    Next) and on Oracle A, are the exact values over every combination of the operands."""
    run, _ = split_corpus()
    exprs = run[part::3]
    (tmp_path / "Corpus.tla").write_text(corpus_spec(exprs))
    m = lower_model("Corpus", [str(tmp_path)], CORPUS_CFG)
    ref = oracle_a("Corpus", [str(tmp_path)], CORPUS_CFG)
    assert_agrees_with_oracle_a(m, ref)
    got: dict[int, set] = {}
    for row in run_host(m, dump=True)["states"]:
        st = m.decode_state([int(w) for w in row])
        if st["tag"]:
            got.setdefault(st["tag"] - 1, set()).add((st["a"], st["b"], st["c"], st["p"], st["r"]))
    for i, e in enumerate(exprs):
        want = {(env["a"], env["b"], env["c"], env["p"], value(e, env)) for env in envs()}
        assert got.get(i) == want, f"{tla(e)}"


def test_corpus_beyond_int64_is_refused(tmp_path):
    """An expression whose interval leaves int64 is refused with a LowerError naming it, unless the lowering folds the
    offending part away (a constant, or a comparison its intervals decide); then its values are exact."""
    _, refused = split_corpus()
    folded = []
    for i, e in enumerate(refused):
        (tmp_path / "Corpus.tla").write_text(corpus_spec([e]))
        try:
            m = lower_model("Corpus", [str(tmp_path)], CORPUS_CFG)
        except LowerError as err:
            # the expression (or the folded constant) that leaves int64
            assert re.match(r"the integer (expression .+ takes values in .+|-?\d+ is) beyond 64-bit integers", str(err)), err
            continue
        folded.append((e, m))
    assert len(folded) < len(refused) / 2
    for e, m in folded[:5]:
        if all(-R_BOUND <= value(e, env) < R_BOUND for env in envs()):
            vals = {m.decode_state([int(w) for w in row])["r"] for row in run_host(m, dump=True)["states"][len(envs()):]}
            assert vals == {value(e, env) for env in envs()}


def test_refusal_names_the_expression(tmp_path):
    (tmp_path / "Corpus.tla").write_text(corpus_spec([("*", ("var", "c"), ("*", ("var", "c"), ("var", "b")))]))
    with pytest.raises(LowerError, match=r"the integer expression c \* b takes values in .* beyond 64-bit integers"):
        lower_model("Corpus", [str(tmp_path)], CORPUS_CFG)


# ---------------------------------------------------------------------------------------------------------------------
# wide sets and ranges

WIDE_TLA = """---- MODULE Wide ----
EXTENDS Integers
VARIABLES x, y
TypeOk == x \\in {1, 2147483647} /\\ y \\in 0 .. 3
Init == x = 1 /\\ y = 0
Grow == y < 3 /\\ x \\in y .. 2147483647 /\\ x' = 2147483647 /\\ y' = y + 1
Enum == \\E k \\in y .. x : x' = x /\\ y' = k % 4
Next == Grow
NextEnum == Grow \\/ Enum
====
"""


def lower_capped(tmp_path, next_name: str) -> subprocess.CompletedProcess:
    """Lower Wide.tla with Next = next_name in a child process limited to 2 GiB of address space."""
    (tmp_path / "Wide.tla").write_text(WIDE_TLA)
    code = textwrap.dedent(f"""
        import resource, sys
        resource.setrlimit(resource.RLIMIT_AS, (2 << 30, 2 << 30))
        sys.path.insert(0, {ROOT!r})
        from kafka_specification_b200.lower.model import lower_model
        from kafka_specification_b200.lower.svals import LowerError
        try:
            m = lower_model("Wide", [{str(tmp_path)!r}], "INIT Init NEXT {next_name} INVARIANT TypeOk\\n")
        except LowerError as err:
            print("LowerError:", err)
        else:
            print("lowered", m.words)
    """)
    return subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)


def test_wide_sparse_set_and_wide_range_membership_lower_in_bounded_memory(tmp_path):
    p = lower_capped(tmp_path, "Next")
    assert p.returncode == 0 and p.stdout.startswith("lowered"), p.stdout + p.stderr
    m = lower_model("Wide", [str(tmp_path)], "INIT Init NEXT Next INVARIANT TypeOk\n")
    r = run_host(m)
    assert (r["distinct"], r["generated"], r["levels"], r["fail"]) == (4, 4, [1, 1, 1, 1], 0)


def test_enumerating_a_wide_runtime_range_is_refused(tmp_path):
    p = lower_capped(tmp_path, "NextEnum")
    assert p.returncode == 0, p.stdout + p.stderr
    assert p.stdout.startswith("LowerError: a run-time range may hold more than 65536 integers"), p.stdout
