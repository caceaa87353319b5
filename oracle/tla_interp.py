"""Oracle A — a direct, slow, exact interpreter for the TLA+ text of the reference specs.

TEST INFRASTRUCTURE ONLY.  Nothing under ``kafka_specification_b200/`` may import this file;
only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline legs may.

PARITY UNPINNED: the reference (hachikuji/kafka-specification @ d68782b) contains no TLC
output, no ``.cfg`` and no golden state counts, and TLC itself (third-party, not vendored, no
version pinned; Toolbox footers bracket it to roughly 1.5.7-1.7.0) cannot run here (no JVM).
This interpreter is therefore pinned only against (a) analytic closed forms derived from the
spec text (IdSequence.tla:30-39 -> MaxId+2 states; FiniteReplicatedLog.tla:97-118 ->
(sum_{e<=L} R^e)^n states, depth n*L+1), (b) the reference's qualitative claims (Kip320.tla:168-171
hold; KafkaTruncateToHighWatermark.tla:23-27, Kip279.tla:20-23, Kip320.tla:126-133,
Kip320FirstTry.tla:27-33 violate StrongIsr), and (c) agreement with the independent hand-written
C restatement in ``oracle/kspec_oracle.c``.

What it does: evaluates ``Init``/``Next``/invariants/constraints exactly as written in the
``.tla`` files (parsed by the shared front-end, no lowering, no packing), with Python
frozensets / immutable maps as TLA+ values and exact object equality for state identity, using
TLC's operational rules (SURVEY.md App. D, from the published TLC design):

* action evaluation branches on every positive-position ``\\/`` and bounded ``\\E``, expanding
  operator definitions and LET in place; everything else is a plain boolean;
* ``states generated`` = #init + every successor produced (duplicates and self-loops count);
* a successor violating a CONSTRAINT is counted as generated and invariant-checked but is
  neither stored nor explored; so is an initial state violating one (``out_of_model`` counts both,
  every generation of such a state);
* depth = number of BFS levels, Init = level 1;
* ``=`` between incomparable kinds (int vs record, string vs int) is an error, except that a
  model value is simply unequal to anything else.
"""
from __future__ import annotations

import itertools
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from kafka_specification_b200.frontend.cfg import Config, ModelValue, parse_cfg  # noqa: E402
from kafka_specification_b200.frontend.modules import ModuleContext, load_root  # noqa: E402
from kafka_specification_b200.frontend.tla_parser import Def  # noqa: E402


from kafka_specification_b200.frontend.values import EvalError, FnVal, fmt, sort_key  # noqa: E402


# ---------------------------------------------------------------------------
# lazy (non-enumerated) sets
# ---------------------------------------------------------------------------
class LazySet:
    def enumerate(self):
        raise EvalError(f"cannot enumerate {self!r}")

    def materialize(self) -> frozenset:
        return frozenset(self.enumerate())


class NatSet(LazySet):
    def __init__(self, lo=0):
        self.lo = lo

    def __contains__(self, v):
        return isinstance(v, int) and not isinstance(v, bool) and v >= self.lo

    def __repr__(self):
        return "Nat"


class IntSet(LazySet):
    def __contains__(self, v):
        return isinstance(v, int) and not isinstance(v, bool)

    def __repr__(self):
        return "Int"


class RecSet(LazySet):
    def __init__(self, fields: dict):
        self.fields = fields

    def __contains__(self, v):
        if not isinstance(v, FnVal) or v.domain() != frozenset(self.fields):
            return False
        return all(set_contains(s, v.apply(f)) for f, s in self.fields.items())

    def enumerate(self):
        names = list(self.fields)
        for combo in itertools.product(*[sorted(set_elems(self.fields[n]), key=sort_key) for n in names]):
            yield FnVal(dict(zip(names, combo)))

    def __repr__(self):
        return "[" + ", ".join(f"{k}: {v!r}" for k, v in self.fields.items()) + "]"


class FnSet(LazySet):
    def __init__(self, dom, rng):
        self.dom, self.rng = dom, rng

    def __contains__(self, v):
        if not isinstance(v, FnVal) or v.domain() != frozenset(set_elems(self.dom)):
            return False
        return all(set_contains(self.rng, x) for _, x in v.items)

    def enumerate(self):
        dom = sorted(set_elems(self.dom), key=sort_key)
        rng = sorted(set_elems(self.rng), key=sort_key)
        for combo in itertools.product(rng, repeat=len(dom)):
            yield FnVal(dict(zip(dom, combo)))

    def __repr__(self):
        return f"[{self.dom!r} -> {self.rng!r}]"


class PowerSet(LazySet):
    def __init__(self, base):
        self.base = base

    def __contains__(self, v):
        if isinstance(v, LazySet):
            v = v.materialize()
        return isinstance(v, frozenset) and all(set_contains(self.base, x) for x in v)

    def enumerate(self):
        elems = sorted(set_elems(self.base), key=sort_key)
        for r in range(len(elems) + 1):
            for c in itertools.combinations(elems, r):
                yield frozenset(c)

    def __repr__(self):
        return f"SUBSET {self.base!r}"


class SeqSet(LazySet):
    """Seq(S): every finite sequence over S -- membership only, never enumerated."""

    def __init__(self, base):
        self.base = base

    def __contains__(self, v):
        return isinstance(v, tuple) and all(set_contains(self.base, x) for x in v)

    def enumerate(self):
        raise EvalError("Seq(S) is infinite and cannot be enumerated")

    def __repr__(self):
        return f"Seq({self.base!r})"


class CrossSet(LazySet):
    """S1 \\X ... \\X Sn with a component that is not enumerable (e.g. Nat): membership only."""

    def __init__(self, parts):
        self.parts = parts

    def __contains__(self, v):
        return isinstance(v, tuple) and len(v) == len(self.parts) and all(set_contains(s, x) for s, x in zip(self.parts, v))

    def enumerate(self):
        for combo in itertools.product(*[sorted(set_elems(s), key=sort_key) for s in self.parts]):
            yield tuple(combo)

    def __repr__(self):
        return " \\X ".join(repr(s) for s in self.parts)


class UnionSet(LazySet):
    def __init__(self, a, b):
        self.a, self.b = a, b

    def __contains__(self, v):
        return set_contains(self.a, v) or set_contains(self.b, v)

    def enumerate(self):
        seen = set()
        for s in (self.a, self.b):
            for x in set_elems(s):
                if x not in seen:
                    seen.add(x)
                    yield x

    def __repr__(self):
        return f"({self.a!r} \\union {self.b!r})"


def is_set(v) -> bool:
    return isinstance(v, (frozenset, LazySet))


def set_contains(s, v) -> bool:
    if isinstance(s, frozenset):
        if isinstance(v, LazySet):
            v = v.materialize()
        return v in s
    if isinstance(s, LazySet):
        return v in s
    raise EvalError(f"\\in applied to non-set {s!r}")


def set_elems(s):
    if isinstance(s, frozenset):
        return s
    if isinstance(s, LazySet):
        return s.materialize()
    raise EvalError(f"not a set: {s!r}")


def kind_of(v) -> str:
    if isinstance(v, bool):
        return "bool"
    if isinstance(v, int):
        return "int"
    if isinstance(v, str):
        return "str"
    if isinstance(v, ModelValue):
        return "mv"
    if isinstance(v, FnVal):
        return "fn"
    if is_set(v):
        return "set"
    if isinstance(v, tuple):
        return "tuple"
    raise EvalError(f"unknown value kind {v!r}")


# module Sequences (a sequence is a Python tuple)
SEQ_BUILTINS = {"Len": 1, "Head": 1, "Tail": 1, "Append": 2, "SubSeq": 3, "Seq": 1}


def seq_builtin(name, args):
    if name == "Seq":
        return SeqSet(args[0])
    s = args[0]
    if not isinstance(s, tuple):
        raise EvalError(f"{name} applied to the non-sequence {fmt(s)}")
    if name == "Len":
        return len(s)
    if name == "Head":
        if not s:
            raise EvalError("Head of the empty sequence")
        return s[0]
    if name == "Tail":
        if not s:
            raise EvalError("Tail of the empty sequence")
        return s[1:]
    if name == "Append":
        return s + (args[1],)
    m, k = args[1], args[2]
    if k < m:
        return ()
    if m < 1 or k > len(s):
        raise EvalError(f"SubSeq bounds {m}..{k} outside 1..{len(s)}")
    return s[m - 1:k]


def tla_eq(a, b) -> bool:
    ka, kb = kind_of(a), kind_of(b)
    if ka == "mv" or kb == "mv":
        return ka == kb and a == b          # untyped model values: unequal to everything else
    if ka != kb:
        raise EvalError(f"attempted to compare incomparable values {fmt(a)} and {fmt(b)}")
    if ka == "set":
        return set_elems(a) == set_elems(b)
    return a == b


class Thunk:
    """Lazily evaluated expression (operator argument or LET definition)."""
    __slots__ = ("expr", "ctx", "fm", "env", "_val", "_done")

    def __init__(self, expr, ctx, fm, env):
        self.expr, self.ctx, self.fm, self.env = expr, ctx, fm, env
        self._done = False
        self._val = None


class Closure:
    """LET-bound operator with parameters."""
    __slots__ = ("defn", "ctx", "fm", "env")

    def __init__(self, defn, ctx, fm, env):
        self.defn, self.ctx, self.fm, self.env = defn, ctx, fm, env


# ---------------------------------------------------------------------------
# interpreter
# ---------------------------------------------------------------------------
class Interp:
    def __init__(self, root: ModuleContext, cfg: Config):
        self.root = root
        self.cfg = cfg
        root.const_overrides = dict(cfg.overrides)
        self.variables = list(root.variables)
        self.const_values = dict(cfg.constants)
        for c in root.constants:
            if c not in self.const_values and c not in cfg.overrides:
                raise EvalError(f"constant {c} has no value in the cfg")
        self._const_cache: dict = {}
        self._reads = 0         # bumped whenever a state variable or bound name is read

    # -- name resolution ---------------------------------------------------
    def lookup(self, name, ctx, fm, env, st, st1):
        if name in env:
            v = env[name]
            self._reads += 1
            if isinstance(v, Thunk):
                return self.force(v, st, st1)
            return v
        r = ctx.resolve(name, fm)
        if r is None:
            if name == "Nat":
                return NatSet()
            if name == "Int":
                return IntSet()
            if name == "BOOLEAN":
                return frozenset({True, False})
            raise EvalError(f"unknown identifier {name} (module {ctx.path})")
        if r.kind == "const":
            return self.const_values[name]
        if r.kind == "var":
            self._reads += 1
            if st is None:
                raise EvalError(f"state variable {name} read in a constant context")
            if name not in st:
                raise EvalError(f"variable {name} read before being assigned")
            return st[name]
        if r.kind == "subst":
            return self.ev(r.expr, r.ctx, r.from_module, {}, st, st1)
        if r.kind == "def":
            d = r.defn
            if d.params:
                raise EvalError(f"operator {name} used without arguments")
            key = (id(r.ctx), d.module, d.name)
            if key in self._const_cache:
                return self._const_cache[key]
            before = self._reads
            v = self.ev(d.body, r.ctx, d.module, {}, st, st1)
            if self._reads == before:
                self._const_cache[key] = v
            return v
        raise EvalError(f"{name} is a module instance, not a value")

    def force(self, t: Thunk, st, st1):
        if not t._done:
            t._val = self.ev(t.expr, t.ctx, t.fm, t.env, st, st1)
            t._done = True
        return t._val

    def resolve_var(self, e, ctx, fm, env):
        """If expression e denotes a state variable (through substitutions), its root name."""
        if e[0] != "id" or e[1] in env:
            return None
        r = ctx.resolve(e[1], fm)
        if r is None:
            return None
        if r.kind == "var":
            return e[1]
        if r.kind == "subst":
            return self.resolve_var(r.expr, r.ctx, r.from_module, {})
        return None

    def find_operator(self, e, ctx, fm, env):
        """For ('id'|'app'|'inst') nodes naming a user definition: (Def, defctx, args, argctx)."""
        k = e[0]
        if k == "inst":
            r = ctx.resolve(e[1], fm)
            if r is None or r.kind != "inst":
                raise EvalError(f"{e[1]} is not a module instance")
            d = r.inst.find_def(e[2], None)
            if d is None:
                raise EvalError(f"{e[1]}!{e[2]} is not defined")
            if d.local:
                raise EvalError(f"{e[1]}!{e[2]} is LOCAL")
            return d, r.inst, e[3]
        name = e[1]
        if name in env:
            v = env[name]
            if isinstance(v, Closure):
                return v, None, (e[2] if k == "app" else [])
            return None
        r = ctx.resolve(name, fm)
        if r is not None and r.kind == "def":
            return r.defn, r.ctx, (e[2] if k == "app" else [])
        return None

    def bind_call(self, target, defctx, args, ctx, fm, env):
        """Returns (body, ctx, fm, env) for evaluating a user operator application."""
        if isinstance(target, Closure):
            d = target.defn
            if len(d.params) != len(args):
                raise EvalError(f"arity mismatch calling {d.name}")
            new_env = dict(target.env)
            for p, a in zip(d.params, args):
                new_env[p] = Thunk(a, ctx, fm, env)
            return d.body, target.ctx, target.fm, new_env
        d: Def = target
        if len(d.params) != len(args):
            raise EvalError(f"arity mismatch calling {d.name}")
        new_env = {p: Thunk(a, ctx, fm, env) for p, a in zip(d.params, args)}
        return d.body, defctx, d.module, new_env

    # -- expression evaluation ----------------------------------------------
    def ev(self, e, ctx, fm, env, st, st1):
        k = e[0]
        if k == "num" or k == "str" or k == "bool":
            return e[1]
        if k == "id":
            if e[1] not in env:
                op = self.find_operator(e, ctx, fm, env)
                if op is not None and not isinstance(op[0], Closure) and op[0].params == []:
                    return self.lookup(e[1], ctx, fm, env, st, st1)
            return self.lookup(e[1], ctx, fm, env, st, st1)
        if k == "app" or k == "inst":
            op = self.find_operator(e, ctx, fm, env)
            if op is None:
                if k == "app" and e[1] == "Cardinality" and len(e[2]) == 1:
                    return len(set_elems(self.ev(e[2][0], ctx, fm, env, st, st1)))
                if k == "app" and e[1] == "Permutations" and len(e[2]) == 1:
                    # TLC module: the set of all permutations (bijections S -> S) of a finite set
                    elems = sorted(set_elems(self.ev(e[2][0], ctx, fm, env, st, st1)), key=sort_key)
                    return frozenset(FnVal(dict(zip(elems, p))) for p in itertools.permutations(elems))
                if k == "app" and SEQ_BUILTINS.get(e[1]) == len(e[2]):
                    return seq_builtin(e[1], [self.ev(x, ctx, fm, env, st, st1) for x in e[2]])
                raise EvalError(f"unknown operator {e[1]}")
            target, defctx, args = op
            if k == "inst" and not target.params:
                key = (id(defctx), target.module, target.name)
                if key in self._const_cache:
                    return self._const_cache[key]
                before = self._reads
                v = self.ev(target.body, defctx, target.module, {}, st, st1)
                if self._reads == before:
                    self._const_cache[key] = v
                return v
            body, c2, fm2, env2 = self.bind_call(target, defctx, args, ctx, fm, env)
            return self.ev(body, c2, fm2, env2, st, st1)
        if k == "and":
            for x in e[1]:
                if not self.ev_bool(x, ctx, fm, env, st, st1):
                    return False
            return True
        if k == "or":
            for x in e[1]:
                if self.ev_bool(x, ctx, fm, env, st, st1):
                    return True
            return False
        if k == "not":
            return not self.ev_bool(e[1], ctx, fm, env, st, st1)
        if k == "neg":
            return -self.ev_int(e[1], ctx, fm, env, st, st1)
        if k == "binop":
            return self.ev_binop(e, ctx, fm, env, st, st1)
        if k == "if":
            if self.ev_bool(e[1], ctx, fm, env, st, st1):
                return self.ev(e[2], ctx, fm, env, st, st1)
            return self.ev(e[3], ctx, fm, env, st, st1)
        if k == "let":
            return self.ev(e[2], ctx, fm, self.let_env(e[1], ctx, fm, env), st, st1)
        if k == "case":
            for g, x in e[1]:
                if self.ev_bool(g, ctx, fm, env, st, st1):
                    return self.ev(x, ctx, fm, env, st, st1)
            if e[2] is None:
                raise EvalError("CASE: no arm applies and there is no OTHER")
            return self.ev(e[2], ctx, fm, env, st, st1)
        if k == "quant":
            is_exists = e[1] == "E"
            for env2 in self.bindings(e[2], ctx, fm, env, st, st1):
                b = self.ev_bool(e[3], ctx, fm, env2, st, st1)
                if b and is_exists:
                    return True
                if not b and not is_exists:
                    return False
            return not is_exists
        if k == "choose":
            s = self.ev(e[2], ctx, fm, env, st, st1)
            for x in sorted(set_elems(s), key=sort_key):
                env2 = dict(env)
                env2[e[1]] = x
                if self.ev_bool(e[3], ctx, fm, env2, st, st1):
                    return x
            raise EvalError("CHOOSE: no element satisfies the predicate")
        if k == "setenum":
            return frozenset(self.ev(x, ctx, fm, env, st, st1) for x in e[1])
        if k == "setmap":
            return frozenset(self.ev(e[1], ctx, fm, env2, st, st1)
                             for env2 in self.bindings(e[2], ctx, fm, env, st, st1))
        if k == "setfilter":
            s = self.ev(e[2], ctx, fm, env, st, st1)
            out = []
            for x in set_elems(s):
                env2 = dict(env)
                env2[e[1]] = x
                if self.ev_bool(e[3], ctx, fm, env2, st, st1):
                    out.append(x)
            return frozenset(out)
        if k == "subset":
            base = self.ev(e[1], ctx, fm, env, st, st1)
            if isinstance(base, frozenset) and len(base) <= 12:
                return PowerSet(base).materialize()
            return PowerSet(base)
        if k == "union_all":
            s = self.ev(e[1], ctx, fm, env, st, st1)
            out = set()
            for x in set_elems(s):
                out |= set_elems(x)
            return frozenset(out)
        if k == "domain":
            f = self.ev(e[1], ctx, fm, env, st, st1)
            if isinstance(f, tuple):
                return frozenset(range(1, len(f) + 1))
            if not isinstance(f, FnVal):
                raise EvalError("DOMAIN of a non-function")
            return f.domain()
        if k == "fnlit":
            d = {}
            for env2, key in self.bindings_with_key(e[1], ctx, fm, env, st, st1):
                d[key] = self.ev(e[2], ctx, fm, env2, st, st1)
            return FnVal(d)
        if k == "fnapp":
            f = self.ev(e[1], ctx, fm, env, st, st1)
            args = [self.ev(a, ctx, fm, env, st, st1) for a in e[2]]
            key = args[0] if len(args) == 1 else tuple(args)
            if isinstance(f, tuple):
                if isinstance(key, bool) or not isinstance(key, int) or not 1 <= key <= len(f):
                    raise EvalError(f"sequence index {fmt(key)} outside 1..{len(f)}")
                return f[key - 1]
            if not isinstance(f, FnVal):
                raise EvalError(f"applying non-function {fmt(f)}")
            return f.apply(key)
        if k == "fnset":
            dom = self.ev(e[1], ctx, fm, env, st, st1)
            rng = self.ev(e[2], ctx, fm, env, st, st1)
            return FnSet(dom, rng)
        if k == "rec":
            return FnVal({f: self.ev(x, ctx, fm, env, st, st1) for f, x in e[1]})
        if k == "recset":
            fields = {f: self.ev(x, ctx, fm, env, st, st1) for f, x in e[1]}
            if all(isinstance(s, frozenset) for s in fields.values()):
                n = 1
                for s in fields.values():
                    n *= len(s)
                if n <= 100000:
                    return RecSet(fields).materialize()
            return RecSet(fields)
        if k == "dot":
            r = self.ev(e[1], ctx, fm, env, st, st1)
            if not isinstance(r, FnVal):
                raise EvalError(f"field .{e[2]} of non-record {fmt(r)}")
            return r.apply(e[2])
        if k == "except":
            f = self.ev(e[1], ctx, fm, env, st, st1)
            for path, rhs in e[2]:
                f = self.except_update(f, path, rhs, ctx, fm, env, st, st1)
            return f
        if k == "at":
            if "@" not in env:
                raise EvalError("@ outside EXCEPT")
            return env["@"]
        if k == "tuple":
            return tuple(self.ev(x, ctx, fm, env, st, st1) for x in e[1])
        if k == "cross":
            parts = [self.ev(x, ctx, fm, env, st, st1) for x in e[1]]
            cs = CrossSet(parts)
            return cs.materialize() if all(isinstance(p, frozenset) for p in parts) else cs
        if k == "prime":
            if st1 is None:
                raise EvalError("primed expression outside an action")
            return self.ev(e[1], ctx, fm, env, st1, None)
        if k == "unchanged":
            for v in self.unchanged_vars(e[1], ctx, fm, env):
                if st1 is None or v not in st1:
                    raise EvalError(f"UNCHANGED {v} evaluated before {v}' is assigned")
                if st1[v] != st[v]:
                    return False
            return True
        raise EvalError(f"cannot evaluate node kind {k}")

    def ev_bool(self, e, ctx, fm, env, st, st1) -> bool:
        v = self.ev(e, ctx, fm, env, st, st1)
        if not isinstance(v, bool):
            raise EvalError(f"expected a boolean, got {fmt(v)}")
        return v

    def ev_int(self, e, ctx, fm, env, st, st1) -> int:
        v = self.ev(e, ctx, fm, env, st, st1)
        if isinstance(v, bool) or not isinstance(v, int):
            raise EvalError(f"expected an integer, got {fmt(v)}")
        return v

    def ev_binop(self, e, ctx, fm, env, st, st1):
        op = e[1]
        if op == "=>":
            return (not self.ev_bool(e[2], ctx, fm, env, st, st1)) or self.ev_bool(e[3], ctx, fm, env, st, st1)
        if op in ("\\in", "\\notin") and e[3][0] == "binop" and e[3][1] == "..":
            # x \in lo .. hi by its bounds: the same truth value without building a set of up to 2^40 integers
            x = self.ev(e[2], ctx, fm, env, st, st1)
            lo, hi = self.ev_int(e[3][2], ctx, fm, env, st, st1), self.ev_int(e[3][3], ctx, fm, env, st, st1)
            inside = not isinstance(x, bool) and isinstance(x, int) and lo <= x <= hi
            return inside if op == "\\in" else not inside
        a = self.ev(e[2], ctx, fm, env, st, st1)
        b = self.ev(e[3], ctx, fm, env, st, st1)
        if op == "=":
            return tla_eq(a, b)
        if op == "#":
            return not tla_eq(a, b)
        if op in ("<", ">", "<=", ">=", "+", "-", "*", "\\div", "%", ".."):
            for x in (a, b):
                if isinstance(x, bool) or not isinstance(x, int):
                    raise EvalError(f"operator {op} applied to non-integer {fmt(x)}")
            if op == "<":
                return a < b
            if op == ">":
                return a > b
            if op == "<=":
                return a <= b
            if op == ">=":
                return a >= b
            if op == "+":
                return a + b
            if op == "-":
                return a - b
            if op == "*":
                return a * b
            if op in ("\\div", "%"):
                if b <= 0:
                    raise EvalError(f"{op} with the non-positive divisor {b}")
                return a // b if op == "\\div" else a % b
            return frozenset(range(a, b + 1))
        if op == "\\o":
            if not isinstance(a, tuple) or not isinstance(b, tuple):
                raise EvalError("\\o applied to a non-sequence")
            return a + b
        if op == "\\in":
            return set_contains(b, a)
        if op == "\\notin":
            return not set_contains(b, a)
        if op == "\\subseteq":
            return all(set_contains(b, x) for x in set_elems(a))
        if op == "\\union":
            if isinstance(a, frozenset) and isinstance(b, frozenset):
                return a | b
            try:
                return frozenset(set_elems(a)) | frozenset(set_elems(b))
            except EvalError:
                return UnionSet(a, b)
        if op == "\\intersect":
            return frozenset(x for x in set_elems(a) if set_contains(b, x))
        if op == "\\":
            return frozenset(x for x in set_elems(a) if not set_contains(b, x))
        if op == "<=>":
            return bool(a) == bool(b)
        raise EvalError(f"unsupported operator {op}")

    def let_env(self, defs, ctx, fm, env):
        env2 = dict(env)
        for d in defs:
            if d.params:
                env2[d.name] = Closure(d, ctx, fm, env2)
            else:
                env2[d.name] = Thunk(d.body, ctx, fm, env2)
        return env2

    def bindings(self, bounds, ctx, fm, env, st, st1):
        for env2, _ in self.bindings_with_key(bounds, ctx, fm, env, st, st1):
            yield env2

    def bindings_with_key(self, bounds, ctx, fm, env, st, st1):
        names, sets = [], []
        for ns, sexpr in bounds:
            s = sorted(set_elems(self.ev(sexpr, ctx, fm, env, st, st1)), key=sort_key)
            for n in ns:
                names.append(n)
                sets.append(s)
        for combo in itertools.product(*sets):
            env2 = dict(env)
            for n, v in zip(names, combo):
                env2[n] = v
            yield env2, (combo[0] if len(combo) == 1 else tuple(combo))

    def except_update(self, f, path, rhs, ctx, fm, env, st, st1):
        step = path[0]
        key = self.ev(step[1], ctx, fm, env, st, st1) if step[0] == "idx" else step[1]
        if isinstance(f, tuple):
            if isinstance(key, bool) or not isinstance(key, int) or not 1 <= key <= len(f):
                raise EvalError(f"EXCEPT on sequence index {fmt(key)} outside 1..{len(f)}")
            old = f[key - 1]
            if len(path) == 1:
                env2 = dict(env)
                env2["@"] = old
                new = self.ev(rhs, ctx, fm, env2, st, st1)
            else:
                new = self.except_update(old, path[1:], rhs, ctx, fm, env, st, st1)
            return f[:key - 1] + (new,) + f[key:]
        if not isinstance(f, FnVal):
            raise EvalError("EXCEPT applied to a non-function")
        old = f.apply(key)
        if len(path) == 1:
            env2 = dict(env)
            env2["@"] = old
            new = self.ev(rhs, ctx, fm, env2, st, st1)
        else:
            new = self.except_update(old, path[1:], rhs, ctx, fm, env, st, st1)
        return f.updated(key, new)

    def unchanged_vars(self, e, ctx, fm, env) -> list[str]:
        if e[0] == "tuple":
            out = []
            for x in e[1]:
                out.extend(self.unchanged_vars(x, ctx, fm, env))
            return out
        v = self.resolve_var(e, ctx, fm, env)
        if v is not None:
            return [v]
        if e[0] == "id":
            r = ctx.resolve(e[1], fm)
            if r is not None and r.kind == "def" and not r.defn.params:
                return self.unchanged_vars(r.defn.body, r.ctx, r.defn.module, {})
            if r is not None and r.kind == "subst":
                return self.unchanged_vars(r.expr, r.ctx, r.from_module, {})
        raise EvalError(f"UNCHANGED of a non-variable expression {e!r}")

    # -- actions (TLC getNextStates rule) ------------------------------------
    def next_states(self, next_expr, st: dict) -> list[dict]:
        out: list[dict] = []
        self._next([(next_expr, self.root, None, {})], st, {}, out)
        return out

    def _next(self, items, st, st1, out):
        if not items:
            for v in self.variables:
                if v not in st1:
                    raise EvalError(f"successor leaves {v}' unassigned")
            out.append(st1)
            return
        (e, ctx, fm, env), rest = items[0], items[1:]
        k = e[0]
        if k == "and":
            self._next([(x, ctx, fm, env) for x in e[1]] + rest, st, st1, out)
            return
        if k == "or":
            for x in e[1]:
                self._next([(x, ctx, fm, env)] + rest, st, st1, out)
            return
        if k == "quant" and e[1] == "E":
            for env2 in self.bindings(e[2], ctx, fm, env, st, st1):
                self._next([(e[3], ctx, fm, env2)] + rest, st, st1, out)
            return
        if k == "let":
            self._next([(e[2], ctx, fm, self.let_env(e[1], ctx, fm, env))] + rest, st, st1, out)
            return
        if k == "if":
            branch = e[2] if self.ev_bool(e[1], ctx, fm, env, st, st1) else e[3]
            self._next([(branch, ctx, fm, env)] + rest, st, st1, out)
            return
        if k in ("id", "app", "inst"):
            op = None
            if not (k == "id" and e[1] in env and not isinstance(env[e[1]], Closure)):
                op = self.find_operator(e, ctx, fm, env)
            if op is not None:
                target, defctx, args = op
                body, c2, fm2, env2 = self.bind_call(target, defctx, args, ctx, fm, env)
                self._next([(body, c2, fm2, env2)] + rest, st, st1, out)
                return
        if k == "binop" and e[1] in ("=", "\\in") and e[2][0] == "prime":
            v = self.resolve_var(e[2][1], ctx, fm, env)
            if v is not None and v not in st1:
                rhs = self.ev(e[3], ctx, fm, env, st, st1)
                if e[1] == "=":
                    self._next(rest, st, {**st1, v: rhs}, out)
                else:
                    for x in sorted(set_elems(rhs), key=sort_key):
                        self._next(rest, st, {**st1, v: x}, out)
                return
        if k == "unchanged":
            new1 = st1
            for v in self.unchanged_vars(e[1], ctx, fm, env):
                if v in new1:
                    if new1[v] != st[v]:
                        return
                else:
                    new1 = {**new1, v: st[v]}
            self._next(rest, st, new1, out)
            return
        if self.ev_bool(e, ctx, fm, env, st, st1):
            self._next(rest, st, st1, out)

    # -- init ----------------------------------------------------------------
    def init_states(self, init_expr) -> list[dict]:
        """Init predicates: conjunctions of ``var = e`` / ``var \\in S`` (+ definitions)."""
        out: list[dict] = []
        self._init([(init_expr, self.root, None, {})], {}, out)
        return out

    def _init(self, items, st, out):
        if not items:
            for v in self.variables:
                if v not in st:
                    raise EvalError(f"Init leaves {v} unassigned")
            out.append(st)
            return
        (e, ctx, fm, env), rest = items[0], items[1:]
        k = e[0]
        if k == "and":
            self._init([(x, ctx, fm, env) for x in e[1]] + rest, st, out)
            return
        if k == "or":
            for x in e[1]:
                self._init([(x, ctx, fm, env)] + rest, st, out)
            return
        if k == "quant" and e[1] == "E":
            for env2 in self.bindings(e[2], ctx, fm, env, st, None):
                self._init([(e[3], ctx, fm, env2)] + rest, st, out)
            return
        if k == "let":
            self._init([(e[2], ctx, fm, self.let_env(e[1], ctx, fm, env))] + rest, st, out)
            return
        if k in ("id", "app", "inst"):
            op = None
            if not (k == "id" and e[1] in env and not isinstance(env[e[1]], Closure)):
                op = self.find_operator(e, ctx, fm, env)
            if op is not None:
                target, defctx, args = op
                body, c2, fm2, env2 = self.bind_call(target, defctx, args, ctx, fm, env)
                self._init([(body, c2, fm2, env2)] + rest, st, out)
                return
        if k == "binop" and e[1] in ("=", "\\in"):
            v = self.resolve_var(e[2], ctx, fm, env)
            if v is not None and v not in st:
                rhs = self.ev(e[3], ctx, fm, env, st, None)
                if e[1] == "=":
                    self._init(rest, {**st, v: rhs}, out)
                else:
                    for x in sorted(set_elems(rhs), key=sort_key):
                        self._init(rest, {**st, v: x}, out)
                return
        if self.ev_bool(e, ctx, fm, env, st, None):
            self._init(rest, st, out)

    # -- predicates on states --------------------------------------------------
    def eval_named_predicate(self, name: str, st: dict) -> bool:
        r = self.root.resolve(name, None)
        if r is None or r.kind != "def":
            raise EvalError(f"{name} is not defined in {self.root.module_name}")
        return self.ev_bool(r.defn.body, r.ctx, r.defn.module, {}, st, None)

    def check_assumes(self):
        for a, mod in self.root.assumes:
            if not self.ev_bool(a, self.root, mod, {}, None, None):
                raise EvalError(f"ASSUME in module {mod} is false")


# ---------------------------------------------------------------------------
# BFS driver
# ---------------------------------------------------------------------------
def resolve_init_next(root: ModuleContext, cfg: Config):
    """(init_expr, next_expr) from INIT/NEXT or from SPECIFICATION Init /\\ [][Next]_v ..."""
    if cfg.init and cfg.next:
        return ("id", cfg.init), ("id", cfg.next)
    if cfg.specification:
        d = root.find_def(cfg.specification, None)
        if d is None:
            raise EvalError(f"SPECIFICATION {cfg.specification} not found")
        init, nxt = None, None

        def walk(e):
            nonlocal init, nxt
            if e[0] == "and":
                for x in e[1]:
                    walk(x)
            elif e[0] == "box" and e[1][0] == "actionbox":
                nxt = e[1][1]
            elif e[0] in ("fair",):
                pass
            elif init is None:
                init = e
        walk(d.body)
        if init is None or nxt is None:
            raise EvalError("SPECIFICATION is not of the form Init /\\ [][Next]_vars")
        return init, nxt
    raise EvalError("cfg needs INIT+NEXT or SPECIFICATION")


def permute_value(v, mapping: dict):
    """Applies a permutation of model values to a TLA+ value (TLC's SYMMETRY semantics)."""
    if isinstance(v, ModelValue):
        return mapping.get(v, v)
    if isinstance(v, frozenset):
        return frozenset(permute_value(x, mapping) for x in v)
    if isinstance(v, FnVal):
        return FnVal({permute_value(k, mapping): permute_value(x, mapping) for k, x in v.items})
    if isinstance(v, tuple):
        return tuple(permute_value(x, mapping) for x in v)
    return v


def state_text(variables, st: dict) -> str:
    return "\n".join(f"/\\ {v} = {fmt(st[v])}" for v in variables)


def run_bfs(module: str, search_dirs: list[str], cfg_text: str, max_states: int | None = None,
            collect_states: bool = False, stop_on_violation: bool = True) -> dict:
    """Level-synchronous BFS with exact state identity.  Returns a result dictionary."""
    cfg = parse_cfg(cfg_text)
    root = load_root(module, search_dirs)
    it = Interp(root, cfg)
    it.check_assumes()
    init_e, next_e = resolve_init_next(root, cfg)
    variables = it.variables

    perms = []
    if cfg.symmetry:
        pv = it.ev(("id", cfg.symmetry), root, None, {}, None, None)
        perms = [dict(f.items) for f in set_elems(pv)]

    def key(st):
        k = tuple(st[v] for v in variables)
        if not perms:
            return k
        # orbit representative: the permuted image with the smallest canonical text
        best, best_text = None, None
        for m in perms:
            kk = tuple(permute_value(x, m) for x in k)
            t = "|".join(fmt(x) for x in kk)
            if best_text is None or t < best_text:
                best, best_text = kk, t
        return best

    def in_model(st):
        return all(it.eval_named_predicate(c, st) for c in cfg.constraints)

    res = {
        "module": module, "distinct": 0, "generated": 0, "depth": 0, "levels": [],
        "deadlocks": 0, "out_of_model": 0, "violation": None, "complete": True,
        "first_violation_level": {inv: None for inv in cfg.invariants},
        "violating_states": {inv: 0 for inv in cfg.invariants},
    }
    seen: dict = {}            # state key -> parent key (None for init)
    frontier = []
    inits = it.init_states(init_e)
    res["generated"] += len(inits)

    def check_invariants(st, level, parent_key):
        for inv in cfg.invariants:
            if not it.eval_named_predicate(inv, st):
                res["violating_states"][inv] += 1
                if res["first_violation_level"][inv] is None:
                    res["first_violation_level"][inv] = level
                if res["violation"] is None:
                    res["violation"] = {"invariant": inv, "level": level, "state": state_text(variables, st),
                                        "key": key(st), "parent": parent_key}
                    if stop_on_violation:
                        return True
        return False

    stop = False
    for st in inits:
        kk = key(st)
        if not in_model(st):
            res["out_of_model"] += 1
            check_invariants(st, 1, None)
            continue
        if kk in seen:
            continue
        seen[kk] = None
        frontier.append(st)
        if check_invariants(st, 1, None):
            stop = True
            break
    level = 1
    while frontier and not stop:
        res["levels"].append(len(frontier))
        nxt_frontier = []
        for st in frontier:
            succs = it.next_states(next_e, st)
            res["generated"] += len(succs)
            if not succs:
                res["deadlocks"] += 1
                if cfg.check_deadlock and res["violation"] is None:
                    res["violation"] = {"invariant": "<deadlock>", "level": level,
                                        "state": state_text(variables, st), "key": key(st), "parent": seen[key(st)]}
                    if stop_on_violation:
                        stop = True
                        break
            pk = key(st)
            for s1 in succs:
                kk = key(s1)
                if not in_model(s1):
                    res["out_of_model"] += 1
                    if check_invariants(s1, level + 1, pk):
                        stop = True
                        break
                    continue
                if kk in seen:
                    continue
                seen[kk] = pk
                nxt_frontier.append(s1)
                if check_invariants(s1, level + 1, pk):
                    stop = True
                    break
            if stop:
                break
            if max_states is not None and len(seen) > max_states:
                res["complete"] = False
                stop = True
                break
        if not stop:
            frontier = nxt_frontier
            level += 1
    res["distinct"] = len(seen)
    res["depth"] = len(res["levels"])
    if res["violation"] is not None:
        # reconstruct the trace through parent links
        trace = []
        v = res["violation"]
        k = v["key"]
        chain = [k]
        p = v["parent"]
        while p is not None:
            chain.append(p)
            p = seen.get(p)
        for kk in reversed(chain):
            trace.append("\n".join(f"/\\ {n} = {fmt(x)}" for n, x in zip(variables, kk)))
        v["trace"] = trace
        del v["key"], v["parent"]
    if collect_states:
        res["states"] = sorted("\n".join(f"/\\ {n} = {fmt(x)}" for n, x in zip(variables, kk)) for kk in seen)
    return res


if __name__ == "__main__":
    import argparse
    import json
    import time

    ap = argparse.ArgumentParser(description="Oracle A: direct TLA+ interpreter BFS")
    ap.add_argument("module")
    ap.add_argument("-config", required=True)
    ap.add_argument("-I", action="append", default=[], help="module search directory")
    ap.add_argument("--max-states", type=int, default=None)
    ap.add_argument("--continue", dest="cont", action="store_true")
    a = ap.parse_args()
    here = os.path.dirname(os.path.abspath(__file__))
    dirs = a.I or [os.path.join(here, "_ref", "spec"), os.path.join(here, "..", "models")]
    t0 = time.time()
    with open(a.config) as f:
        r = run_bfs(a.module, dirs, f.read(), a.max_states, stop_on_violation=not a.cont)
    r["seconds"] = round(time.time() - t0, 3)
    print(json.dumps(r, indent=1))
