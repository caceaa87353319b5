"""Ahead-of-time lowering: TLA+ (``.tla`` + ``.cfg``) -> host/device C++ over packed states.

This is a partial evaluator.  It walks the spec exactly the way TLC's ``getNextStates`` does --
conjunct by conjunct, branching on every positive-position ``\\/`` and bounded ``\\E``, expanding
operator definitions and ``LET`` in place -- but with *symbolic* values (``svals.py``): whatever
depends only on the cfg constants is folded here, whatever depends on the state becomes a C
expression over the unpacked bit-fields.  Each complete branch becomes one guarded block that
packs and emits one successor, so the multiset of successors (TLC's "states generated") is
preserved, not just the set.

Two optimisations keep the emitted code small without changing that multiset:

* equality pinning: in ``\\E x \\in S : ... /\\ x = e /\\ ...`` (``e`` free of ``x``) the enumeration of
  ``S`` is replaced by ``x := e`` guarded by ``e \\in S``.  IdSequence.tla:30-33 (``id = nextId``),
  FiniteReplicatedLog.tla:99-101 (``offset = log.endOffset``) and :50-52
  (``log.records[offset] = record``) are all of this shape, which turns TLC's enumeration of the
  whole record universe (KafkaReplication.tla:82) into one array read;
* common-subexpression temporaries, scoped to the code block that computed them.
"""
from __future__ import annotations

import itertools

from ..frontend.cfg import Config, ModelValue
from ..frontend.modules import ModuleContext
from ..frontend.tla_parser import Def
from ..frontend.values import FnVal, fmt, sort_key
from . import layout as L
from .svals import (INT32_MAX, INT64_MAX, INT64_MIN, SYMBOLIC, LowerError, SAtom, SBool, SFn, SInt, SLazy, SRec, SSeq,
                    SSet, SUnion, c_int, fits_int, is_atom_const, is_const, is_int_const, is_static, kind_sig)

RANGE_ENUM_MAX = 1 << 16       # members of an `a .. b` that the lowering enumerates; a wider one stays a pair of bounds


def expr_text(e, depth: int = 0) -> str:
    """A short rendering of an expression for error messages."""
    if depth > 3:
        return "..."
    k = e[0]
    if k in ("num", "bool"):
        return str(e[1]).upper() if k == "bool" else str(e[1])
    if k == "str":
        return f'"{e[1]}"'
    if k == "id":
        return e[1]
    if k == "app":
        return f"{e[1]}(" + ", ".join(expr_text(x, depth + 1) for x in e[2]) + ")"
    if k == "binop":
        return f"{expr_text(e[2], depth + 1)} {e[1]} {expr_text(e[3], depth + 1)}"
    if k == "neg":
        return f"-{expr_text(e[1], depth + 1)}"
    if k == "prime":
        return f"{expr_text(e[1], depth + 1)}'"
    if k == "if":
        return f"IF {expr_text(e[1], depth + 1)} THEN {expr_text(e[2], depth + 1)} ELSE {expr_text(e[3], depth + 1)}"
    if k == "quant":
        return f"\\{e[1]} ... : {expr_text(e[3], depth + 1)}"
    if k == "subset":
        return f"SUBSET {expr_text(e[1], depth + 1)}"
    return f"<{k} expression>"


class UnpinnedRef(Exception):
    pass


class Marker:
    """A quantified variable that has not been given a value yet."""
    __slots__ = ("name", "domain", "value", "bound")

    def __init__(self, name, domain):
        self.name, self.domain = name, domain
        self.value, self.bound = None, False


class Thunk:
    __slots__ = ("expr", "ctx", "fm", "env", "val", "block", "done", "unit")

    def __init__(self, expr, ctx, fm, env):
        self.expr, self.ctx, self.fm, self.env = expr, ctx, fm, env
        self.val, self.block, self.done, self.unit = None, None, False, -1


class Closure:
    __slots__ = ("defn", "ctx", "fm", "env")

    def __init__(self, defn, ctx, fm, env):
        self.defn, self.ctx, self.fm, self.env = defn, ctx, fm, env


class Block:
    """A block of emitted C: its head (``if (...)``, or empty for a bare block), the condition the head tests and
    its children, which are statements (strings) and blocks.  A block with a ``label`` is a core: the bare block
    emit_successor() opens, which builds one successor and emits it with that action label (-1: the core only
    reports a layout trap), with no further branching on the state."""
    __slots__ = ("head", "cond", "label", "children")

    def __init__(self, head: str = "", cond: str | None = None, label: int | None = None, children=None):
        self.head, self.cond, self.label = head, cond, label
        self.children: list = [] if children is None else children


def render(nodes: list, depth: int) -> list[str]:
    """The C text of a tree: one statement, block head or closing brace per line, two spaces per level."""
    out = []
    for n in nodes:
        pad = "  " * depth
        if isinstance(n, Block):
            out.append(pad + (n.head + " {" if n.head else "{"))
            out.extend(render(n.children, depth + 1))
            out.append(pad + "}")
        else:
            out.append(pad + n)
    return out


class CG:
    """Structured C emitter with block-scoped temporaries; it builds the function body as a tree of Blocks.

    ``root`` is the block id of the function body; a fresh CG continuing the same function
    prologue (``fork``) keeps the root id and the prologue's CSE table, so that values computed in
    the prologue stay valid in every group function that replicates it."""
    _ids = itertools.count(1)

    def __init__(self, root: int | None = None, cse: dict | None = None, next_tmp: int = 0):
        self.body = Block()
        self.stack = [self.body]              # the open blocks, outermost first
        self.root = next(CG._ids) if root is None else root
        self.blocks = [self.root]             # their ids (the scopes of CSE hits)
        self.next_tmp = next_tmp
        self.cse: dict[tuple[str, str], tuple[str, int]] = dict(cse or {})

    def fork(self) -> "CG":
        return CG(self.root, {k: v for k, v in self.cse.items() if v[1] == self.root}, self.next_tmp)

    def pristine(self) -> bool:
        return not self.body.children and len(self.stack) == 1

    def emit(self, s: str):
        self.stack[-1].children.append(s)

    def open(self, head: str = "", cond: str | None = None, label: int | None = None) -> Block:
        b = Block(head, cond, label)
        self.stack[-1].children.append(b)
        self.stack.append(b)
        self.blocks.append(next(CG._ids))
        return b

    def close(self):
        self.stack.pop()
        self.blocks.pop()

    def tmp(self, ctype: str, expr: str) -> str:
        key = (ctype, expr)
        hit = self.cse.get(key)
        if hit is not None and hit[1] in self.blocks:
            return hit[0]
        name = f"t{self.next_tmp}"
        self.next_tmp += 1
        self.emit(f"const {ctype} {name} = {expr};")
        self.cse[key] = (name, self.blocks[-1])
        return name

    def mark(self):
        return (self.stack[-1], len(self.stack[-1].children), self.next_tmp, dict(self.cse))

    def rollback(self, m):
        if self.stack[-1] is not m[0]:
            raise LowerError("internal: unbalanced blocks")
        del m[0].children[m[1]:]
        self.next_tmp = m[2]
        self.cse = m[3]


class Lowerer:
    TMP_THRESHOLD = 40

    def __init__(self, root: ModuleContext, cfg: Config):
        self.root, self.cfg = root, cfg
        root.const_overrides = dict(cfg.overrides)
        self.variables = list(root.variables)
        self.const_values = dict(cfg.constants)
        for c in root.constants:
            if c not in self.const_values and c not in cfg.overrides:
                raise LowerError(f"constant {c} has no value in the cfg")
        self.gids: dict = {}
        self._intern_cfg_atoms()
        self.cg = CG()
        self.cur: dict | None = None          # var -> sval of the current state (None: constant context)
        self.read_cache: dict[int, object] = {}
        self.traps: list = []
        self.warnings: list[str] = []
        self._const_cache: dict = {}
        self._spec_thunks: list[Thunk] | None = None
        self.layout: L.Layout | None = None
        self.actions: list[dict] = []         # {"name", "module", "line", "col", ...}
        self.emit_sites = 0
        self.units: list[list] = []                    # trees of the independently compilable pieces
        self.unit_id = 0
        self.prologue: list[str] = []
        self.enc_cache: dict[int, tuple] = {}          # id(sval) -> (type sig, sval, code expr) for values decoded from a code
        self.mux_origin: dict[int, tuple] = {}         # id(sval) -> (sval, cond, a, b) for composite selects

    # ------------------------------------------------------------------ atoms
    def _intern_cfg_atoms(self):
        atoms = set()

        def walk(v):
            if isinstance(v, ModelValue):
                atoms.add(v)
            elif isinstance(v, frozenset):
                for x in v:
                    walk(x)
        for v in self.const_values.values():
            walk(v)
        for a in sorted(atoms, key=lambda m: m.name):
            self.gids[a] = len(self.gids)

    def gid(self, a) -> int:
        if a not in self.gids:
            self.gids[a] = len(self.gids)
        return self.gids[a]

    # ------------------------------------------------------------- C helpers
    def tmp_int(self, e: str, lo: int = 0, hi: int = 0) -> str:
        """``e`` (in a temporary when it is long) as a C integer that holds every value of [lo, hi]: an ``int`` where
        they fit one, else an ``int64_t``."""
        if len(e) <= self.TMP_THRESHOLD:
            return e
        return self.cg.tmp("int" if fits_int(lo, hi) else "int64_t", e)

    @staticmethod
    def int_ctype(lo: int, hi: int, what) -> str:
        """The C type of an integer expression with values in [lo, hi]; LowerError beyond 64-bit integers."""
        if lo < INT64_MIN or hi > INT64_MAX:
            raise LowerError(f"the integer expression {what() if callable(what) else what} takes values in {lo} .. {hi}, "
                             f"beyond 64-bit integers")
        return "int" if fits_int(lo, hi) else "int64_t"

    @staticmethod
    def wide(A) -> str:
        """The C text of the SInt A as a 64-bit operand, which makes a binary operation on it 64-bit (an SInt outside
        the range of ``int`` is 64-bit already)."""
        return f"(int64_t){A.s}" if fits_int(A.lo, A.hi) else A.s

    def tmp_code(self, ty, e: str) -> str:
        """A layout code of type ``ty``: an ``int``, or a ``uint64_t`` for a type with more codes than an ``int`` holds."""
        if ty.card - 1 <= INT32_MAX:
            return self.tmp_int(e)
        return self.cg.tmp("uint64_t", e) if len(e) > self.TMP_THRESHOLD else e

    def tmp_uint(self, e: str) -> str:
        return self.cg.tmp("unsigned", e) if len(e) > self.TMP_THRESHOLD else e

    def tmp_bool(self, e: str) -> str:
        return self.cg.tmp("bool", e) if len(e) > self.TMP_THRESHOLD else e

    @staticmethod
    def bstr(g) -> str:
        if g is True:
            return "true"
        if g is False:
            return "false"
        return g.s

    def b_and(self, xs):
        out, seen = [], set()
        for x in xs:
            if x is False:
                return False
            if x is True:
                continue
            if not isinstance(x, SBool):
                raise LowerError(f"expected a boolean, got {x!r}")
            if x.s not in seen:
                seen.add(x.s)
                out.append(x)
        if not out:
            return True
        if len(out) == 1:
            return out[0]
        return SBool(self.tmp_bool("(" + " && ".join(o.s for o in out) + ")"))

    def b_or(self, xs):
        out, seen = [], set()
        for x in xs:
            if x is True:
                return True
            if x is False:
                continue
            if not isinstance(x, SBool):
                raise LowerError(f"expected a boolean, got {x!r}")
            if x.s not in seen:
                seen.add(x.s)
                out.append(x)
        if not out:
            return False
        if len(out) == 1:
            return out[0]
        return SBool(self.tmp_bool("(" + " || ".join(o.s for o in out) + ")"))

    def b_not(self, x):
        if x is True:
            return False
        if x is False:
            return True
        if not isinstance(x, SBool):
            raise LowerError(f"expected a boolean, got {x!r}")
        if x.s.startswith("!") and x.s[1:].isidentifier():
            return SBool(x.s[1:])
        return SBool(f"!{x.s}" if x.s.isidentifier() else f"!({x.s})")

    def b_ite(self, c, a, b):
        if c is True:
            return a
        if c is False:
            return b
        if a is b or (isinstance(a, SBool) and isinstance(b, SBool) and a.s == b.s):
            return a
        if a is True:
            return self.b_or([c, b])
        if a is False:
            return self.b_and([self.b_not(c), b])
        if b is True:
            return self.b_or([self.b_not(c), a])
        if b is False:
            return self.b_and([c, a])
        return SBool(self.tmp_bool(f"({c.s} ? {a.s} : {b.s})"))

    def trap_unless(self, cond):
        self.traps.append(cond)

    # -- code cache: values that were decoded from a packed code can be re-encoded (and compared)
    #    by that code instead of field by field; a select between such values is a select of codes
    def remember_code(self, ty, v, code: str):
        if not is_const(v):
            self.enc_cache[id(v)] = (ty.sig(), v, code, self.cg.blocks[-1], self.unit_id)

    def _code_hit(self, v):
        hit = self.enc_cache.get(id(v))
        if hit is None or hit[1] is not v:
            return None
        # a code expression may name temporaries: it is only usable inside the block (and unit) that made it
        if hit[3] not in self.cg.blocks or not (hit[4] == self.unit_id or hit[4] == -2):
            return None
        return hit

    def encode(self, ty, v) -> str:
        """ty.enc(v), short-circuited through the code cache and through recorded selects."""
        if is_const(v):
            return ty.enc(self, v)
        hit = self._code_hit(v)
        if hit is not None and hit[0] == ty.sig():
            return hit[2]
        m = self.mux_origin.get(id(v))
        if m is not None and m[0] is v:
            _, c, a, b = m
            marks = len(self.traps)
            ea = self.encode(ty, a)
            eb = self.encode(ty, b)
            if len(self.traps) == marks:          # no range traps were needed for either branch
                code = self.tmp_code(ty, f"({c.s} ? {ea} : {eb})")
                self.remember_code(ty, v, code)
                return code
            del self.traps[marks:]
        return ty.enc(self, v)

    # ---------------------------------------------------------- value helpers
    def as_sint(self, v) -> SInt:
        if isinstance(v, SInt):
            return v
        if is_int_const(v):
            return SInt(c_int(v), v, v)
        raise LowerError(f"expected an integer, got {v!r}")

    def mk_int(self, s: str, lo: int, hi: int, what="an integer expression"):
        self.int_ctype(lo, hi, what)
        if lo == hi:
            return lo
        return SInt(self.tmp_int(s, lo, hi), lo, hi)

    def arith(self, op: str, A: SInt, B: SInt, what="an integer expression"):
        """A op B (op one of + - *) in the C type its operands and its result need: in ``int`` when all three fit one,
        else in ``int64_t``, so that no intermediate value wraps."""
        if op == "+":
            lo, hi = A.lo + B.lo, A.hi + B.hi
        elif op == "-":
            lo, hi = A.lo - B.hi, A.hi - B.lo
        else:
            c = [A.lo * B.lo, A.lo * B.hi, A.hi * B.lo, A.hi * B.hi]
            lo, hi = min(c), max(c)
        self.int_ctype(lo, hi, what)
        if fits_int(lo, hi) and fits_int(A.lo, A.hi) and fits_int(B.lo, B.hi):
            return self.mk_int(f"({A.s} {op} {B.s})", lo, hi, what)
        return self.mk_int(f"({self.wide(A)} {op} {B.s})", lo, hi, what)

    def atom_expr(self, v) -> str:
        if isinstance(v, SAtom):
            return v.s
        return str(self.gid(v))

    def cmp(self, op: str, a, b):
        if isinstance(a, SUnion) or isinstance(b, SUnion):
            a = self.narrow_union(a, "int") if isinstance(a, SUnion) else a
            b = self.narrow_union(b, "int") if isinstance(b, SUnion) else b
        A, B = self.as_sint(a), self.as_sint(b)
        if op == "<":
            if A.hi < B.lo:
                return True
            if A.lo >= B.hi:
                return False
        elif op == "<=":
            if A.hi <= B.lo:
                return True
            if A.lo > B.hi:
                return False
        elif op == ">":
            return self.cmp("<", b, a)
        elif op == ">=":
            return self.cmp("<=", b, a)
        elif op == "==":
            if A.lo == A.hi == B.lo == B.hi:
                return True
            if A.hi < B.lo or B.hi < A.lo:
                return False
            if A.s == B.s:
                return True
        return SBool(self.tmp_bool(f"({A.s} {op} {B.s})"))

    def alts(self, v):
        return v.alts if isinstance(v, SUnion) else [(True, v)]

    def narrow_union(self, v, kind: str):
        """The alternative(s) of ``v`` of the given kind (the others are assumed impossible;
        at a state write they are trapped)."""
        if not isinstance(v, SUnion):
            return v
        match = [(g, x) for g, x in v.alts if kind_sig(x) == kind]
        if not match:
            self.warnings.append(f"no alternative of kind {kind} in {v!r}")
            return self.poison(kind)
        res = match[-1][1]
        for g, x in reversed(match[:-1]):
            res = self.mux(g, x, res)
        return res

    def enc_union_into(self, ty, v: SUnion) -> str:
        k = ty.kind()
        bad = [g for g, x in v.alts if kind_sig(x) != k]
        if bad:
            self.trap_unless(self.b_not(self.b_or(bad)))
        return ty.enc(self, self.narrow_union(v, k))

    def poison(self, kind: str):
        if kind == "int":
            return 0
        if kind == "bool":
            return False
        if kind.startswith("rec:"):
            return SRec({f: 0 for f in kind[4:].split(",")})
        raise LowerError(f"cannot synthesise a placeholder of kind {kind}")

    def const_eq(self, a, b) -> bool:
        ka, kb = kind_sig(a), kind_sig(b)
        if ka != kb:
            if not (isinstance(a, ModelValue) or isinstance(b, ModelValue)):
                self.warnings.append(f"comparison of incomparable constants {fmt(a)} and {fmt(b)} folded to FALSE")
            return False
        return a == b

    def eq(self, a, b):
        if a is b:
            return True
        if is_const(a) and is_const(b):
            return self.const_eq(a, b)
        ca, cb = self._code_hit(a), self._code_hit(b)
        if ca is not None and cb is not None and ca[0] == cb[0]:
            # both were decoded from codes of the same (injective) layout type: compare the codes
            return True if ca[2] == cb[2] else SBool(self.tmp_bool(f"({ca[2]} == {cb[2]})"))
        if isinstance(a, SUnion) or isinstance(b, SUnion):
            terms = []
            for ga, xa in self.alts(a):
                for gb, xb in self.alts(b):
                    if kind_sig(xa) == kind_sig(xb):
                        terms.append(self.b_and([ga, gb, self.eq(xa, xb)]))
            return self.b_or(terms)
        ka, kb = kind_sig(a), kind_sig(b)
        if ka != kb:
            return False
        if ka == "int":
            return self.cmp("==", a, b)
        if ka == "bool":
            if isinstance(a, bool):
                return b if a else self.b_not(b)
            if isinstance(b, bool):
                return a if b else self.b_not(a)
            return SBool(self.tmp_bool(f"({a.s} == {b.s})"))
        if ka == "atom":
            if is_const(a):
                a, b = b, a
            if is_const(b):
                if b not in a.uni:
                    return False
                if len(a.uni) == 1:
                    return True
            elif not (set(a.uni) & set(b.uni)):
                return False
            ea, eb = self.atom_expr(a), self.atom_expr(b)
            return True if ea == eb else SBool(self.tmp_bool(f"({ea} == {eb})"))
        if ka.startswith("rec:"):
            fa, fb = self.rec_fields(a), self.rec_fields(b)
            return self.b_and([self.eq(fa[f], fb[f]) for f in fa])
        if ka == "fn":
            ma, mb = self.fn_map(a), self.fn_map(b)
            if set(ma) != set(mb):
                return False
            return self.b_and([self.eq(ma[k], mb[k]) for k in ma])
        if ka == "set":
            return self.b_and([self.subseteq(a, b), self.subseteq(b, a)])
        if ka == "tuple":
            return self.seq_eq(a, b)
        raise LowerError(f"cannot compare {a!r} and {b!r}")

    def rec_fields(self, v) -> dict:
        if isinstance(v, SRec):
            return v.fields
        if isinstance(v, FnVal):
            return dict(v.items)
        raise LowerError(f"not a record: {v!r}")

    def fn_map(self, v) -> dict:
        if isinstance(v, SFn):
            return dict(zip(v.keys, v.vals))
        if isinstance(v, FnVal):
            return dict(v.items)
        raise LowerError(f"not a function: {v!r}")

    # --------------------------------------------------------------- mux
    def mux(self, c, a, b):
        if c is True:
            return a
        if c is False:
            return b
        if a is b:
            return a
        if is_const(a) and is_const(b) and kind_sig(a) == kind_sig(b) and a == b:
            return a
        ka, kb = kind_sig(a), kind_sig(b)
        if ka == "union" or kb == "union" or ka != kb:
            res = self.union_merge(c, a, b)
            if not is_const(res):
                self.mux_origin[id(res)] = (res, c, a, b)
            return res
        if ka.startswith("rec:"):
            fa, fb = self.rec_fields(a), self.rec_fields(b)
            res = SRec({f: self.mux(c, fa[f], fb[f]) for f in fa})
            self.mux_origin[id(res)] = (res, c, a, b)
            return res
        if ka == "int":
            A, B = self.as_sint(a), self.as_sint(b)
            if A.s == B.s:
                return a
            lo, hi = min(A.lo, B.lo), max(A.hi, B.hi)
            return SInt(self.tmp_int(f"({c.s} ? {A.s} : {B.s})", lo, hi), lo, hi)
        if ka == "bool":
            return self.b_ite(c, a, b)
        if ka == "atom":
            ea, eb = self.atom_expr(a), self.atom_expr(b)
            ua = a.uni if isinstance(a, SAtom) else (a,)
            ub = b.uni if isinstance(b, SAtom) else (b,)
            uni = tuple(dict.fromkeys(list(ua) + list(ub)))
            if ea == eb:
                return a
            return SAtom(self.tmp_int(f"({c.s} ? {ea} : {eb})"), uni)
        if ka.startswith("rec:"):
            fa, fb = self.rec_fields(a), self.rec_fields(b)
            return SRec({f: self.mux(c, fa[f], fb[f]) for f in fa})
        if ka == "fn":
            ma, mb = self.fn_map(a), self.fn_map(b)
            if set(ma) != set(mb):
                raise LowerError("IF/function application mixes functions with different domains")
            keys = sorted(ma, key=sort_key)
            return SFn(keys, [self.mux(c, ma[k], mb[k]) for k in keys])
        if ka == "set":
            nc = self.b_not(c)
            return SSet([(self.b_and([c, g]), x) for g, x in self.set_items(a)] +
                        [(self.b_and([nc, g]), x) for g, x in self.set_items(b)])
        if ka == "tuple":
            return self.seq_mux(c, a, b)
        raise LowerError(f"cannot merge {a!r} and {b!r}")

    def union_merge(self, c, a, b):
        nc = self.b_not(c)
        by_kind: dict[str, list] = {}
        for g, x in self.alts(a):
            by_kind.setdefault(kind_sig(x), [None, None])[0] = (g, x)
        for g, x in self.alts(b):
            by_kind.setdefault(kind_sig(x), [None, None])[1] = (g, x)
        out = []
        for k, (pa, pb) in by_kind.items():
            if pa is not None and pb is not None:
                out.append((self.b_ite(c, pa[0], pb[0]), self.mux(c, pa[1], pb[1])))
            elif pa is not None:
                out.append((self.b_and([c, pa[0]]), pa[1]))
            else:
                out.append((self.b_and([nc, pb[0]]), pb[1]))
        out = [(g, x) for g, x in out if g is not False]
        if len(out) == 1 and out[0][0] is True:
            return out[0][1]
        return SUnion(out)

    # --------------------------------------------------------------- sets
    def set_items(self, s):
        if isinstance(s, frozenset):
            return [(True, x) for x in sorted(s, key=sort_key)]
        if isinstance(s, SSet):
            return s.items
        if isinstance(s, SLazy):
            return [(True, x) for x in self.enumerate_lazy(s)]
        if isinstance(s, SUnion):
            return self.set_items(self.narrow_union(s, "set"))
        raise LowerError(f"not a set: {s!r}")

    def enumerate_lazy(self, s: SLazy) -> list:
        if s.kind == "range":
            what = f"{s.a} .. {s.b}" if is_const(s.a) and is_const(s.b) else "a run-time range"
            raise LowerError(f"{what} may hold more than {RANGE_ENUM_MAX} integers: too many to enumerate "
                             f"(it can only be tested for membership)")
        if s.kind == "recset":
            names = list(s.a)
            cols = []
            for n in names:
                items = self.set_items(s.a[n])
                if any(g is not True or not is_const(x) for g, x in items):
                    raise LowerError("cannot enumerate a record set with state-dependent fields")
                cols.append([x for _, x in items])
            return [FnVal(dict(zip(names, combo))) for combo in itertools.product(*cols)]
        if s.kind == "powerset":
            items = self.set_items(s.a)
            if any(g is not True or not is_const(x) for g, x in items):
                raise LowerError("cannot enumerate SUBSET of a state-dependent set")
            elems = [x for _, x in items]
            return [frozenset(c) for r in range(len(elems) + 1) for c in itertools.combinations(elems, r)]
        if s.kind == "union":
            out, seen = [], set()
            for part in (s.a, s.b):
                for g, x in self.set_items(part):
                    if g is not True or not is_const(x):
                        raise LowerError("cannot enumerate a state-dependent union")
                    if x not in seen:
                        seen.add(x)
                        out.append(x)
            return out
        if s.kind == "fnset":
            dom = [x for _, x in self.set_items(s.a)]
            rng = [x for _, x in self.set_items(s.b)]
            if len(rng) ** len(dom) > 100000:
                raise LowerError("function set too large to enumerate")
            return [FnVal(dict(zip(dom, combo))) for combo in itertools.product(rng, repeat=len(dom))]
        if s.kind == "cross":
            cols = []
            for part in s.a:
                items = self.set_items(part)
                if any(g is not True or not is_const(x) for g, x in items):
                    raise LowerError("cannot enumerate a Cartesian product with state-dependent components")
                cols.append([x for _, x in items])
            return [tuple(combo) for combo in itertools.product(*cols)]
        raise LowerError(f"cannot enumerate {s!r}")

    def distinct_items(self, s):
        """set_items with every element guarded against an equal earlier element, so that an
        enumeration visits each member of the (runtime) set exactly once."""
        items = self.set_items(s)
        if isinstance(s, frozenset) or isinstance(s, SLazy) or (isinstance(s, SSet) and s.distinct):
            return items
        out = []
        for i, (g, x) in enumerate(items):
            dup = self.b_or([self.b_and([gj, self.eq(xj, x)]) for gj, xj in items[:i]])
            g2 = self.b_and([g, self.b_not(dup)])
            if g2 is not False:
                out.append((g2, x))
        return out

    def member(self, x, s):
        if isinstance(s, SUnion):
            s = self.narrow_union(s, "set")
        if isinstance(s, SLazy):
            return self.member_lazy(x, s)
        if isinstance(s, frozenset) and is_const(x):
            return x in s
        if isinstance(x, SUnion):
            return self.b_or([self.b_and([g, self.member(v, s)]) for g, v in x.alts])
        if isinstance(s, frozenset) and isinstance(x, SInt):
            ints = sorted(v for v in s if is_int_const(v))
            if ints and ints[-1] - ints[0] + 1 == len(ints):          # contiguous (the members are distinct)
                return self.b_and([self.cmp(">=", x, ints[0]), self.cmp("<=", x, ints[-1])])
            return self.b_or([self.cmp("==", x, v) for v in ints])
        return self.b_or([self.b_and([g, self.eq(x, e)]) for g, e in self.set_items(s)])

    def member_lazy(self, x, s: SLazy):
        if isinstance(x, SUnion):
            return self.b_or([self.b_and([g, self.member_lazy(v, s)]) for g, v in x.alts])
        k = kind_sig(x)
        if s.kind == "nat":
            return self.cmp(">=", x, 0) if k == "int" else False
        if s.kind == "range":
            return self.b_and([self.cmp(">=", x, s.a), self.cmp("<=", x, s.b)]) if k == "int" else False
        if s.kind == "int":
            return k == "int"
        if s.kind == "recset":
            if not k.startswith("rec:"):
                return False
            f = self.rec_fields(x)
            if set(f) != set(s.a):
                return False
            return self.b_and([self.member(f[n], s.a[n]) for n in s.a])
        if s.kind == "fnset":
            if k != "fn" and not k.startswith("rec:"):
                return False
            m = self.fn_map(x) if k == "fn" else self.rec_fields(x)
            dom = self.set_items(s.a)
            if any(g is not True or not is_const(e) for g, e in dom):
                raise LowerError("function set with state-dependent domain")
            if set(m) != {e for _, e in dom}:
                return False
            return self.b_and([self.member(v, s.b) for v in m.values()])
        if s.kind == "powerset":
            if k != "set":
                return False
            return self.b_and([self.b_or([self.b_not(g), self.member(e, s.a)]) for g, e in self.set_items(x)])
        if s.kind == "union":
            return self.b_or([self.member(x, s.a), self.member(x, s.b)])
        if s.kind == "seq":
            if k != "tuple":
                return False
            n, items = self.seq_parts(x)
            if is_int_const(n):
                return self.b_and([self.member(items[j], s.a) for j in range(n)])
            return self.b_and([self.b_or([self.cmp("<=", n, j), self.member(items[j], s.a)]) for j in range(len(items))])
        if s.kind == "cross":
            if k != "tuple":
                return False
            n, items = self.seq_parts(x)
            right_len = self.eq(n, len(s.a))
            if right_len is False or len(items) < len(s.a):
                return False
            return self.b_and([right_len] + [self.member(items[j], part) for j, part in enumerate(s.a)])
        raise LowerError(f"membership in {s!r}")

    def subseteq(self, a, b):
        return self.b_and([self.b_or([self.b_not(g), self.member(e, b)]) for g, e in self.set_items(a)])

    def interval(self, a, b):
        """a .. b: the set itself while it has at most RANGE_ENUM_MAX members, else its bounds (an SLazy "range"), which
        membership and layout types use as they are and which is refused where it would have to be enumerated."""
        if is_int_const(a) and is_int_const(b):
            if b - a + 1 > RANGE_ENUM_MAX:
                return SLazy("range", a, b)
            return frozenset(range(a, b + 1))
        A, B = self.as_sint(a), self.as_sint(b)
        if B.hi - A.lo + 1 > RANGE_ENUM_MAX:
            return SLazy("range", a, b)
        return SSet([(self.b_and([self.cmp("<=", a, k), self.cmp("<=", k, b)]), k) for k in range(A.lo, B.hi + 1)])

    # ------------------------------------------------------------ sequences / tuples (module Sequences)
    # A sequence is a Python tuple when every part of it is constant, else an SSeq: a length (int or SInt) and
    # cap item values of which the first `length` are meaningful.  Where TLC would report an error (Head / Tail of
    # the empty sequence, an index outside 1..Len) the lowered code computes an unspecified value of the right kind.
    def seq_parts(self, v):
        if isinstance(v, SUnion):
            v = self.narrow_union(v, "tuple")
        if isinstance(v, tuple):
            return len(v), list(v)
        if isinstance(v, SSeq):
            return v.n, v.items
        raise LowerError(f"not a sequence: {v!r}")

    def mk_seq(self, n, items):
        if is_int_const(n):
            if n < 0 or n > len(items):
                raise LowerError("internal: sequence length outside its items")
            items = list(items[:n])
            return tuple(items) if all(is_const(x) for x in items) else SSeq(n, items)
        if n.hi <= 0:
            return ()
        items = list(items[:n.hi])
        if len(items) < n.hi:
            raise LowerError("internal: sequence length bound exceeds its items")
        return SSeq(n, items)

    def int_add(self, a, k: int):
        if is_int_const(a):
            return a + k
        A = self.as_sint(a)
        return self.mk_int(f"({A.s} + {k})" if k >= 0 else f"({A.s} - {-k})", A.lo + k, A.hi + k)

    def seq_at(self, v, idx):
        n, items = self.seq_parts(v)
        if isinstance(idx, SUnion):
            idx = self.narrow_union(idx, "int")
        if is_int_const(idx):
            if not 1 <= idx <= len(items):
                raise LowerError(f"sequence index {idx} outside 1..{len(items)}")
            return items[idx - 1]
        if not items:
            raise LowerError("indexing a sequence that is always empty")
        return self.fn_apply(SFn(list(range(1, len(items) + 1)), items), idx)

    def seq_tail(self, v):
        n, items = self.seq_parts(v)
        if is_int_const(n):
            if n == 0:
                raise LowerError("Tail of the empty sequence")
            return self.mk_seq(n - 1, items[1:])
        A = self.as_sint(n)
        return self.mk_seq(self.mk_int(f"({A.s} - 1)", max(A.lo - 1, 0), A.hi - 1), items[1:])

    def seq_append(self, v, e):
        n, items = self.seq_parts(v)
        if is_int_const(n):
            return self.mk_seq(n + 1, list(items[:n]) + [e])
        new = []
        for j, old in enumerate(items):
            c = self.eq(n, j)
            new.append(old if c is False else self.mux(c, e, old))
        new.append(e)
        return self.mk_seq(self.int_add(n, 1), new)

    def seq_concat(self, a, b):
        na, ia = self.seq_parts(a)
        nb, ib = self.seq_parts(b)
        if is_int_const(na):
            return self.mk_seq(self.int_add(nb, na) if not is_int_const(nb) else na + nb, list(ia[:na]) + list(ib))
        A = self.as_sint(na)
        out = []
        for j in range(len(ia) + len(ib)):
            opts = []
            if j < len(ia):
                opts.append((self.cmp(">", na, j), ia[j]))
            for alen in range(A.lo, min(A.hi, j) + 1):
                if 0 <= j - alen < len(ib):
                    opts.append((self.eq(na, alen), ib[j - alen]))
            opts = [(c, x) for c, x in opts if c is not False]
            if not opts:
                break
            val = opts[-1][1]
            for c, x in reversed(opts[:-1]):
                val = self.mux(c, x, val)
            out.append(val)
        B = self.as_sint(nb)
        total = self.mk_int(f"({A.s} + {B.s})", A.lo + B.lo, min(A.hi + B.hi, len(out)))
        return self.mk_seq(total, out)

    def seq_subseq(self, v, m, k):
        n, items = self.seq_parts(v)
        if is_int_const(m) and is_int_const(k):
            if k < m:
                return ()
            if m < 1 or k > len(items):
                raise LowerError(f"SubSeq bounds {m}..{k} outside 1..{len(items)}")
            return self.mk_seq(k - m + 1, items[m - 1:k])
        M, K = self.as_sint(m), self.as_sint(k)
        hi = min(K.hi, len(items)) - M.lo + 1
        if hi <= 0:
            return ()
        out = [self.seq_at(v, self.int_add(m, j)) for j in range(hi) if M.lo + j <= len(items)]
        length = self.mk_int(f"(({K.s}) >= ({M.s}) ? ({K.s}) - ({M.s}) + 1 : 0)", max(0, K.lo - M.hi + 1), len(out))
        return self.mk_seq(length, out)

    def seq_domain(self, v):
        n, items = self.seq_parts(v)
        if is_int_const(n):
            return frozenset(range(1, n + 1))
        return SSet([(self.cmp("<=", j + 1, n), j + 1) for j in range(len(items))], distinct=True)

    def seq_eq(self, a, b):
        na, ia = self.seq_parts(a)
        nb, ib = self.seq_parts(b)
        same_len = self.eq(na, nb)
        if same_len is False:
            return False
        terms = [same_len]
        for j in range(min(len(ia), len(ib))):
            if is_int_const(na) and j >= na or is_int_const(nb) and j >= nb:
                break
            beyond = False if is_int_const(na) else self.cmp("<=", na, j)
            terms.append(self.b_or([beyond, self.eq(ia[j], ib[j])]))
        return self.b_and(terms)

    def seq_mux(self, c, a, b):
        na, ia = self.seq_parts(a)
        nb, ib = self.seq_parts(b)
        n = self.mux(c, na, nb)
        items = []
        for j in range(max(len(ia), len(ib))):
            if j >= len(ia):
                items.append(ib[j])
            elif j >= len(ib):
                items.append(ia[j])
            else:
                items.append(self.mux(c, ia[j], ib[j]))
        return self.mk_seq(n, items)

    def seq_except(self, v, idx, leaf):
        """[v EXCEPT ![idx] = leaf(old item)]"""
        n, items = self.seq_parts(v)
        new = []
        for j, old in enumerate(items):
            c = self.eq(idx, j + 1)
            new.append(old if c is False else self.mux(c, leaf(old), old))
        return self.mk_seq(n, new)

    SEQ_BUILTINS = {"Len": 1, "Head": 1, "Tail": 1, "Append": 2, "SubSeq": 3, "Seq": 1}

    def seq_builtin(self, name, args):
        if name == "Seq":
            return SLazy("seq", args[0])
        if name == "Len":
            return self.seq_parts(args[0])[0]
        if name == "Head":
            return self.seq_at(args[0], 1)
        if name == "Tail":
            return self.seq_tail(args[0])
        if name == "Append":
            return self.seq_append(args[0], args[1])
        return self.seq_subseq(args[0], args[1], args[2])

    # ------------------------------------------------------------ evaluation
    def force(self, t: Thunk):
        if t.done and (is_static(t.val) or (t.block in self.cg.blocks and (t.unit == self.unit_id or t.block == self.cg.root and t.unit == -2))):
            return t.val
        v = self.ev(t.expr, t.ctx, t.fm, t.env)
        t.val, t.block, t.done, t.unit = v, self.cg.blocks[-1], True, self.unit_id
        if self._spec_thunks is not None:
            self._spec_thunks.append(t)
        return v

    def lookup(self, name, ctx, fm, env, S):
        if name in env:
            v = env[name]
            if isinstance(v, Thunk):
                return self.force(v)
            if isinstance(v, Marker):
                if not v.bound:
                    raise UnpinnedRef(v.name)
                return v.value
            return v
        r = ctx.resolve(name, fm)
        if r is None:
            if name == "Nat":
                return SLazy("nat")
            if name == "Int":
                return SLazy("int")
            if name == "BOOLEAN":
                return frozenset({True, False})
            raise LowerError(f"unknown identifier {name} (module {ctx.path})")
        if r.kind == "const":
            return self.const_values[name]
        if r.kind == "var":
            if S is None:
                raise LowerError(f"state variable {name} read in a constant context")
            if name not in S:
                raise LowerError(f"variable {name}' read before it is assigned")
            return S[name]
        if r.kind == "subst":
            return self.ev(r.expr, r.ctx, r.from_module, {}, S)
        if r.kind == "def":
            d = r.defn
            if d.params:
                raise LowerError(f"operator {name} used without arguments")
            return self.eval_nullary(d, r.ctx, S)
        raise LowerError(f"{name} is a module instance, not a value")

    def eval_nullary(self, d: Def, dctx, S):
        key = (id(dctx), d.module, d.name)
        if key in self._const_cache:
            return self._const_cache[key]
        v = self.ev(d.body, dctx, d.module, {}, S)
        if is_static(v):
            self._const_cache[key] = v
        return v

    def resolve_var(self, e, ctx, fm, env):
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
        k = e[0]
        if k == "inst":
            r = ctx.resolve(e[1], fm)
            if r is None or r.kind != "inst":
                raise LowerError(f"{e[1]} is not a module instance")
            d = r.inst.find_def(e[2], None)
            if d is None or d.local:
                raise LowerError(f"{e[1]}!{e[2]} is not an exported definition")
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
        if isinstance(target, Closure):
            d = target.defn
            if len(d.params) != len(args):
                raise LowerError(f"arity mismatch calling {d.name}")
            new_env = dict(target.env)
            for p, a in zip(d.params, args):
                new_env[p] = Thunk(a, ctx, fm, env)
            return d.body, target.ctx, target.fm, new_env
        d = target
        if len(d.params) != len(args):
            raise LowerError(f"arity mismatch calling {d.name}")
        return d.body, defctx, d.module, {p: Thunk(a, ctx, fm, env) for p, a in zip(d.params, args)}

    def let_env(self, defs, ctx, fm, env):
        env2 = dict(env)
        for d in defs:
            env2[d.name] = Closure(d, ctx, fm, env2) if d.params else Thunk(d.body, ctx, fm, env2)
        return env2

    _USE_CUR = object()

    def ev(self, e, ctx, fm, env, S=_USE_CUR):
        if S is Lowerer._USE_CUR:
            S = self.cur
        k = e[0]
        if k in ("num", "str", "bool"):
            if k == "str":
                self.gid(e[1])
            return e[1]
        if k == "id":
            return self.lookup(e[1], ctx, fm, env, S)
        if k in ("app", "inst"):
            op = self.find_operator(e, ctx, fm, env)
            if op is None:
                if k == "app" and e[1] == "Cardinality" and len(e[2]) == 1:
                    # FiniteSets: number of distinct present elements = sum of the (de-duplicated) guards
                    sv = self.ev(e[2][0], ctx, fm, env, S)
                    if isinstance(sv, frozenset):
                        return len(sv)
                    if isinstance(sv, SLazy) and sv.kind == "range" and is_const(sv.a) and is_const(sv.b):
                        return max(0, sv.b - sv.a + 1)
                    items = self.distinct_items(sv)
                    fixed = sum(1 for g, _ in items if g is True)
                    dyn = [g for g, _ in items if g is not True]
                    if not dyn:
                        return fixed
                    terms = ([str(fixed)] if fixed else []) + [f"(int){g.s}" for g in dyn]
                    return SInt(self.tmp_int("(" + " + ".join(terms) + ")"), fixed, fixed + len(dyn))
                if k == "app" and e[1] == "Permutations" and len(e[2]) == 1:
                    # TLC module: all permutations of a constant finite set (used by SYMMETRY)
                    base = self.ev(e[2][0], ctx, fm, env, S)
                    if not isinstance(base, frozenset):
                        raise LowerError("Permutations of a non-constant set")
                    elems = sorted(base, key=sort_key)
                    return frozenset(FnVal(dict(zip(elems, p))) for p in itertools.permutations(elems))
                if k == "app" and self.SEQ_BUILTINS.get(e[1]) == len(e[2]):
                    return self.seq_builtin(e[1], [self.ev(x, ctx, fm, env, S) for x in e[2]])
                raise LowerError(f"unknown operator {e[1]}")
            target, defctx, args = op
            if not isinstance(target, Closure) and not target.params:
                return self.eval_nullary(target, defctx, S)
            body, c2, fm2, env2 = self.bind_call(target, defctx, args, ctx, fm, env)
            return self.ev(body, c2, fm2, env2, S)
        if k == "and":
            return self.b_and([self.ev_bool(x, ctx, fm, env, S) for x in e[1]])
        if k == "or":
            return self.b_or([self.ev_bool(x, ctx, fm, env, S) for x in e[1]])
        if k == "not":
            return self.b_not(self.ev_bool(e[1], ctx, fm, env, S))
        if k == "neg":
            v = self.ev(e[1], ctx, fm, env, S)
            if is_int_const(v):
                return -v
            A = self.as_sint(v)
            what = lambda: expr_text(e)
            self.int_ctype(-A.hi, -A.lo, what)
            return self.mk_int(f"(-{A.s})" if fits_int(A.lo, A.hi) and fits_int(-A.hi, -A.lo) else f"(-{self.wide(A)})",
                               -A.hi, -A.lo, what)
        if k == "binop":
            return self.ev_binop(e, ctx, fm, env, S)
        if k == "if":
            c = self.ev_bool(e[1], ctx, fm, env, S)
            if c is True:
                return self.ev(e[2], ctx, fm, env, S)
            if c is False:
                return self.ev(e[3], ctx, fm, env, S)
            return self.mux(c, self.ev(e[2], ctx, fm, env, S), self.ev(e[3], ctx, fm, env, S))
        if k == "let":
            return self.ev(e[2], ctx, fm, self.let_env(e[1], ctx, fm, env), S)
        if k == "case":
            # CASE p1 -> e1 [] ... [] OTHER -> e: a select chain (the first true guard wins, like TLC)
            if e[2] is not None:
                res = self.ev(e[2], ctx, fm, env, S)
                arms = e[1]
            else:
                res = self.ev(e[1][-1][1], ctx, fm, env, S)      # no OTHER: the last arm is the fall-through
                arms = e[1][:-1]
            for g, x in reversed(arms):
                c = self.ev_bool(g, ctx, fm, env, S)
                if c is True:
                    res = self.ev(x, ctx, fm, env, S)
                elif c is not False:
                    res = self.mux(c, self.ev(x, ctx, fm, env, S), res)
            return res
        if k == "quant":
            if e[1] == "E":
                return self.exists_bool(e[2], e[3], ctx, fm, env, S)
            terms = []
            for guard, env2 in self.bindings(e[2], ctx, fm, env, S):
                terms.append(self.b_or([self.b_not(guard), self.ev_bool(e[3], ctx, fm, env2, S)]))
            return self.b_and(terms)
        if k == "choose":
            items = self.set_items(self.ev(e[2], ctx, fm, env, S))
            cands = []
            for g, x in items:
                env2 = dict(env)
                env2[e[1]] = x
                cands.append((self.b_and([g, self.ev_bool(e[3], ctx, fm, env2, S)]), x))
            cands = [(c, x) for c, x in cands if c is not False]
            if not cands:
                raise LowerError("CHOOSE over a statically empty candidate set")
            res = cands[-1][1]
            for c, x in reversed(cands[:-1]):
                res = self.mux(c, x, res)
            return res
        if k == "setenum":
            vals = [self.ev(x, ctx, fm, env, S) for x in e[1]]
            if all(is_const(v) for v in vals):
                return frozenset(vals)
            return SSet([(True, v) for v in vals])
        if k == "setmap":
            items = [(g, self.ev(e[1], ctx, fm, env2, S)) for g, env2 in self.bindings(e[2], ctx, fm, env, S)]
            if all(g is True and is_const(x) for g, x in items):
                return frozenset(x for _, x in items)
            return SSet(items)
        if k == "setfilter":
            items = []
            src_set = self.ev(e[2], ctx, fm, env, S)
            for g, x in self.set_items(src_set):
                env2 = dict(env)
                env2[e[1]] = x
                items.append((self.b_and([g, self.ev_bool(e[3], ctx, fm, env2, S)]), x))
            items = [(g, x) for g, x in items if g is not False]
            if all(g is True and is_const(x) for g, x in items):
                return frozenset(x for _, x in items)
            return SSet(items, distinct=isinstance(src_set, (frozenset, SLazy)) or getattr(src_set, "distinct", False))
        if k == "subset":
            return SLazy("powerset", self.ev(e[1], ctx, fm, env, S))
        if k == "domain":
            f = self.ev(e[1], ctx, fm, env, S)
            if not isinstance(f, SUnion) and kind_sig(f) == "tuple":
                return self.seq_domain(f)
            return frozenset(self.fn_map(f))
        if k == "fnlit":
            keys, vals = [], []
            for g, env2, key in self.bindings(e[1], ctx, fm, env, S, with_key=True):
                if g is not True:
                    raise LowerError("function constructor over a state-dependent domain")
                keys.append(key)
                vals.append(self.ev(e[2], ctx, fm, env2, S))
            if all(is_const(v) for v in vals):
                return FnVal(dict(zip(keys, vals)))
            return SFn(keys, vals)
        if k == "fnapp":
            f = self.ev(e[1], ctx, fm, env, S)
            args = [self.ev(a, ctx, fm, env, S) for a in e[2]]
            if len(args) != 1:
                raise LowerError("multi-argument function application is not supported")
            if not isinstance(f, SUnion) and kind_sig(f) == "tuple":
                return self.seq_at(f, args[0])
            return self.fn_apply(f, args[0])
        if k == "fnset":
            return SLazy("fnset", self.ev(e[1], ctx, fm, env, S), self.ev(e[2], ctx, fm, env, S))
        if k == "rec":
            fields = {f: self.ev(x, ctx, fm, env, S) for f, x in e[1]}
            if all(is_const(v) for v in fields.values()):
                return FnVal(fields)
            return SRec(fields)
        if k == "recset":
            return SLazy("recset", {f: self.ev(x, ctx, fm, env, S) for f, x in e[1]})
        if k == "dot":
            return self.dot(self.ev(e[1], ctx, fm, env, S), e[2])
        if k == "except":
            f = self.ev(e[1], ctx, fm, env, S)
            for path, rhs in e[2]:
                f = self.except_update(f, path, rhs, ctx, fm, env, S)
            return f
        if k == "at":
            return env["@"]
        if k == "tuple":
            items = [self.ev(x, ctx, fm, env, S) for x in e[1]]
            return self.mk_seq(len(items), items)
        if k == "cross":
            parts = [self.ev(x, ctx, fm, env, S) for x in e[1]]
            if all(isinstance(p, frozenset) for p in parts):
                return frozenset(tuple(c) for c in itertools.product(*[sorted(p, key=sort_key) for p in parts]))
            return SLazy("cross", parts)
        if k == "prime":
            st1 = env.get("'")
            if st1 is None:
                raise LowerError("primed expression outside an action")
            return self.ev(e[1], ctx, fm, env, st1)
        if k == "unchanged":
            st1 = env.get("'")
            if st1 is None:
                raise LowerError("UNCHANGED outside an action")
            return self.b_and([self.eq(st1[v], self.cur[v]) for v in self.unchanged_vars(e[1], ctx, fm, env)])
        raise LowerError(f"cannot lower node kind {k}")

    def ev_bool(self, e, ctx, fm, env, S=_USE_CUR):
        v = self.ev(e, ctx, fm, env, S)
        if isinstance(v, SUnion):
            v = self.narrow_union(v, "bool")
        if not isinstance(v, (bool, SBool)):
            raise LowerError(f"expected a boolean, got {v!r}")
        return v

    def ev_binop(self, e, ctx, fm, env, S):
        op = e[1]
        if op == "=>":
            return self.b_or([self.b_not(self.ev_bool(e[2], ctx, fm, env, S)), self.ev_bool(e[3], ctx, fm, env, S)])
        a = self.ev(e[2], ctx, fm, env, S)
        b = self.ev(e[3], ctx, fm, env, S)
        if op == "=":
            return self.eq(a, b)
        if op == "#":
            return self.b_not(self.eq(a, b))
        if op in ("<", ">", "<=", ">="):
            return self.cmp(op, a, b)
        if op in ("+", "-", "*"):
            if is_int_const(a) and is_int_const(b):
                return a + b if op == "+" else a - b if op == "-" else a * b
            if isinstance(a, SUnion):
                a = self.narrow_union(a, "int")
            if isinstance(b, SUnion):
                b = self.narrow_union(b, "int")
            return self.arith(op, self.as_sint(a), self.as_sint(b), lambda: expr_text(e))
        if op in ("\\div", "%"):
            # Integers: floor division and the modulus with a positive divisor (TLA+ defines a % b only for b > 0)
            if isinstance(a, SUnion):
                a = self.narrow_union(a, "int")
            if isinstance(b, SUnion):
                b = self.narrow_union(b, "int")
            if is_int_const(a) and is_int_const(b):
                if b <= 0:
                    raise LowerError(f"{op} with the non-positive divisor {b}")
                return a // b if op == "\\div" else a % b
            A, B = self.as_sint(a), self.as_sint(b)
            if B.lo <= 0:
                raise LowerError(f"{op}: the divisor may be non-positive ({B.lo}..{B.hi})")
            what = lambda: expr_text(e)
            # with a negative dividend, C's truncating / and % are corrected through -a + b - 1 (\div) or (a % b) + b (%):
            # the C type is chosen from the operands, those intermediate values and the result
            if op == "\\div":
                c = [A.lo // B.lo, A.lo // B.hi, A.hi // B.lo, A.hi // B.hi]
                lo, hi = min(c), max(c)
                mid = (0, 0) if A.lo >= 0 else (max(1, -A.hi) + B.lo - 1, -A.lo + B.hi - 1)
            else:
                lo, hi = 0, min(B.hi - 1, A.hi) if A.lo >= 0 else B.hi - 1
                mid = (0, 0) if A.lo >= 0 else (B.lo - B.hi + 1, 2 * B.hi - 1)
            self.int_ctype(*mid, what)
            narrow = all(fits_int(*r) for r in ((A.lo, A.hi), (B.lo, B.hi), mid, (lo, hi)))
            sa, sb = (A.s, B.s) if narrow else (self.wide(A), B.s)
            if op == "\\div":
                code = f"({sa} / {sb})" if A.lo >= 0 else f"(({sa}) >= 0 ? ({sa}) / ({sb}) : -((-({sa}) + ({sb}) - 1) / ({sb})))"
            else:
                code = f"({sa} % {sb})" if A.lo >= 0 else f"(((({sa}) % ({sb})) + ({sb})) % ({sb}))"
            return self.mk_int(code, lo, hi, what)
        if op == "..":
            return self.interval(a, b)
        if op == "\\o":
            return self.seq_concat(a, b)
        if op == "\\in":
            return self.member(a, b)
        if op == "\\notin":
            return self.b_not(self.member(a, b))
        if op == "\\subseteq":
            return self.subseteq(a, b)
        if op == "\\union":
            if isinstance(a, frozenset) and isinstance(b, frozenset):
                return a | b
            if isinstance(a, SLazy) or isinstance(b, SLazy):
                return SLazy("union", a, b)
            return SSet(list(self.set_items(a)) + list(self.set_items(b)))
        if op == "\\intersect":
            if isinstance(a, frozenset) and isinstance(b, frozenset):
                return a & b
            return SSet([(self.b_and([g, self.member(x, b)]), x) for g, x in self.set_items(a)],
                        distinct=isinstance(a, (frozenset, SLazy)) or getattr(a, "distinct", False))
        if op == "\\":
            if isinstance(a, SLazy) and isinstance(b, frozenset) and a.kind in ("powerset", "recset", "union"):
                try:
                    a = frozenset(self.enumerate_lazy(a))          # e.g. (SUBSET Replicas) \\ {{}} in a type expression
                except LowerError:
                    pass
            if isinstance(a, frozenset) and isinstance(b, frozenset):
                return a - b
            return SSet([(self.b_and([g, self.b_not(self.member(x, b))]), x) for g, x in self.set_items(a)],
                        distinct=isinstance(a, (frozenset, SLazy)) or getattr(a, "distinct", False))
        if op == "<=>":
            return self.eq(self.ev_bool(e[2], ctx, fm, env, S), self.ev_bool(e[3], ctx, fm, env, S))
        raise LowerError(f"unsupported operator {op}")

    def dot(self, r, field: str):
        if isinstance(r, FnVal):
            return r.apply(field)
        if isinstance(r, SRec):
            if field not in r.fields:
                raise LowerError(f"record has no field {field}")
            return r.fields[field]
        if isinstance(r, SUnion):
            match = [(g, x) for g, x in r.alts if kind_sig(x).startswith("rec:") and field in self.rec_fields(x)]
            if not match:
                self.warnings.append(f".{field} applied to a value with no record alternative")
                return 0
            res = self.dot(match[-1][1], field)
            for g, x in reversed(match[:-1]):
                res = self.mux(g, self.dot(x, field), res)
            return res
        raise LowerError(f".{field} applied to non-record {r!r}")

    def fn_apply(self, f, idx):
        if isinstance(f, SUnion):
            f = self.narrow_union(f, "fn")
        m = self.fn_map(f)
        if is_const(idx):
            if idx not in m:
                raise LowerError(f"function applied outside its domain: {fmt(idx)}")
            return m[idx]
        keys = sorted(m, key=sort_key)
        # candidates the index can actually take
        if isinstance(idx, SInt):
            keys = [k for k in keys if is_int_const(k) and idx.lo <= k <= idx.hi]
        elif isinstance(idx, SAtom):
            keys = [k for k in keys if k in idx.uni]
        if not keys:
            self.warnings.append("function application with an index that is never in the domain")
            keys = sorted(m, key=sort_key)[:1]
        res = m[keys[-1]]
        for k in reversed(keys[:-1]):
            res = self.mux(self.eq(idx, k), m[k], res)
        return res

    def except_update(self, f, path, rhs, ctx, fm, env, S):
        step = path[0]
        if step[0] == "fld":
            fields = dict(self.rec_fields(f))
            key = step[1]
            if key not in fields:
                raise LowerError(f"EXCEPT on missing field {key}")
            fields[key] = self.except_leaf(fields[key], path, rhs, ctx, fm, env, S)
            return FnVal(fields) if all(is_const(v) for v in fields.values()) else SRec(fields)
        idx = self.ev(step[1], ctx, fm, env, S)
        if not isinstance(f, SUnion) and kind_sig(f) == "tuple":
            return self.seq_except(f, idx, lambda old: self.except_leaf(old, path, rhs, ctx, fm, env, S))
        m = self.fn_map(f)
        keys = list(f.keys) if isinstance(f, SFn) else [k for k, _ in f.items]
        if is_const(idx):
            if idx not in m:
                raise LowerError(f"EXCEPT on key {fmt(idx)} outside the domain")
            vals = [self.except_leaf(m[k], path, rhs, ctx, fm, env, S) if k == idx else m[k] for k in keys]
        else:
            vals = []
            for k in keys:
                c = self.eq(idx, k)
                vals.append(m[k] if c is False else self.mux(c, self.except_leaf(m[k], path, rhs, ctx, fm, env, S), m[k]))
        if all(is_const(v) for v in vals):
            return FnVal(dict(zip(keys, vals)))
        return SFn(keys, vals)

    def except_leaf(self, old, path, rhs, ctx, fm, env, S):
        if len(path) == 1:
            env2 = dict(env)
            env2["@"] = old
            return self.ev(rhs, ctx, fm, env2, S)
        return self.except_update(old, path[1:], rhs, ctx, fm, env, S)

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
        raise LowerError(f"UNCHANGED of a non-variable expression {e!r}")

    # ------------------------------------------------------------ quantifiers
    def bindings(self, bounds, ctx, fm, env, S, with_key=False):
        """All (guard, env) bindings of a bounded quantifier, by enumeration."""
        names, cols = [], []
        for ns, sexpr in bounds:
            items = self.set_items(self.ev(sexpr, ctx, fm, env, S))
            for n in ns:
                names.append(n)
                cols.append(items)
        out = []
        for combo in itertools.product(*cols):
            env2 = dict(env)
            guards = []
            for n, (g, x) in zip(names, combo):
                env2[n] = x
                guards.append(g)
            guard = self.b_and(guards)
            if guard is False:
                continue
            if with_key:
                key = combo[0][1] if len(combo) == 1 else tuple(x for _, x in combo)
                out.append((guard, env2, key))
            else:
                out.append((guard, env2))
        return out

    def flatten(self, item):
        """Conjuncts reachable without branching (expands /\\, LET and operator applications)."""
        out, work = [], [item]
        while work:
            e, ctx, fm, env = work.pop(0)
            k = e[0]
            if k == "and":
                work = [(x, ctx, fm, env) for x in e[1]] + work
            elif k == "let":
                work.insert(0, (e[2], ctx, fm, self.let_env(e[1], ctx, fm, env)))
            elif k in ("id", "app", "inst"):
                op = None
                if not (k == "id" and e[1] in env and not isinstance(env[e[1]], Closure)):
                    try:
                        op = self.find_operator(e, ctx, fm, env)
                    except LowerError:
                        op = None
                if op is not None:
                    target, defctx, args = op
                    work.insert(0, self.bind_call(target, defctx, args, ctx, fm, env))
                else:
                    out.append((e, ctx, fm, env))
            else:
                out.append((e, ctx, fm, env))
        return out

    def peek_marker(self, e, env):
        while e[0] == "id" and e[1] in env:
            v = env[e[1]]
            if isinstance(v, Marker):
                return v if not v.bound else None
            if isinstance(v, Thunk) and not v.done:
                e, env = v.expr, v.env
                continue
            return None
        return None

    def speculate(self, fn):
        """Run fn(); on UnpinnedRef undo every emitted line / memoised thunk and return None."""
        mark = self.cg.mark()
        saved, self._spec_thunks = self._spec_thunks, []
        try:
            return fn()
        except UnpinnedRef:
            self.cg.rollback(mark)
            for t in self._spec_thunks:
                t.done, t.val = False, None
            return None
        finally:
            forced = self._spec_thunks
            self._spec_thunks = saved
            if saved is not None:
                saved.extend(forced)

    def try_pin(self, markers, body_item, S):
        """Pin as many markers as possible through ``x = e`` conjuncts; returns membership guards."""
        guards = []
        progress = True
        while progress and any(not m.bound for m in markers):
            progress = False
            for (e, ctx, fm, env) in self.flatten(body_item):
                if e[0] != "binop" or e[1] != "=":
                    continue
                for lhs, rhs in ((e[2], e[3]), (e[3], e[2])):
                    m = self.peek_marker(lhs, env)
                    if m is None or m not in markers:
                        continue
                    val = self.speculate(lambda: (self.ev(rhs, ctx, fm, env, S),))
                    if val is None:
                        continue
                    m.value, m.bound = val[0], True
                    guards.append(self.member(val[0], m.domain))
                    progress = True
                    break
                if progress:
                    break
        return guards

    def exists_each(self, bounds, body, ctx, fm, env, S, k, split=False):
        """Calls k(guard, env2) for every binding of ``\\E bounds : body`` (pinned or enumerated)."""
        markers = []
        env2 = dict(env)
        for ns, sexpr in bounds:
            dom = self.ev(sexpr, ctx, fm, env, S)
            for n in ns:
                m = Marker(n, dom)
                env2[n] = m
                markers.append(m)
        body_item = (body, ctx, fm, env2)

        def rec(guards):
            mine = [m for m in markers if not m.bound]
            pinned_guards = self.try_pin(markers, body_item, S)
            newly = [m for m in mine if m.bound]
            g_all = guards + pinned_guards
            if self.b_and(g_all) is not False:
                rest = [m for m in markers if not m.bound]
                if not rest:
                    k(self.b_and(g_all), env2)
                else:
                    m = rest[0]
                    for g, x in self.distinct_items(m.domain):
                        # in action context an unconditional binding reached before any code was
                        # emitted is a point where expand() can be cut into separate functions
                        cut = split and g is True and self.b_and(g_all) is True and self.cg.pristine()
                        m.value, m.bound = x, True
                        rec(g_all + [g])
                        m.bound, m.value = False, None
                        if cut:
                            self.end_unit()
            for m in newly:
                m.bound, m.value = False, None

        rec([])

    def exists_bool(self, bounds, body, ctx, fm, env, S):
        terms = []

        def k(guard, env2):
            # freeze marker values into a plain env (markers are reset after the callback)
            env3 = {n: (v.value if isinstance(v, Marker) else v) for n, v in env2.items()}
            terms.append(self.b_and([guard, self.ev_bool(body, ctx, fm, env3, S)]))

        self.exists_each(bounds, body, ctx, fm, env, S, k)
        return self.b_or(terms)

    # --------------------------------------------------------------- actions
    def gen_next(self, items, st1: dict, label):
        """Emit code for the conjunct list ``items`` (TLC getNextStates order)."""
        if not items:
            self.emit_successor(st1, label)
            return
        (e, ctx, fm, env), rest = items[0], items[1:]
        k = e[0]
        if k == "and":
            self.gen_next([(x, ctx, fm, env) for x in e[1]] + rest, st1, label)
            return
        if k == "or":
            split = self.cg.pristine()
            for x in e[1]:
                if split:
                    self.gen_next([(x, ctx, fm, env)] + rest, st1, label)
                    self.end_unit()
                else:
                    self.cg.open()
                    self.gen_next([(x, ctx, fm, env)] + rest, st1, label)
                    self.cg.close()
            return
        if k == "quant" and e[1] == "E":
            def kont(guard, env2):
                env3 = {n: (v.value if isinstance(v, Marker) else v) for n, v in env2.items()}
                split = guard is True and self.cg.pristine()
                self.guarded(guard, lambda: self.gen_next([(e[3], ctx, fm, env3)] + rest, st1, label))
                if split:
                    self.end_unit()
            self.exists_each(e[2], e[3], ctx, fm, env, self.cur, kont, split=True)
            return
        if k == "let":
            self.gen_next([(e[2], ctx, fm, self.let_env(e[1], ctx, fm, env))] + rest, st1, label)
            return
        if k == "if":
            c = self.ev_bool(e[1], ctx, fm, self.with_next(env, st1))
            if c is not False:
                self.guarded(c, lambda: self.gen_next([(e[2], ctx, fm, env)] + rest, st1, label))
            if c is not True:
                self.guarded(self.b_not(c), lambda: self.gen_next([(e[3], ctx, fm, env)] + rest, st1, label))
            return
        if k in ("id", "app", "inst"):
            op = None
            if not (k == "id" and e[1] in env and not isinstance(env[e[1]], Closure)):
                op = self.find_operator(e, ctx, fm, env)
            if op is not None:
                target, defctx, args = op
                if label is None and not isinstance(target, Closure):
                    label = self.action_id(target)
                self.gen_next([self.bind_call(target, defctx, args, ctx, fm, env)] + rest, st1, label)
                return
        if k == "binop" and e[1] == "=" and e[2][0] == "prime":
            v = self.resolve_var(e[2][1], ctx, fm, env)
            if v is not None and v not in st1:
                rhs = self.ev(e[3], ctx, fm, self.with_next(env, st1))
                self.gen_next(rest, {**st1, v: rhs}, label)
                return
        if k == "binop" and e[1] == "\\in" and e[2][0] == "prime":
            # x' \in S: one successor per member of S (TLC enumerates S)
            v = self.resolve_var(e[2][1], ctx, fm, env)
            if v is not None and v not in st1:
                dom = self.ev(e[3], ctx, fm, self.with_next(env, st1))
                for g, x in self.distinct_items(dom):
                    self.guarded(g, lambda x=x: self.gen_next(rest, {**st1, v: x}, label))
                return
        if k == "unchanged":
            new1, conds = st1, []
            for v in self.unchanged_vars(e[1], ctx, fm, env):
                if v in new1:
                    conds.append(self.eq(new1[v], self.cur[v]))
                else:
                    new1 = {**new1, v: self.cur[v]}
            self.guarded(self.b_and(conds), lambda: self.gen_next(rest, new1, label))
            return
        c = self.ev_bool(e, ctx, fm, self.with_next(env, st1))
        self.guarded(c, lambda: self.gen_next(rest, st1, label))

    @staticmethod
    def with_next(env, st1):
        env2 = dict(env)
        env2["'"] = st1
        return env2

    def guarded(self, cond, body):
        if cond is False:
            return
        if cond is True:
            body()
            return
        if any(b.cond == cond.s for b in self.cg.stack):
            body()
            return
        self.cg.open(f"if ({cond.s})", cond.s)
        body()
        self.cg.close()

    def end_unit(self):
        """Close the current independently-compilable piece of expand() and start a new one."""
        if len(self.cg.stack) != 1:
            raise LowerError("internal: end_unit inside an open block")
        if self.cg.body.children:
            self.units.append(self.cg.body.children)
        self.unit_id += 1
        self.cg = self._unit_base.fork()

    def action_id(self, d: Def) -> int:
        for i, a in enumerate(self.actions):
            if a["name"] == d.name and a["module"] == d.module:
                return i
        self.actions.append({"name": d.name, "module": d.module, "line": d.line, "col": d.col,
                             "end_line": d.end_line, "end_col": d.end_col})
        return len(self.actions) - 1

    def read_ty(self, t):
        v = t.read(self)
        self.read_cache[id(t)] = v
        return v

    def emit_successor(self, st1: dict, label):
        for v in self.variables:
            if v not in st1:
                raise LowerError(f"an action branch leaves {v}' unassigned")
        if label is None:
            label = self.action_id(Def("Next", [], ("id", "Next"), False, self.root.module_name))
        lay = self.layout
        core = self.cg.open(label=label)
        self.traps = []
        out: dict[int, str] = {}
        for v in self.variables:
            ty = lay.var_types[v]
            if st1[v] is self.read_cache.get(id(ty)):
                continue
            ty.write(self, st1[v], out)
        ok = self.b_and(self.traps)
        self.traps = []
        by_word: dict[int, list] = {}
        for idx, code in out.items():
            a = lay.atoms[idx]
            if code == f"a{idx}":
                continue
            by_word.setdefault(a.word, []).append((a, code))
        if ok is False:
            core.label = -1
            self.cg.emit("sink.fail(KMC_FAIL_LAYOUT);")
            self.cg.close()
            return
        if ok is not True:
            self.cg.open(f"if ({ok.s})")
        self.cg.emit("State n = s;")
        for w, lst in sorted(by_word.items()):
            mask = 0
            parts = []
            for a, code in lst:
                mask |= a.mask << a.shift
                parts.append(f"((uint64_t)({code}) << {a.shift})" if a.shift else f"(uint64_t)({code})")
            self.cg.emit(f"n.w[{w}] = (s.w[{w}] & ~0x{mask:x}ull) | " + " | ".join(parts) + ";")
        self.cg.emit(f"sink.emit(n, {label});")
        self.emit_sites += 1
        if ok is not True:
            self.cg.close()
            self.cg.emit("else sink.fail(KMC_FAIL_LAYOUT);")
        self.cg.close()

    # ------------------------------------------------------------ symmetry
    def permute_const(self, v, pmap: dict):
        if is_atom_const(v):
            return pmap.get(v, v)
        if isinstance(v, frozenset):
            return frozenset(self.permute_const(x, pmap) for x in v)
        if isinstance(v, FnVal):
            return FnVal({self.permute_const(k, pmap): self.permute_const(x, pmap) for k, x in v.items})
        if isinstance(v, tuple):
            return tuple(self.permute_const(x, pmap) for x in v)
        return v

    def permute_sval(self, v, pmap: dict):
        """Image of a (symbolic) value under a permutation of model values; returns ``v`` itself
        when nothing in it can move, so that unchanged variables are not re-encoded."""
        if is_const(v):
            return self.permute_const(v, pmap)
        if isinstance(v, (SInt, SBool)):
            return v
        if isinstance(v, SAtom):
            moved = [a for a in v.uni if pmap.get(a, a) != a]
            if not moved:
                return v
            e = v.s
            for a in moved:
                e = f"({v.s} == {self.gid(a)} ? {self.gid(pmap[a])} : {e})"
            return SAtom(self.tmp_int(e), tuple(dict.fromkeys(pmap.get(a, a) for a in v.uni)))
        if isinstance(v, SRec):
            new = {f: self.permute_sval(x, pmap) for f, x in v.fields.items()}
            return v if all(new[f] is v.fields[f] for f in new) else SRec(new)
        if isinstance(v, SFn):
            keys = [self.permute_const(k, pmap) for k in v.keys]
            vals = [self.permute_sval(x, pmap) for x in v.vals]
            if keys == list(v.keys) and all(a is b for a, b in zip(vals, v.vals)):
                return v
            order = sorted(range(len(keys)), key=lambda i: sort_key(keys[i]))
            return SFn([keys[i] for i in order], [vals[i] for i in order])
        if isinstance(v, SSet):
            items = [(g, self.permute_sval(x, pmap)) for g, x in v.items]
            if all(a[1] is b[1] for a, b in zip(items, v.items)):
                return v
            return SSet(items, distinct=v.distinct)
        if isinstance(v, SUnion):
            alts = [(g, self.permute_sval(x, pmap)) for g, x in v.alts]
            return v if all(a[1] is b[1] for a, b in zip(alts, v.alts)) else SUnion(alts)
        raise LowerError(f"cannot permute {v!r}")

    def gen_permuted_words(self, pmap: dict) -> list[str]:
        """C expressions of the packed words of the current state's image under ``pmap``."""
        lay = self.layout
        out: dict[int, str] = {}
        self.traps = []
        for v in self.variables:
            ty = lay.var_types[v]
            img = self.permute_sval(self.cur[v], pmap)
            if img is self.cur[v]:
                continue
            ty.write(self, img, out)
        self.traps = []          # a permuted reachable value always fits its own layout
        by_word: dict[int, list] = {}
        for idx, code in out.items():
            a = lay.atoms[idx]
            by_word.setdefault(a.word, []).append((a, code))
        words = []
        for w in range(lay.words):
            lst = by_word.get(w, [])
            if not lst:
                words.append(f"s.w[{w}]")
                continue
            mask = 0
            parts = []
            for a, code in lst:
                mask |= a.mask << a.shift
                parts.append(f"((uint64_t)({code}) << {a.shift})" if a.shift else f"(uint64_t)({code})")
            words.append(f"((s.w[{w}] & ~0x{mask:x}ull) | " + " | ".join(parts) + ")")
        return words

    # ------------------------------------------------------------ predicates
    def named_def(self, name: str) -> tuple[Def, ModuleContext]:
        r = self.root.resolve(name, None)
        if r is None or r.kind != "def":
            raise LowerError(f"{name} is not defined in module {self.root.module_name}")
        return r.defn, r.ctx

    def begin_function(self):
        """Fresh emitter + symbolic reads of every state atom.  Whatever the reads emit (decode
        temporaries) becomes the function prologue, replicated in every group function."""
        self.cg = CG()
        self.read_cache = {}
        self.enc_cache = {}
        self.mux_origin = {}
        self.unit_id = -2                      # values forced while reading belong to the prologue
        self.cur = {v: self.read_ty(self.layout.var_types[v]) for v in self.variables}
        self.prologue = render(self.cg.body.children, 1)
        self.cg.body.children = []
        self._unit_base = self.cg
        self.units = []
        self.unit_id = 0
        self.cg = self._unit_base.fork()

    def unpack_lines(self) -> list[str]:
        out = []
        for a in self.layout.atoms:
            sh = f" >> {a.shift}" if a.shift else ""
            if a.bits > 32:
                out.append(f"  [[maybe_unused]] const uint64_t a{a.index} = (s.w[{a.word}]{sh}) & 0x{a.mask:x}ull;  // {a.path}")
                continue
            out.append(f"  [[maybe_unused]] const unsigned a{a.index} = (unsigned)((s.w[{a.word}]{sh}) & 0x{a.mask:x}ull);"
                       f"  // {a.path}")
        return out
