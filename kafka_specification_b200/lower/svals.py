"""Symbolic values used by the ahead-of-time lowering.

The lowering evaluates the spec with *partially known* values: everything that depends only on
the ``.cfg`` constants is an ordinary Python value (int, bool, str, ModelValue, frozenset,
FnVal), everything that depends on the packed state is one of the classes below, whose leaves
are C expression strings over the unpacked state atoms.

  SInt   runtime integer with a static interval [lo, hi]
  SBool  runtime boolean
  SAtom  runtime model-value/string, represented by its global atom id (gid)
  SRec   record with symbolic fields          SFn   function over a constant finite domain
  SSet   guarded element list [(guard, elem)] -- the set of elems whose guard holds
  SUnion value of one of several kinds [(guard, value)], guards mutually exclusive
  SLazy  non-enumerated set descriptor (record sets, function sets, SUBSET, Nat, Seq(S), S \\X T, a wide a .. b)
  SSeq   sequence / tuple: a length (int or SInt) and ``cap`` item values; item i (0-based) is meaningful
         iff i < length.  A fully constant sequence is a Python tuple.
"""
from __future__ import annotations

from ..frontend.cfg import ModelValue
from ..frontend.values import FnVal


class LowerError(Exception):
    pass


INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1


def fits_int(lo: int, hi: int) -> bool:
    """Does every value of [lo, hi] fit a C `int`?"""
    return INT32_MIN <= lo and hi <= INT32_MAX


def c_int(v: int) -> str:
    """The C literal of an integer constant (the most negative int64_t has none: -2^63 + 1 would be its negation)."""
    if not INT64_MIN <= v <= INT64_MAX:
        raise LowerError(f"the integer {v} is beyond 64-bit integers")
    return "(-9223372036854775807ll - 1)" if v == INT64_MIN else str(v)


class SInt:
    __slots__ = ("s", "lo", "hi")

    def __init__(self, s: str, lo: int, hi: int):
        self.s, self.lo, self.hi = s, lo, hi

    def __repr__(self):
        return f"SInt({self.s} in {self.lo}..{self.hi})"


class SBool:
    __slots__ = ("s",)

    def __init__(self, s: str):
        self.s = s

    def __repr__(self):
        return f"SBool({self.s})"


class SAtom:
    __slots__ = ("s", "uni")

    def __init__(self, s: str, uni: tuple):
        self.s, self.uni = s, tuple(uni)

    def __repr__(self):
        return f"SAtom({self.s} in {self.uni})"


class SRec:
    __slots__ = ("fields",)

    def __init__(self, fields: dict):
        self.fields = fields

    def __repr__(self):
        return f"SRec({self.fields})"


class SFn:
    __slots__ = ("keys", "vals")

    def __init__(self, keys: list, vals: list):
        self.keys, self.vals = list(keys), list(vals)

    def __repr__(self):
        return f"SFn({dict(zip(self.keys, self.vals))})"


class SSet:
    __slots__ = ("items", "distinct")

    def __init__(self, items: list, distinct: bool = False):
        self.items = [(g, x) for g, x in items if g is not False]
        self.distinct = distinct      # True: no two present elements are equal (canonical layouts, filters of them)

    def __repr__(self):
        return f"SSet({self.items})"


class SUnion:
    __slots__ = ("alts",)

    def __init__(self, alts: list):
        self.alts = [(g, x) for g, x in alts if g is not False]

    def __repr__(self):
        return f"SUnion({self.alts})"


class SSeq:
    __slots__ = ("n", "items")

    def __init__(self, n, items: list):
        self.n, self.items = n, list(items)     # n: int or SInt with hi <= len(items)

    @property
    def cap(self) -> int:
        return len(self.items)

    def __repr__(self):
        return f"SSeq(len={self.n}, {self.items})"


class SLazy:
    """Constant set descriptors that are never enumerated unless asked to."""
    __slots__ = ("kind", "a", "b")

    def __init__(self, kind: str, a=None, b=None):
        self.kind, self.a, self.b = kind, a, b   # 'nat' | 'int' | 'recset'(a=dict) | 'fnset'(a=dom,b=rng) | 'powerset'(a=base) | 'union'(a,b) | 'seq'(a=elem set) | 'cross'(a=[sets]) | 'range'(a=lo, b=hi: int or SInt)

    def __repr__(self):
        return f"SLazy({self.kind}, {self.a}, {self.b})"


SYMBOLIC = (SInt, SBool, SAtom, SRec, SFn, SSet, SUnion, SLazy, SSeq)


def is_const(v) -> bool:
    return not isinstance(v, SYMBOLIC)


def is_atom_const(v) -> bool:
    return isinstance(v, (str, ModelValue))


def is_int_const(v) -> bool:
    return isinstance(v, int) and not isinstance(v, bool)


def is_static(v) -> bool:
    """True if v contains no runtime expression (safe to cache across code blocks)."""
    if is_const(v):
        return True
    if isinstance(v, SLazy):
        if v.kind in ("nat", "int"):
            return True
        if v.kind == "recset":
            return all(is_static(x) for x in v.a.values())
        if v.kind == "cross":
            return all(is_static(x) for x in v.a)
        return is_static(v.a) and (v.b is None or is_static(v.b))
    return False


def kind_sig(v) -> str:
    """Coarse TLA+ kind of a (symbolic or constant) value."""
    if isinstance(v, bool) or isinstance(v, SBool):
        return "bool"
    if isinstance(v, SInt) or is_int_const(v):
        return "int"
    if isinstance(v, SAtom) or is_atom_const(v):
        return "atom"
    if isinstance(v, SRec):
        return "rec:" + ",".join(sorted(v.fields))
    if isinstance(v, FnVal):
        dom = list(v.domain())
        if dom and all(isinstance(k, str) for k in dom):
            return "rec:" + ",".join(sorted(dom))
        return "fn"
    if isinstance(v, SFn):
        return "fn"
    if isinstance(v, (SSet, SLazy, frozenset)):
        return "set"
    if isinstance(v, SUnion):
        return "union"
    if isinstance(v, (tuple, SSeq)):
        return "tuple"
    raise LowerError(f"unknown value kind {v!r}")
