"""Fixed-width packed state layout.

A state is ``W`` 64-bit words.  Every state variable gets a *layout type* (inferred from the
spec's own type invariant, e.g. KafkaReplication.tla:101-107, see ``typeinfer.py``); the leaves
of the type tree are *atoms*: unsigned bit-fields that never straddle a word.

Type            encoding
--------------  -----------------------------------------------------------------------------
TInt(lo, hi)    code = value - lo; the one type whose atom may be wider than 32 bits (up to 63: read as int64_t)
TEnum(atoms)    code = index of the model value / string in the (gid-sorted) universe
TUnion(alts)    code = offset(alt) + alt code          (records[o] is a record or Nil, FiniteReplicatedLog.tla:41-44)
TRec / TFn      product of the members: separate atoms at top level, mixed radix when nested in a set/union
TSet bitmap     one bit per possible element (element code = bit index)
TSet array      count + ``cap`` element codes kept sorted ascending, unused slots 0 -> canonical, so
                equal sets pack to equal bits (leaderAndIsrRequests, KafkaReplication.tla:66)
TKeyedSet       set of records in which one field (the key) determines the record (checked): one entry per key
                value, 0 = absent, c + 1 = mixed-radix code c of the other fields  (``\\* kspec: KEYED v BY f``)
TPrefixFn       function over 0..n-1 into X \\union {Nil} whose Nil entries are exactly those at index >= a sibling
                length field (checked; FiniteReplicatedLog.tla:84-87 states it): only X is coded
                (``\\* kspec: PREFIX v arrayField lengthField``)

TTuple          fixed-length tuple (an element of S \\X T): one member per position
TSeq            sequence of at most ``cap`` scalar-codeable elements (``v \\in Seq(S)`` + ``\\* kspec: CAPACITY v = cap``):
                a length field and cap element codes; the slots at index >= length hold code 0, so equal sequences
                pack to equal bits

Every type offers the same operations in two worlds: ``py_*`` on Python values (Init states,
decoding traces, tests) and ``read``/``write``/``enc``/``dec`` on symbolic values, emitting C.
"""
from __future__ import annotations

from ..frontend.cfg import ModelValue
from ..frontend.values import FnVal, fmt, sort_key
from .svals import (INT32_MAX, INT64_MAX, INT64_MIN, LowerError, SAtom, SBool, SFn, SInt, SRec, SSeq, SSet, SUnion,
                    c_int, fits_int, is_atom_const, is_const, is_int_const, kind_sig)


def bits_for(card: int) -> int:
    return max(0, (card - 1).bit_length())


def parse_value(text: str):
    """A key or enum value as ``fmt`` printed it into a description: quoted text is a string, digits an int, anything
    else a model value."""
    if text.startswith('"'):
        return text[1:-1]
    try:
        return int(text)
    except ValueError:
        return ModelValue(text)


class Atom:
    __slots__ = ("index", "path", "bits", "word", "shift", "card")

    def __init__(self, index, path, bits, card=None):
        self.index, self.path, self.bits = index, path, bits
        self.word = self.shift = 0
        self.card = card if card is not None else (1 << bits)     # number of codes a valid state can hold

    @property
    def mask(self) -> int:
        return (1 << self.bits) - 1


class Layout:
    def __init__(self):
        self.atoms: list[Atom] = []
        self.var_types: dict[str, "Ty"] = {}
        self.variables: list[str] = []
        self.spans: dict[str, tuple[int, int]] = {}      # variable -> the index range [begin, end) of its atoms
        self.words = 0
        self.bits = 0

    def add_variable(self, v: str, ty: "Ty"):
        """Allocates the atoms of ``v`` after those of the variables added before it."""
        begin = len(self.atoms)
        ty.alloc(self, v)
        self.variables.append(v)
        self.var_types[v] = ty
        self.spans[v] = (begin, len(self.atoms))

    @classmethod
    def from_description(cls, desc: dict) -> "Layout":
        """The inverse of ``describe()`` (what model.json holds), for decoding: the variables' types are rebuilt, their
        atoms allocated in variable order and placed at the described word / shift.  A description these types do not
        allocate atom for atom (a model.json written by another version of the lowering) raises."""
        lay = cls()
        for v in desc["variables"]:
            lay.add_variable(v, ty_from_description(desc["types"][v]))
        got = [(a.path, a.bits) for a in lay.atoms]
        want = [(a["path"], a["bits"]) for a in desc["atoms"]]
        if got != want:
            i = next((i for i, (g, w) in enumerate(zip(got, want)) if g != w), min(len(got), len(want)))
            raise LowerError(f"layout description does not match its types: atom {i} is described as "
                             f"{want[i] if i < len(want) else None}, the types allocate {got[i] if i < len(got) else None}")
        for a, d in zip(lay.atoms, desc["atoms"]):
            a.word, a.shift = d["word"], d["shift"]
        lay.words, lay.bits = desc["words"], desc["bits"]
        return lay

    def new_atom(self, path: str, bits: int, card: int | None = None, max_bits: int = 32) -> Atom:
        """A new atom; only an integer field may be wider than 32 bits (its code is computed in 64-bit arithmetic)."""
        if bits > max_bits:
            raise LowerError(f"atom {path} needs {bits} bits (> {max_bits})")
        a = Atom(len(self.atoms), path, bits, card)
        self.atoms.append(a)
        return a

    def finish(self):
        word, used = 0, 0
        for a in self.atoms:
            if used + a.bits > 64:
                word, used = word + 1, 0
            a.word, a.shift = word, used
            used += a.bits
            self.bits += a.bits
        if word + 1 > max(1, -(-self.bits // 64)):
            # declaration order wastes a word (atoms never straddle words): first-fit decreasing over the bit
            # widths, declaration order among equals -- e.g. the 128-bit Kafka layout fits two words exactly
            fill: list[int] = []
            place = {}
            for a in sorted(self.atoms, key=lambda a: (-a.bits, a.index)):
                for w, u in enumerate(fill):
                    if u + a.bits <= 64:
                        break
                else:
                    fill.append(0)
                    w = len(fill) - 1
                place[a.index] = (w, fill[w])
                fill[w] += a.bits
            if len(fill) < word + 1:
                for a in self.atoms:
                    a.word, a.shift = place[a.index]
                word = len(fill) - 1
        self.words = word + 1
        # can the packed words of a valid state be all ones?  (No, as soon as one field cannot hold its top code
        # or a word has unused high bits: the engine then uses all-ones as the empty marker of its exact set.)
        last_used = sum(a.bits for a in self.atoms if a.word == word)
        self.all_ones_possible = all(a.card == (1 << a.bits) for a in self.atoms) and last_used == 64

    # -- python-side packing -------------------------------------------------
    def py_pack(self, state: dict) -> list[int]:
        codes: dict[int, int] = {}
        for v in self.variables:
            self.var_types[v].py_write(state[v], codes)
        words = [0] * self.words
        for a in self.atoms:
            c = codes.get(a.index, 0)
            if c < 0 or c > a.mask:
                raise LowerError(f"value for {a.path} does not fit its layout ({c} in {a.bits} bits)")
            words[a.word] |= c << a.shift
        return words

    def py_unpack(self, words) -> dict:
        codes = {a.index: (int(words[a.word]) >> a.shift) & a.mask for a in self.atoms}
        return {v: self.var_types[v].py_read(codes) for v in self.variables}

    def describe(self) -> dict:
        return {
            "words": self.words, "bits": self.bits, "variables": self.variables,
            "atoms": [{"path": a.path, "bits": a.bits, "word": a.word, "shift": a.shift} for a in self.atoms],
            "types": {v: self.var_types[v].describe() for v in self.variables},
        }


# ---------------------------------------------------------------------------
class Ty:
    card: int = 0          # number of values if the type is codeable as one integer, else 0
    _sig = None

    def sig(self) -> str:
        """Structural identity of the encoding: equal sig <=> equal value/code mapping."""
        if self._sig is None:
            import json
            self._sig = json.dumps(self.describe(), sort_keys=True)
        return self._sig

    def alloc(self, lay: Layout, path: str):
        raise NotImplementedError

    def describe(self):
        raise NotImplementedError

    def kind(self) -> str:
        raise NotImplementedError

    # python values
    def py_enc(self, v) -> int:
        raise LowerError(f"type {self.describe()} is not scalar-codeable")

    def py_dec(self, code: int):
        raise LowerError(f"type {self.describe()} is not scalar-codeable")

    def py_write(self, v, codes: dict):
        codes[self.atom.index] = self.py_enc(v)

    def py_read(self, codes: dict):
        return self.py_dec(codes[self.atom.index]) if self.atom is not None else self.py_dec(0)

    # symbolic values; ``lw`` is the Lowerer
    def enc(self, lw, v) -> str:
        raise LowerError(f"type {self.describe()} is not scalar-codeable")

    def dec(self, lw, code: str):
        raise LowerError(f"type {self.describe()} is not scalar-codeable")

    def read(self, lw):
        if self.atom is None:
            return self.py_dec(0)
        v = self.dec(lw, f"a{self.atom.index}")
        lw.remember_code(self, v, f"a{self.atom.index}")
        return v

    def write(self, lw, v, out: dict):
        if self.atom is None:
            return
        out[self.atom.index] = lw.encode(self, v)

    def _alloc_scalar(self, lay: Layout, path: str, max_bits: int = 32):
        b = bits_for(self.card)
        self.atom = lay.new_atom(path, b, self.card, max_bits) if b > 0 else None


class TInt(Ty):
    def __init__(self, lo: int, hi: int):
        self.lo, self.hi = lo, hi
        self.card = hi - lo + 1
        self.atom = None

    def kind(self):
        return "int"

    def describe(self):
        return {"t": "int", "lo": self.lo, "hi": self.hi}

    def alloc(self, lay, path):
        if not INT64_MIN < self.lo <= self.hi <= INT64_MAX:
            raise LowerError(f"integer field {path} ranges over {self.lo} .. {self.hi}, beyond 64-bit integers")
        self._alloc_scalar(lay, path, max_bits=63)

    def narrow(self) -> bool:
        """Do the values and the codes of this field fit a C `int`?  (Else they are read as `int64_t`.)"""
        return fits_int(self.lo, self.hi) and self.card - 1 <= INT32_MAX

    def py_enc(self, v):
        if not is_int_const(v) or not (self.lo <= v <= self.hi):
            raise LowerError(f"value {fmt(v)} outside layout range {self.lo}..{self.hi}")
        return v - self.lo

    def py_dec(self, code):
        return code + self.lo

    def enc(self, lw, v):
        if is_const(v):
            return str(self.py_enc(v))
        if isinstance(v, SUnion):
            return lw.enc_union_into(self, v)
        if not isinstance(v, SInt):
            raise LowerError(f"cannot store {v!r} in an integer field")
        if v.lo < self.lo or v.hi > self.hi:
            lw.trap_unless(lw.b_and([lw.cmp(">=", v, self.lo), lw.cmp("<=", v, self.hi)]))
        if fits_int(v.lo, v.hi) and fits_int(v.lo - self.lo, v.hi - self.lo):
            return lw.tmp_int(f"({v.s} - {self.lo})" if self.lo else v.s)
        if not self.lo:
            return lw.tmp_int(v.s, v.lo, v.hi)
        # in 64-bit unsigned arithmetic, where the code of a value that traps (and is never stored) cannot overflow
        return lw.tmp_code(self, f"((uint64_t){v.s} - 0x{self.lo & ((1 << 64) - 1):x}ull)")

    def dec(self, lw, code):
        if self.card == 1:
            return self.lo
        if not self.narrow():
            return SInt(f"((int64_t){code} + {c_int(self.lo)})" if self.lo else f"(int64_t){code}", self.lo, self.hi)
        return SInt(f"((int){code} + {self.lo})" if self.lo else f"(int){code}", self.lo, self.hi)


class TBool(Ty):
    """BOOLEAN-valued field: one bit."""

    def __init__(self):
        self.card = 2
        self.atom = None

    def kind(self):
        return "bool"

    def describe(self):
        return {"t": "bool"}

    def alloc(self, lay, path):
        self._alloc_scalar(lay, path)

    def py_enc(self, v):
        if not isinstance(v, bool):
            raise LowerError(f"value {fmt(v)} is not a boolean")
        return 1 if v else 0

    def py_dec(self, code):
        return bool(code)

    def enc(self, lw, v):
        if is_const(v):
            return str(self.py_enc(v))
        if isinstance(v, SUnion):
            return lw.enc_union_into(self, v)
        if not isinstance(v, SBool):
            raise LowerError(f"cannot store {v!r} in a boolean field")
        return lw.tmp_int(f"({v.s} ? 1 : 0)")

    def dec(self, lw, code):
        return SBool(f"({code} != 0)")


class TEnum(Ty):
    def __init__(self, atoms: list, gids: dict):
        self.atoms = sorted(atoms, key=lambda a: gids[a])
        self.gid = {a: gids[a] for a in self.atoms}
        self.card = len(self.atoms)
        g = [self.gid[a] for a in self.atoms]
        self.base = g[0]
        self.contiguous = g == list(range(g[0], g[0] + len(g)))
        self.atom = None

    def kind(self):
        return "atom"

    def describe(self):
        return {"t": "enum", "values": [fmt(a) for a in self.atoms]}

    def alloc(self, lay, path):
        self._alloc_scalar(lay, path)

    def py_enc(self, v):
        if v not in self.gid:
            raise LowerError(f"value {fmt(v)} outside layout enum {[fmt(a) for a in self.atoms]}")
        return self.atoms.index(v)

    def py_dec(self, code):
        return self.atoms[code]

    def enc(self, lw, v):
        if is_const(v):
            return str(self.py_enc(v))
        if isinstance(v, SUnion):
            return lw.enc_union_into(self, v)
        if not isinstance(v, SAtom):
            raise LowerError(f"cannot store {v!r} in an enum field")
        if not set(v.uni) <= set(self.atoms):
            lw.trap_unless(lw.b_or([SBool(f"({v.s} == {self.gid[a]})") for a in self.atoms]))
        if self.contiguous:
            return lw.tmp_int(f"({v.s} - {self.base})" if self.base else v.s)
        e = "0"
        for i, a in reversed(list(enumerate(self.atoms))):
            e = f"({v.s} == {self.gid[a]} ? {i} : {e})"
        return lw.tmp_int(e)

    def dec(self, lw, code):
        if self.card == 1:
            return self.atoms[0]
        if self.contiguous:
            return SAtom(f"((int){code} + {self.base})" if self.base else f"(int){code}", tuple(self.atoms))
        e = str(self.gid[self.atoms[-1]])
        for i, a in reversed(list(enumerate(self.atoms[:-1]))):
            e = f"({code} == {i} ? {self.gid[a]} : {e})"
        return SAtom(lw.tmp_int(e), tuple(self.atoms))


class TRec(Ty):
    def __init__(self, fields: dict):
        self.fields = dict(fields)          # name -> Ty, in declaration order
        self.card = 1
        for t in self.fields.values():
            self.card = self.card * t.card if (t.card and self.card) else 0
        if self.card > (1 << 30):
            self.card = 0
        self.atom = None

    def kind(self):
        return "rec:" + ",".join(sorted(self.fields))

    def describe(self):
        return {"t": "rec", "fields": {f: t.describe() for f, t in self.fields.items()}}

    def alloc(self, lay, path):
        for f, t in self.fields.items():
            t.alloc(lay, f"{path}.{f}")

    def apply_prefix(self, arr: str, length: str):
        """``fields[arr]`` (a function over 0..n-1 into X \\union {nil}) becomes a TPrefixFn governed by ``fields[length]``."""
        ft, lt = self.fields.get(arr), self.fields.get(length)
        if not isinstance(ft, TFn) or not isinstance(lt, TInt):
            raise LowerError(f"PREFIX needs a function field {arr} and an integer field {length}")
        if list(ft.keys) != list(range(len(ft.keys))):
            raise LowerError(f"PREFIX: the domain of {arr} must be 0..n-1")
        u = ft.elems[0]
        if not isinstance(u, TUnion) or len(u.alts) != 2 or sorted(t.card == 1 for t in u.alts) != [False, True]:
            raise LowerError(f"PREFIX: {arr} must map into X \\union {{Nil}} with a single Nil value")
        nil_t = next(t for t in u.alts if t.card == 1)
        inner_t = next(t for t in u.alts if t.card != 1)
        pf = TPrefixFn(ft.keys, inner_t, nil_t.py_dec(0), length)
        # the length field must be read / written before the array
        order = [f for f in self.fields if f != arr]
        order.insert(order.index(length) + 1, arr)
        self.fields = {f: (pf if f == arr else self.fields[f]) for f in order}
        self.card = 0
        self._sig = None

    def _get(self, v, f):
        if isinstance(v, FnVal):
            return v.apply(f)
        return v.fields[f]

    def _check(self, v):
        names = set(v.domain()) if isinstance(v, FnVal) else set(v.fields) if isinstance(v, SRec) else None
        if names != set(self.fields):
            raise LowerError(f"cannot store {v!r} in record layout {list(self.fields)}")

    def py_enc(self, v):
        if not isinstance(v, FnVal) or set(v.domain()) != set(self.fields):
            raise LowerError(f"value {fmt(v)} is not a record with fields {list(self.fields)}")
        code, stride = 0, 1
        for f, t in self.fields.items():
            code += t.py_enc(v.apply(f)) * stride
            stride *= t.card
        return code

    def py_dec(self, code):
        d = {}
        for f, t in self.fields.items():
            d[f] = t.py_dec(code % t.card)
            code //= t.card
        return FnVal(d)

    def py_write(self, v, codes):
        if not isinstance(v, FnVal) or set(v.domain()) != set(self.fields):
            raise LowerError(f"value {fmt(v)} is not a record with fields {list(self.fields)}")
        for f, t in self.fields.items():
            if isinstance(t, TPrefixFn):
                t.py_write_len(v.apply(f), v.apply(t.len_field), codes)
            else:
                t.py_write(v.apply(f), codes)

    def py_read(self, codes):
        d = {}
        for f, t in self.fields.items():
            d[f] = t.py_read_len(codes, d[t.len_field]) if isinstance(t, TPrefixFn) else t.py_read(codes)
        return FnVal(d)

    def enc(self, lw, v):
        if is_const(v):
            return str(self.py_enc(v))
        if isinstance(v, SUnion):
            return lw.enc_union_into(self, v)
        self._check(v)
        terms, stride = [], 1
        for f, t in self.fields.items():
            c = lw.encode(t, self._get(v, f))
            terms.append(c if stride == 1 else f"{c} * {stride}")
            stride *= t.card
        return lw.tmp_int("(" + " + ".join(terms) + ")")

    def dec(self, lw, code):
        out, stride = {}, 1
        for f, t in self.fields.items():
            if t.card == 1:
                out[f] = t.py_dec(0)
            else:
                x = code if stride == 1 else f"({code} / {stride})"
                if stride * t.card < self.card:
                    x = f"({x} % {t.card})"
                out[f] = t.dec(lw, lw.tmp_int(x))
            stride *= t.card
        return SRec(out)

    def read(self, lw):
        d = {}
        for f, t in self.fields.items():
            if isinstance(t, TPrefixFn):
                d[f] = t.read_len(lw, d[t.len_field])
                lw.read_cache[id(t)] = d[f]
            else:
                d[f] = lw.read_ty(t)
        return SRec(d)

    def write(self, lw, v, out):
        if isinstance(v, SUnion):
            v = lw.narrow_union(v, self.kind())
        self._check(v)
        for f, t in self.fields.items():
            x = self._get(v, f)
            if isinstance(t, TPrefixFn):
                newlen = self._get(v, t.len_field)
                t.write_len(lw, x, newlen, newlen is not lw.read_cache.get(id(self.fields[t.len_field])), out)
                continue
            if x is lw.read_cache.get(id(t)):
                continue                      # member untouched since it was read
            t.write(lw, x, out)


class TFn(Ty):
    def __init__(self, keys: list, elem_types: list):
        self.keys = list(keys)
        self.elems = list(elem_types)       # one Ty instance per key (separate atoms)
        self.card = 1
        for t in self.elems:
            self.card = self.card * t.card if (t.card and self.card) else 0
        if self.card > (1 << 30):
            self.card = 0
        self.atom = None

    def kind(self):
        return "fn"

    def describe(self):
        return {"t": "fn", "keys": [fmt(k) for k in self.keys], "elem": self.elems[0].describe()}

    def alloc(self, lay, path):
        for k, t in zip(self.keys, self.elems):
            t.alloc(lay, f"{path}[{fmt(k)}]")

    def _vals(self, v):
        if isinstance(v, FnVal):
            if set(v.domain()) != set(self.keys):
                raise LowerError(f"function domain mismatch storing {fmt(v)}")
            return [v.apply(k) for k in self.keys]
        if isinstance(v, SFn):
            if set(v.keys) != set(self.keys):
                raise LowerError("function domain mismatch")
            m = dict(zip(v.keys, v.vals))
            return [m[k] for k in self.keys]
        raise LowerError(f"cannot store {v!r} in a function layout")

    def py_enc(self, v):
        code, stride = 0, 1
        for t, x in zip(self.elems, self._vals(v)):
            code += t.py_enc(x) * stride
            stride *= t.card
        return code

    def py_dec(self, code):
        d = {}
        for k, t in zip(self.keys, self.elems):
            d[k] = t.py_dec(code % t.card)
            code //= t.card
        return FnVal(d)

    def py_write(self, v, codes):
        for t, x in zip(self.elems, self._vals(v)):
            t.py_write(x, codes)

    def py_read(self, codes):
        return FnVal({k: t.py_read(codes) for k, t in zip(self.keys, self.elems)})

    def enc(self, lw, v):
        if is_const(v):
            return str(self.py_enc(v))
        terms, stride = [], 1
        for t, x in zip(self.elems, self._vals(v)):
            c = lw.encode(t, x)
            terms.append(c if stride == 1 else f"{c} * {stride}")
            stride *= t.card
        return lw.tmp_int("(" + " + ".join(terms) + ")")

    def dec(self, lw, code):
        vals, stride = [], 1
        for t in self.elems:
            x = code if stride == 1 else f"({code} / {stride})"
            if stride * t.card < self.card:
                x = f"({x} % {t.card})"
            vals.append(t.dec(lw, lw.tmp_int(x)) if t.card > 1 else t.py_dec(0))
            stride *= t.card
        return SFn(self.keys, vals)

    def read(self, lw):
        return SFn(self.keys, [lw.read_ty(t) for t in self.elems])

    def write(self, lw, v, out):
        for t, x in zip(self.elems, self._vals(v)):
            if x is lw.read_cache.get(id(t)):
                continue
            t.write(lw, x, out)


class TUnion(Ty):
    def __init__(self, alts: list):
        self.alts = list(alts)
        if any(not t.card for t in alts):
            raise LowerError("union alternatives must be scalar-codeable")
        kinds = [t.kind() for t in alts]
        if len(set(kinds)) != len(kinds):
            raise LowerError(f"union alternatives must have distinct kinds, got {kinds}")
        self.offsets, off = [], 0
        for t in alts:
            self.offsets.append(off)
            off += t.card
        self.card = off
        self.atom = None

    def kind(self):
        return "union"

    def describe(self):
        return {"t": "union", "alts": [t.describe() for t in self.alts]}

    def alloc(self, lay, path):
        self._alloc_scalar(lay, path)

    def _alt_for_kind(self, k: str):
        for i, t in enumerate(self.alts):
            if t.kind() == k:
                return i
        return None

    def py_enc(self, v):
        i = self._alt_for_kind(kind_sig(v))
        if i is None:
            raise LowerError(f"value {fmt(v)} fits no alternative of {self.describe()}")
        return self.offsets[i] + self.alts[i].py_enc(v)

    def py_dec(self, code):
        for t, off in zip(reversed(self.alts), reversed(self.offsets)):
            if code >= off:
                return t.py_dec(code - off)
        raise LowerError("bad union code")

    def enc(self, lw, v):
        if is_const(v):
            return str(self.py_enc(v))
        if isinstance(v, SUnion):
            e = None
            for g, x in reversed(v.alts):
                c = lw.encode(self, x)
                e = c if e is None else f"({lw.bstr(g)} ? {c} : {e})"
            return lw.tmp_int(e if e is not None else "0")
        i = self._alt_for_kind(kind_sig(v))
        if i is None:
            raise LowerError(f"value {v!r} fits no alternative of {self.describe()}")
        c = lw.encode(self.alts[i], v)
        return lw.tmp_int(f"({c} + {self.offsets[i]})" if self.offsets[i] else c)

    def dec(self, lw, code):
        alts = []
        n = len(self.alts)
        for i, (t, off) in enumerate(zip(self.alts, self.offsets)):
            conds = []
            if i > 0:
                conds.append(f"{code} >= {off}")
            if i < n - 1:
                conds.append(f"{code} < {off + t.card}")
            g = SBool(lw.tmp_bool("(" + " && ".join(conds) + ")")) if conds else True
            if t.card == 1:
                val = t.py_dec(0)
            else:
                val = t.dec(lw, lw.tmp_int(f"({code} - {off})") if off else code)
            alts.append((g, val))
        return SUnion(alts)


class TSet(Ty):
    """Set of ``elem``; bitmap over element codes, or sorted bounded array when ``cap`` is given."""

    def __init__(self, elem: Ty, cap: int | None = None, nonempty: bool = False):
        if not elem.card:
            raise LowerError("set element type must be scalar-codeable")
        self.elem, self.cap = elem, cap
        # nonempty: the type excludes {} (checked); as a scalar code the bitmap is stored minus one
        self.nonempty = bool(nonempty) and cap is None
        self.card = ((1 << elem.card) - (1 if self.nonempty else 0)) if (cap is None and elem.card <= 30) else 0
        self.chunks: list[Atom] = []
        self.count_atom = None
        self.slots: list[Atom] = []
        self.atom = None

    def kind(self):
        return "set"

    def describe(self):
        d = {"t": "set", "elem": self.elem.describe(), "repr": "bitmap" if self.cap is None else "array"}
        if self.cap is not None:
            d["cap"] = self.cap
        if self.nonempty:
            d["nonempty"] = True
        return d

    def alloc(self, lay, path):
        if self.cap is None:
            n, i = self.elem.card, 0
            while n > 0:
                b = min(32, n)
                self.chunks.append(lay.new_atom(f"{path}#bits{i}", b))
                n -= b
                i += 1
        else:
            self.count_atom = lay.new_atom(f"{path}#count", bits_for(self.cap + 1), self.cap + 1)
            eb = bits_for(self.elem.card)
            self.slots = [lay.new_atom(f"{path}#slot{i}", eb, self.elem.card) for i in range(self.cap)]

    # python
    def _py_codes(self, v) -> list[int]:
        if not isinstance(v, frozenset):
            raise LowerError(f"value {fmt(v)} is not a set")
        return sorted(self.elem.py_enc(x) for x in v)

    def py_enc(self, v):
        if not self.card:
            return super().py_enc(v)
        m = 0
        for c in self._py_codes(v):
            m |= 1 << c
        if self.nonempty:
            if m == 0:
                raise LowerError("empty set stored in a non-empty set layout")
            m -= 1
        return m

    def py_dec(self, code):
        if not self.card:
            return super().py_dec(code)
        if self.nonempty:
            code += 1
        return frozenset(self.elem.py_dec(j) for j in range(self.elem.card) if (code >> j) & 1)

    def py_write(self, v, codes):
        cs = self._py_codes(v)
        if self.nonempty and not cs:
            raise LowerError("empty set stored in a non-empty set layout")
        if self.cap is None:
            for i, a in enumerate(self.chunks):
                codes[a.index] = sum(1 << (c - 32 * i) for c in cs if 32 * i <= c < 32 * i + a.bits)
        else:
            if len(cs) > self.cap:
                raise LowerError(f"set {fmt(v)} exceeds layout capacity {self.cap}")
            codes[self.count_atom.index] = len(cs)
            for a, c in zip(self.slots, cs):
                codes[a.index] = c

    def py_read(self, codes):
        if self.cap is None:
            out = []
            for i, a in enumerate(self.chunks):
                m = codes[a.index]
                out += [self.elem.py_dec(32 * i + j) for j in range(a.bits) if (m >> j) & 1]
            return frozenset(out)
        n = codes[self.count_atom.index]
        return frozenset(self.elem.py_dec(codes[a.index]) for a in self.slots[:n])

    # symbolic
    def enc(self, lw, v):
        if not self.card:
            return super().enc(lw, v)
        if is_const(v):
            return str(self.py_enc(v))
        bm = self._bitmap_exprs(lw, v, 1)[0]
        if self.nonempty:
            lw.trap_unless(SBool(f"({bm} != 0u)"))
            return lw.tmp_int(f"((int){bm} - 1)")
        return bm

    def dec(self, lw, code):
        if not self.card:
            return super().dec(lw, code)
        if self.nonempty:
            code = lw.tmp_uint(f"((unsigned){code} + 1u)")
        return SSet([(SBool(f"(({code} >> {j}) & 1u)"), self.elem.py_dec(j)) for j in range(self.elem.card)], distinct=True)

    def _items(self, lw, v):
        if isinstance(v, frozenset):
            return [(True, x) for x in sorted(v, key=sort_key)]
        if isinstance(v, SSet):
            return v.items
        raise LowerError(f"cannot store {v!r} in a set field")

    def _bitmap_exprs(self, lw, v, nchunks: int) -> list[str]:
        terms: list[list[str]] = [[] for _ in range(nchunks)]
        for g, x in self._items(lw, v):
            if is_const(x):
                try:
                    j = self.elem.py_enc(x)
                except LowerError:
                    lw.trap_unless(lw.b_not(g))
                    continue
                bit = f"{1 << (j % 32)}u"
                terms[j // 32].append(bit if g is True else f"({g.s} ? {bit} : 0u)")
            else:
                c = lw.encode(self.elem, x)
                gs = lw.bstr(g)
                if nchunks == 1:
                    terms[0].append(f"({gs} ? (1u << {c}) : 0u)")
                else:
                    for k in range(nchunks):
                        terms[k].append(f"(({gs} && ({c} >> 5) == {k}) ? (1u << ({c} & 31)) : 0u)")
        return [lw.tmp_uint("(" + " | ".join(t) + ")") if t else "0u" for t in terms]

    def read(self, lw):
        if self.cap is None:
            items = []
            for i, a in enumerate(self.chunks):
                for j in range(a.bits):
                    items.append((SBool(f"((a{a.index} >> {j}) & 1u)"), self.elem.py_dec(32 * i + j)))
            return SSet(items, distinct=True)
        items = []
        for i, a in enumerate(self.slots):
            g = SBool(f"({i} < (int)a{self.count_atom.index})")
            x = self.elem.dec(lw, f"a{a.index}")
            lw.remember_code(self.elem, x, f"a{a.index}")               # re-encoding x is the identity
            items.append((g, x))
        return SSet(items, distinct=True)            # canonical array: sorted, no duplicates

    def write(self, lw, v, out):
        if self.cap is None:
            if is_const(v):
                codes: dict = {}
                self.py_write(v, codes)
                for a in self.chunks:
                    out[a.index] = f"{codes[a.index]}u"
                return
            exprs = self._bitmap_exprs(lw, v, len(self.chunks))
            if self.nonempty:
                lw.trap_unless(lw.b_or([SBool(f"({e} != 0u)") for e in exprs]))
            for a, e in zip(self.chunks, exprs):
                out[a.index] = e
            return
        if is_const(v):
            codes = {}
            self.py_write(v, codes)
            out[self.count_atom.index] = str(codes[self.count_atom.index])
            for a in self.slots:
                out[a.index] = str(codes.get(a.index, 0))
            return
        # canonical sorted array: dedup, rank, scatter  (O(m^2) compares, m = #candidate elements)
        items = self._items(lw, v)
        cs = []
        for _, x in items:
            cs.append(lw.tmp_int(lw.encode(self.elem, x)))
        ps: list[str] = []
        for i, (g, _) in enumerate(items):
            terms = [lw.bstr(g)] + [f"!({ps[j]} && {cs[j]} == {cs[i]})" for j in range(i)]
            ps.append(lw.tmp_bool("(" + " && ".join(terms) + ")"))
        ranks = []
        for i in range(len(items)):
            terms = [f"(int)({ps[j]} && {cs[j]} < {cs[i]})" for j in range(len(items)) if j != i]
            ranks.append(lw.tmp_int("(" + " + ".join(terms) + ")") if terms else "0")
        count = lw.tmp_int("(" + " + ".join(f"(int){p}" for p in ps) + ")") if ps else "0"
        if len(items) > self.cap:
            lw.trap_unless(SBool(f"({count} <= {self.cap})"))
        out[self.count_atom.index] = count
        for r, a in enumerate(self.slots):
            terms = [f"(({ps[i]} && {ranks[i]} == {r}) ? {cs[i]} : 0)" for i in range(len(items))]
            out[a.index] = lw.tmp_int("(" + " | ".join(terms) + ")") if terms else "0"


class TKeyedSet(Ty):
    """Set of records in which the field ``key`` determines the record -- a functional dependency the spec
    maintains and the generated code checks (a second, different record with an existing key traps
    KMC_FAIL_LAYOUT).  One entry per key value: 0 = no record with that key, c + 1 = code c of the other
    fields.  Compared with the sorted array this needs no count, no re-sorting on insert and no division to
    decode, and every element read from it has a CONSTANT key (leaderAndIsrRequests, KafkaReplication.tla:66,
    138-146: every request carries a fresh leaderEpoch)."""

    def __init__(self, elem: "TRec", key: str):
        if not isinstance(elem, TRec) or key not in elem.fields:
            raise LowerError(f"KEYED: the set elements must be records with a field {key}")
        self.elem, self.key = elem, key
        self.key_ty = elem.fields[key]
        self.rest = TRec({f: t for f, t in elem.fields.items() if f != key})
        if not self.key_ty.card or not self.rest.card:
            raise LowerError("KEYED: key and remaining fields must be scalar-codeable")
        self.card = 0
        self.atom = None
        self.entries: list[Atom] = []

    def kind(self):
        return "set"

    def describe(self):
        return {"t": "set", "repr": "keyed", "key": self.key, "elem": self.elem.describe()}

    def alloc(self, lay, path):
        b = bits_for(self.rest.card + 1)
        self.entries = [lay.new_atom(f"{path}#{self.key}={fmt(self.key_ty.py_dec(j))}", b, self.rest.card + 1)
                        for j in range(self.key_ty.card)]

    def _rest_of(self, v):
        if isinstance(v, FnVal):
            return FnVal({f: v.apply(f) for f in self.rest.fields})
        return SRec({f: v.fields[f] for f in self.rest.fields})

    # python
    def py_write(self, v, codes):
        if not isinstance(v, frozenset):
            raise LowerError(f"value {fmt(v)} is not a set")
        for a in self.entries:
            codes[a.index] = 0
        for x in v:
            if not isinstance(x, FnVal) or set(x.domain()) != set(self.elem.fields):
                raise LowerError(f"value {fmt(x)} is not a record with fields {list(self.elem.fields)}")
            a = self.entries[self.key_ty.py_enc(x.apply(self.key))]
            c = self.rest.py_enc(self._rest_of(x)) + 1
            if codes[a.index] not in (0, c):
                raise LowerError(f"two records with {self.key} = {fmt(x.apply(self.key))} in a KEYED set")
            codes[a.index] = c

    def py_read(self, codes):
        out = []
        for j, a in enumerate(self.entries):
            c = codes[a.index]
            if c:
                d = dict(self.rest.py_dec(c - 1).items)
                d[self.key] = self.key_ty.py_dec(j)
                out.append(FnVal({f: d[f] for f in self.elem.fields}))
        return frozenset(out)

    # symbolic
    def _entry_sig(self):
        return "keyed-entry:" + self.rest.sig()

    def read(self, lw):
        items = []
        for j, a in enumerate(self.entries):
            g = SBool(f"(a{a.index} != 0u)")
            rv = self.rest.dec(lw, lw.tmp_int(f"((int)a{a.index} - 1)"))
            d = dict(rv.fields)
            d[self.key] = self.key_ty.py_dec(j)
            x = SRec({f: d[f] for f in self.elem.fields})
            lw.enc_cache[id(x)] = (self._entry_sig(), x, f"a{a.index}", lw.cg.blocks[-1], lw.unit_id)
            items.append((g, x))
        return SSet(items, distinct=True)

    def write(self, lw, v, out):
        if is_const(v):
            codes: dict = {}
            self.py_write(v, codes)
            for a in self.entries:
                out[a.index] = str(codes[a.index])
            return
        if isinstance(v, frozenset):
            items = [(True, x) for x in sorted(v, key=sort_key)]
        elif isinstance(v, SSet):
            items = v.items
        else:
            raise LowerError(f"cannot store {v!r} in a set field")
        contrib: list[list] = [[] for _ in self.entries]          # per entry: (match guard, entry code expr)
        for g, x in items:
            if isinstance(x, SUnion):
                x = lw.narrow_union(x, self.elem.kind())
            kx = x.apply(self.key) if isinstance(x, FnVal) else x.fields[self.key]
            hit = lw._code_hit(x)
            if hit is not None and hit[0] == self._entry_sig():
                code = hit[2]                                     # an element read from this layout: its entry as is
            else:
                code = lw.tmp_int(f"({lw.encode(self.rest, self._rest_of(x))} + 1)")
            if is_const(kx):
                try:
                    js = [(self.key_ty.py_enc(kx), g)]
                except LowerError:
                    lw.trap_unless(lw.b_not(g))
                    continue
            else:
                js = []
                covered = []
                for j in range(self.key_ty.card):
                    m = lw.eq(kx, self.key_ty.py_dec(j))
                    if m is not False:
                        js.append((j, lw.b_and([g, m])))
                        covered.append(m)
                in_range = (isinstance(kx, SInt) and isinstance(self.key_ty, TInt) and
                            self.key_ty.lo <= kx.lo and kx.hi <= self.key_ty.hi)
                if not in_range:
                    lw.trap_unless(lw.b_or([lw.b_not(g)] + covered))   # a key outside the layout's key range
            for j, m in js:
                if m is not False:
                    contrib[j].append((m, code))
        for a, lst in zip(self.entries, contrib):
            for i in range(len(lst)):
                for k in range(i):
                    (m1, c1), (m2, c2) = lst[k], lst[i]
                    if c1 != c2:                                    # two different records with this key: not a function
                        lw.trap_unless(lw.b_not(lw.b_and([m1, m2, SBool(f"({c1} != {c2})")])))
            terms = [c if m is True else f"({lw.bstr(m)} ? {c} : 0)" for m, c in lst]
            out[a.index] = lw.tmp_int("(" + " | ".join(terms) + ")") if terms else "0"


class TPrefixFn(Ty):
    """``[0..n-1 -> X \\union {nil}]`` whose entries are nil exactly at the indexes >= the record's length field
    (FiniteReplicatedLog.tla:84-87 states this as part of TypeOk; the generated code re-checks it whenever a
    record is written).  Only X is stored: ``bits_for(card X)`` per entry, unwritten entries hold 0."""

    def __init__(self, keys: list, inner: Ty, nil, len_field: str):
        import copy
        self.keys = list(keys)
        self.inner = [copy.deepcopy(inner) for _ in keys]
        self.nil, self.len_field = nil, len_field
        self.card = 0
        self.atom = None

    def kind(self):
        return "fn"

    def describe(self):
        return {"t": "prefixfn", "keys": [fmt(k) for k in self.keys], "inner": self.inner[0].describe(),
                "nil": fmt(self.nil), "len": self.len_field}

    def alloc(self, lay, path):
        for k, t in zip(self.keys, self.inner):
            t._alloc_scalar(lay, f"{path}[{fmt(k)}]")

    # python
    def py_write_len(self, v, length, codes):
        if not isinstance(v, FnVal) or set(v.domain()) != set(self.keys):
            raise LowerError(f"function domain mismatch storing {fmt(v)}")
        for k, t in zip(self.keys, self.inner):
            x = v.apply(k)
            is_nil = kind_sig(x) == kind_sig(self.nil) and x == self.nil
            if is_nil != (k >= length):
                raise LowerError(f"PREFIX layout violated: entry {k} of {fmt(v)} with length {length}")
            if t.atom is not None:
                codes[t.atom.index] = 0 if is_nil else t.py_enc(x)

    def py_read_len(self, codes, length):
        return FnVal({k: (t.py_dec(codes[t.atom.index] if t.atom is not None else 0) if k < length else self.nil)
                      for k, t in zip(self.keys, self.inner)})

    def py_write(self, v, codes):
        raise LowerError("internal: TPrefixFn is written through its record")

    def py_read(self, codes):
        raise LowerError("internal: TPrefixFn is read through its record")

    # symbolic
    def read_len(self, lw, length):
        vals = []
        for k, t in zip(self.keys, self.inner):
            g = lw.cmp("<", k, length)
            if t.atom is None:
                x = t.py_dec(0)
            else:
                x = t.dec(lw, f"a{t.atom.index}")
                lw.remember_code(t, x, f"a{t.atom.index}")
            if g is True:
                vals.append(x)
            elif g is False:
                vals.append(self.nil)
            else:
                # same alternative order as TUnion.dec: sorted by kind
                alts = sorted([(lw.b_not(g), self.nil), (g, x)], key=lambda a: kind_sig(a[1]))
                vals.append(SUnion(alts))
        self._read_vals = vals
        return SFn(self.keys, vals)

    def write_len(self, lw, v, newlen, len_changed: bool, out):
        if isinstance(v, FnVal):
            m = dict(v.items)
        elif isinstance(v, SFn):
            m = dict(zip(v.keys, v.vals))
        else:
            raise LowerError(f"cannot store {v!r} in a function layout")
        if set(m) != set(self.keys):
            raise LowerError("function domain mismatch")
        old = getattr(self, "_read_vals", [None] * len(self.keys))
        nil_kind = kind_sig(self.nil)
        for i, (k, t) in enumerate(zip(self.keys, self.inner)):
            x = m[k]
            untouched = x is old[i]
            if untouched and not len_changed:
                continue
            if is_const(x):
                nil_g = kind_sig(x) == nil_kind and x == self.nil
            elif isinstance(x, SUnion):
                nil_g = lw.b_or([lw.b_and([g, lw.eq(a, self.nil)]) for g, a in x.alts if kind_sig(a) == nil_kind])
            else:
                nil_g = False if kind_sig(x) != nil_kind else lw.eq(x, self.nil)
            expect_nil = lw.cmp(">=", k, newlen)
            lw.trap_unless(lw.b_or([lw.b_and([nil_g, expect_nil]), lw.b_and([lw.b_not(nil_g), lw.b_not(expect_nil)])]))
            if untouched or t.atom is None:
                continue
            if nil_g is True:
                out[t.atom.index] = "0"
                continue
            xv = lw.narrow_union(x, t.kind()) if isinstance(x, SUnion) else x
            c = lw.encode(t, xv)
            out[t.atom.index] = c if expect_nil is False else lw.tmp_int(f"({lw.bstr(expect_nil)} ? 0 : {c})")


class TTuple(Ty):
    """Fixed-length tuple <<x1, ..., xn>> (an element of a Cartesian product): one member type per position."""

    def __init__(self, elems: list):
        self.elems = list(elems)
        self.card = 1
        for t in self.elems:
            self.card = self.card * t.card if (t.card and self.card) else 0
        if self.card > (1 << 30):
            self.card = 0
        self.atom = None

    def kind(self):
        return "tuple"

    def describe(self):
        return {"t": "tuple", "elems": [t.describe() for t in self.elems]}

    def alloc(self, lay, path):
        for i, t in enumerate(self.elems):
            t.alloc(lay, f"{path}[{i + 1}]")

    def _items(self, v):
        if isinstance(v, tuple):
            items = list(v)
        elif isinstance(v, SSeq) and is_int_const(v.n):
            items = list(v.items[:v.n])
        else:
            raise LowerError(f"cannot store {v!r} in a tuple of {len(self.elems)}")
        if len(items) != len(self.elems):
            raise LowerError(f"tuple of length {len(items)} stored in a layout of length {len(self.elems)}")
        return items

    def py_enc(self, v):
        code, stride = 0, 1
        for t, x in zip(self.elems, self._items(v)):
            code += t.py_enc(x) * stride
            stride *= t.card
        return code

    def py_dec(self, code):
        out = []
        for t in self.elems:
            out.append(t.py_dec(code % t.card))
            code //= t.card
        return tuple(out)

    def py_write(self, v, codes):
        for t, x in zip(self.elems, self._items(v)):
            t.py_write(x, codes)

    def py_read(self, codes):
        return tuple(t.py_read(codes) for t in self.elems)

    def enc(self, lw, v):
        if is_const(v):
            return str(self.py_enc(v))
        if isinstance(v, SUnion):
            return lw.enc_union_into(self, v)
        terms, stride = [], 1
        for t, x in zip(self.elems, self._items(v)):
            c = lw.encode(t, x)
            terms.append(c if stride == 1 else f"{c} * {stride}")
            stride *= t.card
        return lw.tmp_int("(" + " + ".join(terms) + ")")

    def dec(self, lw, code):
        out, stride = [], 1
        for t in self.elems:
            if t.card == 1:
                out.append(t.py_dec(0))
            else:
                x = code if stride == 1 else f"({code} / {stride})"
                if stride * t.card < self.card:
                    x = f"({x} % {t.card})"
                out.append(t.dec(lw, lw.tmp_int(x)))
            stride *= t.card
        return lw.mk_seq(len(out), out)

    def read(self, lw):
        items = [lw.read_ty(t) for t in self.elems]
        return lw.mk_seq(len(items), items)

    def write(self, lw, v, out):
        if isinstance(v, SUnion):
            v = lw.narrow_union(v, "tuple")
        for t, x in zip(self.elems, self._items(v)):
            if x is lw.read_cache.get(id(t)):
                continue
            t.write(lw, x, out)


class TSeq(Ty):
    """Sequence of at most ``cap`` elements of a scalar-codeable type: length atom + one code atom per slot;
    unused slots hold code 0 (canonical packing).  A longer sequence traps (KMC_E_LAYOUT_OVERFLOW)."""

    def __init__(self, elem: Ty, cap: int | None = None):
        if not elem.card:
            raise LowerError("Seq(S): the element type must be codeable as one integer (scalars, small records)")
        self.elem, self.cap = elem, cap
        self.card = 0
        self.atom = None
        self.len_ty = None
        self.slots: list[Ty] = []

    def set_cap(self, cap: int):
        self.cap = cap
        self._sig = None

    def kind(self):
        return "tuple"

    def describe(self):
        return {"t": "seq", "cap": self.cap, "elem": self.elem.describe()}

    def alloc(self, lay, path):
        import copy
        if self.cap is None:
            raise LowerError(f"{path} \\in Seq(...) needs a bound: add '\\* kspec: CAPACITY {path} = <max length>' to the cfg")
        self.len_ty = TInt(0, self.cap)
        self.len_ty.alloc(lay, f"{path}.len")
        # every slot is ONE atom holding the element's scalar code (mixed radix for records), like the slots of an
        # array set -- not the per-field atoms a top-level record would get
        self.slots = [copy.deepcopy(self.elem) for _ in range(self.cap)]
        for i, t in enumerate(self.slots):
            t._alloc_scalar(lay, f"{path}[{i + 1}]")

    def py_write(self, v, codes):
        if not isinstance(v, tuple) or len(v) > self.cap:
            raise LowerError(f"value {fmt(v)} is not a sequence of at most {self.cap} elements")
        if self.len_ty.atom is not None:
            codes[self.len_ty.atom.index] = len(v)
        for i, t in enumerate(self.slots):
            code = t.py_enc(v[i]) if i < len(v) else 0
            if t.atom is not None:
                codes[t.atom.index] = code

    def py_read(self, codes):
        n = codes[self.len_ty.atom.index] if self.len_ty.atom is not None else 0
        return tuple(t.py_dec(codes[t.atom.index] if t.atom is not None else 0) for t in self.slots[:n])

    def read(self, lw):
        n = lw.read_ty(self.len_ty)
        items = []
        for t in self.slots:
            v = Ty.read(t, lw)                     # scalar read: dec(a<idx>), remembered as that code
            lw.read_cache[id(t)] = v
            items.append(v)
        return lw.mk_seq(n, items)

    def write(self, lw, v, out):
        if isinstance(v, SUnion):
            v = lw.narrow_union(v, "tuple")
        n, items = lw.seq_parts(v)
        if is_int_const(n):
            if n > self.cap:
                lw.trap_unless(False)
                return
        elif n.hi > self.cap:
            lw.trap_unless(lw.cmp("<=", n, self.cap))
        if self.len_ty.atom is not None:
            out[self.len_ty.atom.index] = str(n) if is_int_const(n) else n.s
        for j, t in enumerate(self.slots):
            if t.atom is None:
                continue
            if j >= len(items) or (is_int_const(n) and j >= n):
                out[t.atom.index] = "0"
                continue
            if is_int_const(n):
                out[t.atom.index] = lw.encode(t, items[j])
                continue
            # slot j is live iff j < n; a dead slot packs to 0.  Range traps of a dead item must not fire: its
            # traps are folded into the live condition.
            marks = len(lw.traps)
            code = lw.encode(t, items[j])
            live = lw.cmp(">", n, j)
            new_traps = lw.traps[marks:]
            del lw.traps[marks:]
            for tr in new_traps:
                lw.trap_unless(lw.b_or([lw.b_not(live), tr]))
            if live is True:
                out[t.atom.index] = code
            elif live is False:
                out[t.atom.index] = "0"
            else:
                out[t.atom.index] = lw.tmp_int(f"({live.s} ? {code} : 0)")


def ty_from_description(d: dict) -> Ty:
    """The unallocated layout type whose ``describe()`` is ``d``.  Only for decoding: enum gids are list positions."""
    k = d["t"]
    if k == "int":
        return TInt(d["lo"], d["hi"])
    if k == "bool":
        return TBool()
    if k == "enum":
        vals = [parse_value(x) for x in d["values"]]
        return TEnum(vals, {x: i for i, x in enumerate(vals)})
    if k == "rec":
        return TRec({f: ty_from_description(fd) for f, fd in d["fields"].items()})
    if k == "fn":           # one type per key: every element allocates its own atoms
        return TFn([parse_value(x) for x in d["keys"]], [ty_from_description(d["elem"]) for _ in d["keys"]])
    if k == "prefixfn":
        return TPrefixFn([parse_value(x) for x in d["keys"]], ty_from_description(d["inner"]), parse_value(d["nil"]),
                         d["len"])
    if k == "tuple":
        return TTuple([ty_from_description(e) for e in d["elems"]])
    if k == "union":
        return TUnion([ty_from_description(a) for a in d["alts"]])
    if k == "set":
        if d["repr"] == "keyed":
            return TKeyedSet(ty_from_description(d["elem"]), d["key"])
        return TSet(ty_from_description(d["elem"]), d.get("cap"), d.get("nonempty", False))
    if k == "seq":
        return TSeq(ty_from_description(d["elem"]), d["cap"])
    raise LowerError(f"layout description has an unknown type {k!r}")
