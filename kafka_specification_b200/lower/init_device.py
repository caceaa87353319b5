"""The device form of Init: initial states decoded from a candidate index and filtered on the GPU.

TLC computes the initial states by enumerating Init on one thread, and the host form of the lowering (model.py,
``_init_states``) does the same at lowering time: fine for the one-state Inits of the Kafka specs, out of reach for an
Init written as ``v \\in S`` over a type (TLC's inductive-invariant check, ``INIT TypeOk /\\ Inv``).

The device form splits Init into branches, one per alternative of every ``\\/`` in conjunct position (the same walk as
the host form: ``/\\``, ``\\/``, ``LET``, operator calls, ``\\E``).  A branch has, in source order:

* generators   ``v \\in S`` for a variable not assigned yet, and the bound variables of ``\\E x \\in S``;
* fixed assignments ``v = e``;
* filters      every other conjunct.

S must be a constant set of a form that decodes from an index without being materialised (``decode``): the candidate
space of a branch is the mixed-radix product of its generators' cardinalities.  ``init_candidate(b, idx, out, fail)``
decodes candidate ``idx`` of branch ``b`` into symbolic values, runs the filters (each one returns false as soon as it
fails, before anything is packed, so that a rejected candidate never traps the layout) and packs the survivor with the
same layout traps as a successor.  Every solution of every branch is one generated initial state, duplicates
included, as in TLC.
"""
from __future__ import annotations

from ..frontend.values import sort_key
from .compiler import CG, Closure, Marker, UnpinnedRef, render
from .compiler import expr_text as _text
from .svals import LowerError, SBool, SFn, SInt, SLazy, SRec, SSet, c_int, fits_int, is_const, is_int_const, kind_sig

INIT_DEVICE_THRESHOLD = 65536          # Init candidates above which Init is enumerated on the GPU without the cfg hint
MAX_BRANCH_CANDIDATES = 1 << 40        # candidate space of one branch (~10^12): beyond it the device form is refused


class DeviceInit:
    """Shape (branches, cardinalities) and generated code of the device form of one Init."""

    def __init__(self, lw, init_e):
        self.lw = lw
        self.branches: list[list[tuple]] = []
        self._walk([(init_e, lw.root, None, {})], [], frozenset())
        self.spaces = [self._space(b) for b in self.branches]
        self.candidates = sum(self.spaces)

    # ------------------------------------------------------------------ shape
    def _const_set(self, sexpr, ctx, fm, env, conj):
        try:
            s = self.lw.ev(sexpr, ctx, fm, env, None)
        except UnpinnedRef:
            raise LowerError(f"Init conjunct '{_text(conj)}': its generator set depends on a bound variable") from None
        except LowerError as err:
            if "constant context" in str(err):
                raise LowerError(f"Init conjunct '{_text(conj)}': its generator set depends on a state variable") from None
            raise
        self.card(s, conj)
        return s

    def _walk(self, items, prefix: list, assigned: frozenset):
        lw = self.lw
        if not items:
            for v in lw.variables:
                if v not in assigned:
                    raise LowerError(f"Init leaves {v} unassigned")
            self.branches.append(prefix)
            return
        (e, ctx, fm, env), rest = items[0], items[1:]
        k = e[0]
        if k == "and":
            self._walk([(x, ctx, fm, env) for x in e[1]] + rest, prefix, assigned)
            return
        if k == "or":
            for x in e[1]:
                self._walk([(x, ctx, fm, env)] + rest, prefix, assigned)
            return
        if k == "quant" and e[1] == "E":
            env2, gens = dict(env), []
            for names, sexpr in e[2]:
                s = self._const_set(sexpr, ctx, fm, env, e)
                for n in names:
                    m = Marker(n, s)
                    env2[n] = m
                    gens.append(("gen", m, s, e))
            self._walk([(e[3], ctx, fm, env2)] + rest, prefix + gens, assigned)
            return
        if k == "let":
            self._walk([(e[2], ctx, fm, lw.let_env(e[1], ctx, fm, env))] + rest, prefix, assigned)
            return
        if k in ("id", "app", "inst"):
            op = None
            if not (k == "id" and e[1] in env and not isinstance(env[e[1]], Closure)):
                op = lw.find_operator(e, ctx, fm, env)
            if op is not None:
                target, defctx, args = op
                self._walk([lw.bind_call(target, defctx, args, ctx, fm, env)] + rest, prefix, assigned)
                return
        if k == "binop" and e[1] in ("=", "\\in"):
            v = lw.resolve_var(e[2], ctx, fm, env)
            if v is not None and v not in assigned:
                if e[1] == "=":
                    item = ("fix", v, (e[3], ctx, fm, env), e)
                else:
                    item = ("gen", v, self._const_set(e[3], ctx, fm, env, e), e)
                self._walk(rest, prefix + [item], assigned | {v})
                return
        self._walk(rest, prefix + [("filter", (e, ctx, fm, env), e)], assigned)

    def _space(self, branch) -> int:
        n = 1
        for it in branch:
            if it[0] == "gen":
                n *= self.card(it[2], it[3])
        if n > MAX_BRANCH_CANDIDATES:
            raise LowerError(f"an Init branch has {n:,} candidates, more than the device form enumerates "
                             f"({MAX_BRANCH_CANDIDATES:,})")
        return n

    # ------------------------------------------------------------------ digits
    def _parts(self, s) -> list:
        """The operands of a (nested) lazy union."""
        if isinstance(s, SLazy) and s.kind == "union":
            return self._parts(s.a) + self._parts(s.b)
        return [s]

    def _kinds(self, s, conj) -> set:
        if isinstance(s, frozenset):
            return {kind_sig(x) for x in s}
        if s.kind == "recset":
            return {"rec:" + ",".join(sorted(s.a))}
        if s.kind == "fnset":
            dom = [x for _, x in self.lw.set_items(s.a)]
            return {"rec:" + ",".join(sorted(dom))} if dom and all(isinstance(x, str) for x in dom) else {"fn"}
        if s.kind == "powerset":
            return {"set"}
        if s.kind == "cross":
            return {"tuple"}
        if s.kind == "range":
            return {"int"}
        raise LowerError(f"Init conjunct '{_text(conj)}': cannot decode a generator over {s.kind}")

    def card(self, s, conj) -> int:
        """Members of the constant set s, computed from its form (never enumerated unless it is a leaf)."""
        if isinstance(s, frozenset):
            return len(s)
        if not isinstance(s, SLazy):
            raise LowerError(f"Init conjunct '{_text(conj)}': the generator set is not a constant set")
        if s.kind == "range" and is_int_const(s.a) and is_int_const(s.b):
            return max(0, s.b - s.a + 1)
        if s.kind in ("nat", "int", "seq"):
            name = {"nat": "Nat", "int": "Int", "seq": "Seq(S)"}[s.kind]
            raise LowerError(f"Init conjunct '{_text(conj)}': a generator over {name} is unbounded")
        if s.kind == "recset":
            n = 1
            for f in s.a.values():
                n *= self.card(f, conj)
            return n
        if s.kind == "fnset":
            dom = self.lw.set_items(s.a)
            if any(g is not True or not is_const(x) for g, x in dom):
                raise LowerError(f"Init conjunct '{_text(conj)}': a function set over a non-constant domain")
            return self.card(s.b, conj) ** len(dom)
        if s.kind == "powerset":
            base = self._base(s, conj)
            return 1 << len(base)
        if s.kind == "cross":
            n = 1
            for p in s.a:
                n *= self.card(p, conj)
            return n
        if s.kind == "union":
            parts = self._parts(s)
            seen: set = set()
            for p in parts:
                ks = self._kinds(p, conj)
                if ks & seen:
                    raise LowerError(f"Init conjunct '{_text(conj)}': a union of sets of the same kind "
                                     f"({', '.join(sorted(ks & seen))}) may overlap; write it as one set")
                seen |= ks
            return sum(self.card(p, conj) for p in parts)
        raise LowerError(f"Init conjunct '{_text(conj)}': cannot decode a generator over {s.kind}")

    def _base(self, s, conj) -> list:
        items = self.lw.set_items(s.a)
        if any(g is not True or not is_const(x) for g, x in items):
            raise LowerError(f"Init conjunct '{_text(conj)}': SUBSET of a non-constant set")
        if len(items) > 62:
            raise LowerError(f"Init conjunct '{_text(conj)}': SUBSET of {len(items)} elements")
        return [x for _, x in items]

    def _digit(self, x: str, stride: int, radix: int, total: int) -> str:
        """Digit (x / stride) % radix of an index x in [0, total), in the narrowest unsigned type: the divisors are
        constants, so the compiler turns each division into a multiply and a shift."""
        narrow = total <= (1 << 32)
        sfx = "u" if narrow else "ull"
        if narrow and x == "idx":
            x = "(unsigned)idx"
        e = x if stride == 1 else f"{x} / {stride}{sfx}"
        if stride * radix < total:
            e = f"({e}) % {radix}{sfx}" if stride != 1 else f"{x} % {radix}{sfx}"
        ctype = "unsigned" if radix <= (1 << 32) else "uint64_t"
        return self.lw.cg.tmp(ctype, f"({ctype})({e})")

    def _int_range(self, x: str, lo: int, hi: int) -> SInt:
        """Member number x of lo .. hi: in `int` arithmetic where the members and x fit one, else in `int64_t`."""
        if fits_int(lo, hi) and hi - lo <= (1 << 31) - 1:
            e = f"((int){x} + {lo})" if lo else f"(int){x}"
        else:
            e = f"((int64_t){x} + {c_int(lo)})" if lo else f"(int64_t){x}"
        return SInt(self.lw.tmp_int(e, lo, hi), lo, hi)

    def decode(self, s, x: str, conj):
        """The symbolic member number x (a C expression in [0, card(s))) of the constant set s."""
        lw = self.lw
        n = self.card(s, conj)
        if isinstance(s, frozenset):
            items = sorted(s, key=sort_key)
            if len(items) == 1:
                return items[0]
            if all(is_int_const(v) for v in items) and items[-1] - items[0] + 1 == len(items):
                return self._int_range(x, items[0], items[-1])
            res = items[-1]
            for i in range(len(items) - 2, -1, -1):
                res = lw.mux(SBool(lw.tmp_bool(f"({x} == {i}u)")), items[i], res)
            return res
        if s.kind == "range":
            return self._int_range(x, s.a, s.b)
        if s.kind in ("recset", "cross"):
            parts = list(s.a.values()) if s.kind == "recset" else list(s.a)
            vals, stride = [], 1
            for p in parts:
                c = self.card(p, conj)
                vals.append(self.decode(p, self._digit(x, stride, c, n), conj))
                stride *= c
            if s.kind == "recset":
                return SRec(dict(zip(s.a, vals)))
            return lw.mk_seq(len(vals), vals)
        if s.kind == "fnset":
            keys = sorted((k for _, k in lw.set_items(s.a)), key=sort_key)
            c = self.card(s.b, conj)
            vals = [self.decode(s.b, self._digit(x, c ** i, c, n), conj) for i in range(len(keys))]
            if keys and all(isinstance(k, str) for k in keys):
                return SRec(dict(zip(keys, vals)))
            return SFn(keys, vals)
        if s.kind == "powerset":
            base = self._base(s, conj)
            return SSet([(SBool(f"(((({x}) >> {i}) & 1u) != 0u)"), e) for i, e in enumerate(base)], distinct=True)
        # union of parts of disjoint kinds: part i holds the indices [off_i, off_i + card_i)
        parts = self._parts(s)
        offs, off = [], 0
        for p in parts:
            offs.append(off)
            off += self.card(p, conj)
        ctype, sfx = ("unsigned", "u") if n <= (1 << 32) else ("uint64_t", "ull")
        res = self.decode(parts[-1], lw.cg.tmp(ctype, f"{x} - {offs[-1]}{sfx}") if offs[-1] else x, conj)
        for i in range(len(parts) - 2, -1, -1):
            sub = lw.cg.tmp(ctype, f"{x} - {offs[i]}{sfx}") if offs[i] else x
            res = lw.mux(SBool(lw.tmp_bool(f"({x} < {offs[i + 1]}{sfx})")), self.decode(parts[i], sub, conj), res)
        return res

    # ------------------------------------------------------------------ code
    def _branch_lines(self, b: int) -> list[str]:
        lw, lay = self.lw, self.lw.layout
        branch, space = self.branches[b], self.spaces[b]
        lw.cg = CG()
        lw.read_cache, lw.enc_cache, lw.mux_origin = {}, {}, {}
        lw.unit_id = 0
        lw.traps = []
        state: dict = {}
        lw.cur = state
        stride = 1
        for it in branch:
            if it[0] == "gen":
                c = self.card(it[2], it[3])
                val = self.decode(it[2], self._digit("idx", stride, c, space), it[3])
                stride *= c
                if isinstance(it[1], Marker):
                    it[1].value, it[1].bound = val, True
                else:
                    state[it[1]] = val
            elif it[0] == "fix":
                e, ctx, fm, env = it[2]
                try:
                    state[it[1]] = lw.ev(e, ctx, fm, env, state)
                except (LowerError, UnpinnedRef) as err:
                    raise LowerError(f"Init conjunct '{_text(it[3])}': {err}") from None
            else:
                e, ctx, fm, env = it[1]
                try:
                    c = lw.ev_bool(e, ctx, fm, env, state)
                except (LowerError, UnpinnedRef) as err:
                    raise LowerError(f"Init conjunct '{_text(it[2])}': {err}") from None
                if c is False:
                    lw.cg.emit("return false;")
                    break
                if c is not True:
                    lw.cg.emit(f"if (!({c.s})) return false;")
        else:
            out: dict[int, str] = {}
            for v in lw.variables:
                lay.var_types[v].write(lw, state[v], out)
            ok = lw.b_and(lw.traps)
            lw.traps = []
            if ok is False:
                lw.cg.emit("fail = KMC_FAIL_LAYOUT;")
                lw.cg.emit("return false;")
            else:
                if ok is not True:
                    lw.cg.emit(f"if (!({ok.s})) {{ fail = KMC_FAIL_LAYOUT; return false; }}")
                by_word: dict[int, list] = {}
                for idx, code in out.items():
                    a = lay.atoms[idx]
                    by_word.setdefault(a.word, []).append(
                        f"((uint64_t)({code}) << {a.shift})" if a.shift else f"(uint64_t)({code})")
                for w in range(lay.words):
                    lw.cg.emit(f"out.w[{w}] = " + (" | ".join(by_word[w]) if w in by_word else "0ull") + ";")
                lw.cg.emit("return true;")
        for it in branch:
            if it[0] == "gen" and isinstance(it[1], Marker):
                it[1].value, it[1].bound = None, False
        return render(lw.cg.body.children, 1)

    def emit(self) -> list[str]:
        """The header section of the device form: HAS_DEVICE_INIT, INIT_BRANCHES, INIT_SPACE and init_candidate()."""
        lw = self.lw
        saved_cache = lw._const_cache
        lines = [
            "/* Init, device form: candidate idx < INIT_SPACE[b] of branch b decodes into one assignment of the branch's",
            "   generators; init_candidate() returns true and packs it into `out` iff it satisfies the branch's filters, and",
            "   sets `fail` when a solution does not fit the packed layout.  NUM_INIT is 0 and INIT_STATES is never read. */",
            "static const uint64_t INIT_STATES[1][W] = {{0}};",
            "#define KMC_HAS_DEVICE_INIT 1",
            "static constexpr bool HAS_DEVICE_INIT = true;",
            f"static constexpr int INIT_BRANCHES = {len(self.branches)};",
            f"static constexpr uint64_t INIT_CANDIDATES = {self.candidates}ull;",
            "static constexpr uint64_t INIT_SPACE[INIT_BRANCHES] = {" + ", ".join(f"{n}ull" for n in self.spaces) + "};",
        ]
        for b in range(len(self.branches)):
            lw._const_cache = dict(saved_cache)        # values cached in one branch may depend on its state
            saved_thunks, lw._spec_thunks = lw._spec_thunks, []
            try:
                body = self._branch_lines(b)
            finally:
                for t in lw._spec_thunks:
                    t.done, t.val = False, None
                lw._spec_thunks = saved_thunks
            lines.append(f"KMC_HD bool init_candidate_{b}(uint64_t idx, State& out, unsigned& fail) {{")
            lines.append("  (void)idx; (void)out; (void)fail;")
            lines.extend(body)
            lines.append("}")
        lw._const_cache = saved_cache
        lw.cur = None
        lines.append("KMC_HD bool init_candidate(int b, uint64_t idx, State& out, unsigned& fail) {")
        lines.append("  switch (b) {")
        for b in range(len(self.branches)):
            lines.append(f"    case {b}: return init_candidate_{b}(idx, out, fail);")
        lines.append("    default: return false;")
        lines.append("  }")
        lines.append("}")
        return lines

    def describe(self) -> dict:
        return {"device": True, "candidates": self.candidates,
                "branches": [{"space": n, "generators": sum(it[0] == "gen" for it in br)}
                             for n, br in zip(self.spaces, self.branches)]}


def device_init(lw, init_e, cfg) -> DeviceInit | None:
    """The device form of Init when the cfg asks for it (``\\* kspec: INIT DEVICE``) or when Init has more than
    INIT_DEVICE_THRESHOLD candidates; None (the host table) otherwise.  Without the hint, an Init whose shape the device
    form refuses stays with the host form, which reports its own errors."""
    gids, warnings = dict(lw.gids), list(lw.warnings)
    saved_thunks, lw._spec_thunks = lw._spec_thunks, []
    try:
        d = DeviceInit(lw, init_e)
    except (LowerError, UnpinnedRef) as err:
        if cfg.init_device:
            raise LowerError(str(err)) from None
        d = None
    finally:
        for t in lw._spec_thunks:
            t.done, t.val = False, None
        lw._spec_thunks = saved_thunks
    if d is not None and (cfg.init_device or d.candidates > INIT_DEVICE_THRESHOLD):
        return d
    lw.gids.clear()
    lw.gids.update(gids)            # the host form interns atoms in its own order: its header must not change
    lw.warnings[:] = warnings
    return None
