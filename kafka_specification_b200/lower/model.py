"""Lowering driver: ``Module.tla`` + ``Module.cfg``  ->  ``LoweredModel`` (C++ header + layout).

The header is the "CUDA-side switch table" of the hot path: ``expand`` evaluates every ``Next``
disjunct/binding of the spec on one packed state and hands each successor to a sink,
``first_violated_invariant`` / ``in_model`` evaluate the cfg's INVARIANTs / CONSTRAINTs.  The same
header compiles for the device (engine kernels) and for the host (init-state packing checks and
the CPU-side self-tests of the lowering).
"""
from __future__ import annotations

import copy
import hashlib
import json
from dataclasses import dataclass, field

from ..frontend.cfg import Config, ModelValue, parse_cfg
from ..frontend.modules import ModuleContext, load_root
from ..frontend.tla_parser import parse_expression_text
from ..frontend.values import FnVal, fmt, sort_key
from . import layout as L
from .compiler import Block, Closure, Lowerer, Marker, Thunk, render
from .init_device import device_init
from .svals import LowerError, SLazy, is_atom_const, is_const, is_int_const

LOWERING_VERSION = 3
MAX_MASK_INVARIANTS = 64       # violated_invariants() returns one bit per INVARIANT
MAX_WORDS = 7                  # widest packed state the expand kernel's shared-memory tile holds (kmc_engine.cu, SPT)


@dataclass
class LoweredModel:
    name: str
    module: str
    header: str
    layout: dict
    words: int
    state_bits: int
    init_states: list[list[int]]
    actions: list[dict]
    invariants: list[str]
    constraints: list[str]
    check_deadlock: bool
    max_fanout: int
    warnings: list[str] = field(default_factory=list)
    digest: str = ""
    lowerer: object = None
    variables: list[str] = field(default_factory=list)
    sites: list[dict] = field(default_factory=list)     # per emit site: {"action": index into actions, -1 = trap only}
    init: dict = field(default_factory=dict)            # the initial predicate: name, module and source span
    invariants_header: str = ""                         # invariants.h: violated_invariants(), compiled after the header


    def meta(self) -> dict:
        return {
            "name": self.name, "module": self.module, "words": self.words, "state_bits": self.state_bits,
            "init_states": [[str(w) for w in s] for s in self.init_states],
            "actions": self.actions, "invariants": self.invariants, "constraints": self.constraints,
            "check_deadlock": self.check_deadlock, "max_fanout": self.max_fanout,
            "layout": self.layout, "digest": self.digest, "warnings": self.warnings,
            "lowering_version": LOWERING_VERSION, "sites": self.sites, "init": self.init,
        }

    def decode_state(self, words) -> dict:
        return self.lowerer.layout.py_unpack(words)

    def state_text(self, words) -> str:
        st = self.decode_state(words)
        return "\n".join(f"/\\ {v} = {fmt(st[v])}" for v in self.variables)


# ---------------------------------------------------------------------------
# layout inference
# ---------------------------------------------------------------------------
class TypeInference:
    def __init__(self, lw: Lowerer):
        self.lw = lw
        self.found: dict[str, list] = {}     # var -> [(steps, Ty)]
        self.seq_caps: dict[str, int] = {}   # var -> bound from a conjunct `Len(var) <= e` / `Len(var) < e` of the layout operator

    def type_from_setval(self, v) -> L.Ty:
        lw = self.lw
        if isinstance(v, SLazy):
            if v.kind == "range" and is_int_const(v.a) and is_int_const(v.b):
                return L.TInt(v.a, v.b)
            if v.kind == "recset":
                return L.TRec({f: self.type_from_setval(s) for f, s in v.a.items()})
            if v.kind == "fnset":
                keys = sorted((x for _, x in lw.set_items(v.a)), key=sort_key)
                elem = self.type_from_setval(v.b)
                return L.TFn(keys, [copy.deepcopy(elem) for _ in keys])
            if v.kind == "powerset":
                return L.TSet(self.type_from_setval(v.a))
            if v.kind == "union":
                return self.merge(self.type_from_setval(v.a), self.type_from_setval(v.b))
            if v.kind == "seq":
                return L.TSeq(self.type_from_setval(v.a))          # the bound comes from the cfg's CAPACITY hint
            if v.kind == "cross":
                return L.TTuple([self.type_from_setval(p) for p in v.a])
            raise LowerError(f"unbounded set {v.kind} in a layout type: give the variable a bounded "
                             f"type through a '\\* kspec: LAYOUT Op' operator")
        if not isinstance(v, frozenset):
            raise LowerError(f"layout type is not a constant set: {v!r}")
        if not v:
            raise LowerError("empty set used as a layout type")
        bools = [x for x in v if isinstance(x, bool)]
        ints = [x for x in v if is_int_const(x)]
        atoms = [x for x in v if is_atom_const(x)]
        recs = [x for x in v if isinstance(x, FnVal)]
        sets = [x for x in v if isinstance(x, frozenset)]
        tups = [x for x in v if isinstance(x, tuple)]
        parts: list[L.Ty] = []
        if tups:
            if len({len(t) for t in tups}) != 1:
                raise LowerError("layout type mixes tuples of different lengths (use Seq(S) with a CAPACITY hint)")
            parts.append(L.TTuple([self.type_from_setval(frozenset(t[i] for t in tups)) for i in range(len(tups[0]))]))
        if bools:
            parts.append(L.TBool())
        if ints:
            parts.append(L.TInt(min(ints), max(ints)))
        if atoms:
            for a in atoms:
                lw.gid(a)
            parts.append(L.TEnum(atoms, lw.gids))
        if recs:
            doms = {frozenset(r.domain()) for r in recs}
            if len(doms) != 1:
                raise LowerError("layout type mixes records/functions with different domains")
            dom = sorted(next(iter(doms)), key=sort_key)
            if all(isinstance(k, str) for k in dom):
                parts.append(L.TRec({f: self.type_from_setval(frozenset(r.apply(f) for r in recs)) for f in dom}))
            else:
                parts.append(L.TFn(dom, [self.type_from_setval(frozenset(r.apply(k) for r in recs)) for k in dom]))
        if sets:
            universe = frozenset().union(*sets)
            parts.append(L.TSet(self.type_from_setval(universe), nonempty=frozenset() not in sets))
        if len(bools) + len(ints) + len(atoms) + len(recs) + len(sets) + len(tups) != len(v):
            raise LowerError("unsupported element kind in a layout type")
        return parts[0] if len(parts) == 1 else L.TUnion(sorted(parts, key=lambda t: t.kind()))

    def merge(self, a: L.Ty, b: L.Ty) -> L.Ty:
        if isinstance(a, L.TInt) and isinstance(b, L.TInt):
            return L.TInt(min(a.lo, b.lo), max(a.hi, b.hi))
        if isinstance(a, L.TEnum) and isinstance(b, L.TEnum):
            return L.TEnum(list(dict.fromkeys(a.atoms + b.atoms)), self.lw.gids)
        alts = []
        for t in (a, b):
            alts.extend(t.alts if isinstance(t, L.TUnion) else [t])
        merged: dict[str, L.Ty] = {}
        for t in alts:
            k = t.kind()
            if k in merged:
                if k in ("int", "atom"):
                    merged[k] = self.merge(merged[k], t)
                else:
                    raise LowerError(f"cannot merge two layout alternatives of kind {k}")
            else:
                merged[k] = t
        out = sorted(merged.values(), key=lambda t: t.kind())
        return out[0] if len(out) == 1 else L.TUnion(out)

    def as_path(self, e, ctx, fm, env):
        lw = self.lw
        k = e[0]
        if k == "id":
            if e[1] in env:
                v = env[e[1]]
                if isinstance(v, Thunk):
                    return self.as_path(v.expr, v.ctx, v.fm, v.env)
                return None
            r = ctx.resolve(e[1], fm)
            if r is None:
                return None
            if r.kind == "var":
                return (e[1], [])
            if r.kind == "subst":
                return self.as_path(r.expr, r.ctx, r.from_module, {})
            return None
        if k == "fnapp" and len(e[2]) == 1:
            base = self.as_path(e[1], ctx, fm, env)
            if base is None:
                return None
            try:
                idx = lw.ev(e[2][0], ctx, fm, env, None)
            except LowerError:
                return None
            if not is_const(idx):
                return None
            return (base[0], base[1] + [("idx", idx)])
        if k == "dot":
            base = self.as_path(e[1], ctx, fm, env)
            if base is None:
                return None
            return (base[0], base[1] + [("fld", e[2])])
        return None

    def collect(self, e, ctx, fm, env):
        lw = self.lw
        k = e[0]
        if k == "and":
            for x in e[1]:
                self.collect(x, ctx, fm, env)
            return
        if k == "let":
            self.collect(e[2], ctx, fm, lw.let_env(e[1], ctx, fm, env))
            return
        if k == "quant" and e[1] == "A":
            try:
                binds = lw.bindings(e[2], ctx, fm, env, None)
            except LowerError:
                return                      # state-dependent domain: not a type conjunct
            for g, env2 in binds:
                if g is True:
                    self.collect(e[3], ctx, fm, env2)
            return
        if k in ("id", "app", "inst"):
            op = None
            if not (k == "id" and e[1] in env and not isinstance(env[e[1]], Closure)):
                try:
                    op = lw.find_operator(e, ctx, fm, env)
                except LowerError:
                    op = None
            if op is not None:
                target, defctx, args = op
                body, c2, fm2, env2 = lw.bind_call(target, defctx, args, ctx, fm, env)
                self.collect(body, c2, fm2, env2)
            return
        if k == "binop" and e[1] in ("<=", "<") and e[2][0] == "app" and e[2][1] == "Len" and len(e[2][2]) == 1:
            # `Len(v) <= N` next to `v \in Seq(S)` in the type invariant bounds the sequence's layout (a checked bound,
            # like an explicit `\* kspec: CAPACITY v = N`, which takes precedence)
            p = self.as_path(e[2][2][0], ctx, fm, env)
            if p is not None and not p[1]:
                try:
                    bound = lw.ev(e[3], ctx, fm, env, None)
                except LowerError:
                    return
                if is_int_const(bound):
                    cap = bound if e[1] == "<=" else bound - 1
                    self.seq_caps[p[0]] = min(cap, self.seq_caps.get(p[0], cap))
            return
        if k == "binop" and e[1] in ("\\in", "\\subseteq"):
            p = self.as_path(e[2], ctx, fm, env)
            if p is None:
                return
            try:
                sv = lw.ev(e[3], ctx, fm, env, None)
            except LowerError:
                return
            ty = self.type_from_setval(sv)
            if e[1] == "\\subseteq":
                ty = L.TSet(ty)
            self.found.setdefault(p[0], []).append((p[1], ty))

    def variable_type(self, var: str) -> L.Ty:
        cons = self.found.get(var, [])
        whole = [t for steps, t in cons if not steps]
        if whole:
            return whole[0]
        by_key: dict = {}
        for steps, t in cons:
            if len(steps) == 1 and steps[0][0] == "idx":
                by_key.setdefault(steps[0][1], t)
        if by_key:
            keys = sorted(by_key, key=sort_key)
            return L.TFn(keys, [by_key[k] for k in keys])
        raise LowerError(
            f"no layout type found for variable {var}: the layout operator must contain a conjunct "
            f"'{var} \\in <finite type set>' (or '\\subseteq')")



# ---------------------------------------------------------------------------
# guard/body decomposition of the emitted units ("items")
# ---------------------------------------------------------------------------
def _prune(nodes: list) -> list:
    """A copy of the tree without its empty blocks (e.g. statically dead disjuncts)."""
    out = []
    for n in nodes:
        if isinstance(n, Block):
            kids = _prune(n.children)
            if not kids:
                continue
            n = Block(n.head, n.cond, n.label, kids)
        out.append(n)
    return out


def _split_unit(nodes: list, max_blocks: int) -> list[list]:
    """Cuts a pruned unit with many top-level blocks (e.g. an enumeration over an 80-element bitmap set) into
    sub-units of at most ``max_blocks`` blocks; the unit's root-level temporaries are pure and are
    replicated in every sub-unit."""
    temps = [n for n in nodes if not isinstance(n, Block)]
    blocks = [n for n in nodes if isinstance(n, Block)]
    return [temps + blocks[i:i + max_blocks] for i in range(0, len(blocks), max_blocks)]


def _site_core(n: Block) -> Block | None:
    """The core of the emit site that block ``n`` is, or None.  A site is a core, or else a bare block (one disjunct
    of an `\\/`) holding only temporaries and one core that emits without a layout check: such a block is a site
    as a whole and its body keeps the block.  The kip101 and kip279 models have such blocks, and their generated
    headers (hence their device code) are cut this way."""
    if n.label is not None:
        return n
    blocks = [k for k in n.children if isinstance(k, Block)]
    if n.head or len(blocks) != 1:
        return None
    core = blocks[0]
    unchecked = core.label is not None and core.label >= 0 and not any(isinstance(k, Block) for k in core.children)
    return core if unchecked else None


def _unit_sites(nodes: list):
    """Splits one pruned unit into emit sites, one per core.  Returns (guard_tree, sites):

    * ``guard_tree`` is the unit's own code with every site's block replaced by its site index k (within the
      unit); rendered by ``_render_guard`` it evaluates, for one state, the COMPLETE path condition of every site
      (all the `if`s between the unit root and the site), sharing the common prefixes exactly as expand() does;
    * ``sites[k]`` = (action label of its core, body lines) of site k.  The body is the (pure, hence safely
      speculated) temporaries of the blocks on its path, flattened, followed by the site's block.  It does not
      re-check the path condition: it is run only for (state, site) pairs whose mask bit is set.
    """
    sites: list[tuple[int, list[str]]] = []

    def walk(ns: list, path_temps: list[str]) -> list:
        out: list = []
        temps_here: list[str] = []
        for n in ns:
            if not isinstance(n, Block):
                temps_here.append(n)
                out.append(n)
            elif (core := _site_core(n)) is not None:
                out.append(len(sites))
                sites.append((core.label, render(path_temps + temps_here, 1) + render([n], 1)))
            else:
                out.append(Block(n.head, n.cond, None, walk(n.children, path_temps + temps_here)))
        return out

    return walk(nodes, []), sites


def _render_guard(tree: list, lo: int, hi: int, bit0: int) -> list[str]:
    """Guard code of the sites lo <= k < hi of one unit: site k sets mask bit (bit0 + k - lo).  Blocks without a
    site in the window are dropped; temporaries stay (the C++ compiler removes the unused ones)."""
    def prune(ns):
        out, live = [], False
        for n in ns:
            if isinstance(n, Block):
                sub, sub_live = prune(n.children)
                if sub_live:
                    out.append(Block(n.head, n.cond, None, sub))
                    live = True
            elif isinstance(n, int):
                if lo <= n < hi:
                    out.append(f"m |= 1ull << {bit0 + n - lo};")
                    live = True
            else:
                out.append(n)
        return out, live

    nodes, live = prune(tree)
    return render(nodes, 2) if live else []


# ---------------------------------------------------------------------------
def _init_states(lw: Lowerer, init_expr) -> list[dict]:
    out: list[dict] = []

    def rec(items, st):
        lw.cur = st                 # what an operator argument or a LET definition reads when it is forced
        if not items:
            for v in lw.variables:
                if v not in st:
                    raise LowerError(f"Init leaves {v} unassigned")
            out.append(st)
            return
        (e, ctx, fm, env), rest = items[0], items[1:]
        k = e[0]
        if k == "and":
            rec([(x, ctx, fm, env) for x in e[1]] + rest, st)
            return
        if k == "or":
            for x in e[1]:
                rec([(x, ctx, fm, env)] + rest, st)
            return
        if k == "quant" and e[1] == "E":
            for g, env2 in lw.bindings(e[2], ctx, fm, env, st):
                if g is not True:
                    raise LowerError("Init quantifies over a non-constant set")
                rec([(e[3], ctx, fm, env2)] + rest, st)
            return
        if k == "let":
            rec([(e[2], ctx, fm, lw.let_env(e[1], ctx, fm, env))] + rest, st)
            return
        if k in ("id", "app", "inst"):
            op = None
            if not (k == "id" and e[1] in env and not isinstance(env[e[1]], Closure)):
                op = lw.find_operator(e, ctx, fm, env)
            if op is not None:
                target, defctx, args = op
                rec([lw.bind_call(target, defctx, args, ctx, fm, env)] + rest, st)
                return
        if k == "binop" and e[1] in ("=", "\\in"):
            v = lw.resolve_var(e[2], ctx, fm, env)
            if v is not None and v not in st:
                rhs = lw.ev(e[3], ctx, fm, env, st)
                if e[1] == "=":
                    if not is_const(rhs):
                        raise LowerError(f"Init value of {v} is not a constant")
                    rec(rest, {**st, v: rhs})
                else:
                    for g, x in lw.set_items(rhs):
                        rec(rest, {**st, v: x})
                return
        c = lw.ev_bool(e, ctx, fm, env, st)
        if c is True:
            rec(rest, st)
        elif c is not False:
            raise LowerError("Init contains a non-constant condition")

    rec([(init_expr, lw.root, None, {})], {})
    lw.cur = None
    return out


def _init_info(lw: Lowerer, init_e, module: str) -> dict:
    """Name and source span of the initial predicate (the <Init ...> line of a coverage report)."""
    if init_e[0] == "id":
        r = lw.root.resolve(init_e[1], None)
        if r is not None and r.kind == "def":
            d = r.defn
            return {"name": d.name, "module": d.module or module, "line": d.line, "col": d.col,
                    "end_line": d.end_line, "end_col": d.end_col}
    return {"name": "Init", "module": module}


def _resolve_init_next(lw: Lowerer):
    cfg, root = lw.cfg, lw.root
    if cfg.init and cfg.next:
        return ("id", cfg.init), ("id", cfg.next)
    if cfg.specification:
        d = root.find_def(cfg.specification, None)
        if d is None:
            raise LowerError(f"SPECIFICATION {cfg.specification} not found")
        found = {"init": None, "next": None}

        def walk(e):
            if e[0] == "and":
                for x in e[1]:
                    walk(x)
            elif e[0] == "box" and e[1][0] == "actionbox":
                found["next"] = e[1][1]
            elif e[0] != "fair" and found["init"] is None:
                found["init"] = e
        walk(d.body)
        if found["init"] is None or found["next"] is None:
            raise LowerError("SPECIFICATION is not of the form Init /\\ [][Next]_vars")
        return found["init"], found["next"]
    raise LowerError("cfg needs INIT+NEXT or SPECIFICATION")


HEADER_PROLOGUE = """\
// AUTO-GENERATED by kafka_specification_b200.lower -- do not edit.
// model   : {name}
// module  : {module}
// digest  : {digest}
#pragma once
#include <stdint.h>
#ifndef KMC_HD
#  ifdef __CUDACC__
#    define KMC_HD __host__ __device__ __forceinline__
#  else
#    define KMC_HD inline
#  endif
#endif
#ifndef KMC_FAIL_LAYOUT
#  define KMC_FAIL_LAYOUT 1   /* a successor value does not fit the packed layout */
#endif
#define KMC_MODEL_NAME "{name}"
#define KMC_MODEL_DIGEST "{digest}"
namespace kmc_model {{
static constexpr int W = {words};
static constexpr int STATE_BITS = {bits};
static constexpr bool ALL_ONES_POSSIBLE = {all_ones};   /* can a valid state pack to all-ones words? */
static constexpr int NUM_ACTIONS = {num_actions};
static constexpr int NUM_INVARIANTS = {num_invariants};
static constexpr int NUM_CONSTRAINTS = {num_constraints};
static constexpr int NUM_INIT = {num_init};
static constexpr int MAX_FANOUT = {max_fanout};   /* static bound: emit sites in expand() */
static constexpr bool CHECK_DEADLOCK = {check_deadlock};
struct State {{ uint64_t w[W]; }};
"""


GROUP_LINES = 160         # one-phase form: lines of Next per expand_group
MAX_GROUP_SITES = 64      # two-phase form: emit sites per site group (one 64-bit mask word)
GUARD_LINES = 3000        # two-phase form: a site group closes once its guard code is longer than this


def lower_model(module: str, search_dirs: list[str], cfg_text: str, name: str | None = None) -> LoweredModel:
    cfg = parse_cfg(cfg_text)
    root = load_root(module, search_dirs)
    lw = Lowerer(root, cfg)
    if cfg.view or cfg.properties or cfg.action_constraints:
        raise LowerError("VIEW / PROPERTY / ACTION_CONSTRAINT are not supported")

    # ASSUMEs of the root module (TLC evaluates them once at start-up)
    for a, mod in root.assumes:
        if lw.ev_bool(a, root, mod, {}, None) is not True:
            raise LowerError(f"ASSUME in module {mod} is not TRUE for this cfg")

    # layout
    layout_op = cfg.layout or "TypeOk"
    d, dctx = lw.named_def(layout_op)
    ti = TypeInference(lw)
    ti.collect(d.body, dctx, d.module, {})
    lay = L.Layout()
    def apply_prefix(ty, arr, length):
        if isinstance(ty, L.TFn):
            for t in ty.elems:
                apply_prefix(t, arr, length)
            ty.card = 0
            ty._sig = None
        elif isinstance(ty, L.TRec):
            ty.apply_prefix(arr, length)
        else:
            raise LowerError("PREFIX applies to a record variable or a function of records")

    for v in lw.variables:
        if v in cfg.type_hints:
            # checked hint: the layout type of this variable as written in the cfg (narrower than the type
            # invariant states, e.g. request epochs are never Nil); a value outside it traps at run time
            op, text = cfg.type_hints[v]
            sv = lw.ev(parse_expression_text(text), root, None, {}, None)
            ty = ti.type_from_setval(sv)
            if op == "\\subseteq":
                ty = L.TSet(ty)
        else:
            ty = copy.deepcopy(ti.variable_type(v))
        if v in cfg.keyed:
            if not isinstance(ty, L.TSet):
                raise LowerError(f"KEYED given for {v}, which is not a set")
            ty = L.TKeyedSet(ty.elem, cfg.keyed[v])
        elif v in cfg.capacities:
            if not isinstance(ty, (L.TSet, L.TSeq)):
                raise LowerError(f"CAPACITY given for {v}, which is neither a set nor a sequence")
            cap = lw.ev(parse_expression_text(cfg.capacities[v]), root, None, {}, None)
            if not is_int_const(cap) or cap < 0:
                raise LowerError(f"CAPACITY {v} does not evaluate to a natural number")
            if isinstance(ty, L.TSeq):
                ty.set_cap(cap)
            else:
                ty = L.TSet(ty.elem, cap)
        if isinstance(ty, L.TSeq) and ty.cap is None and v in ti.seq_caps:
            if ti.seq_caps[v] < 0:
                raise LowerError(f"Len({v}) is bounded by a negative number in {layout_op}")
            ty.set_cap(ti.seq_caps[v])
        if v in cfg.prefix:
            apply_prefix(ty, *cfg.prefix[v])
        lay.add_variable(v, ty)
    lay.finish()
    if lay.words > MAX_WORDS:
        raise LowerError(f"the state packs into {lay.words} 64-bit words ({lay.bits} bits); the expand kernel "
                         f"takes at most {MAX_WORDS} words")
    lw.layout = lay

    init_e, next_e = _resolve_init_next(lw)
    dev = device_init(lw, init_e, cfg)
    init_lines: list[str] = []
    if dev is not None:
        # device form: k_init decodes, filters and packs the candidates; the header has no table
        init_words = []
        init_lines = dev.emit()
    else:
        inits = _init_states(lw, init_e)
        if not inits:
            raise LowerError("Init has no solution")
        init_words = [lay.py_pack(st) for st in inits]
        for st, wds in zip(inits, init_words):
            if lay.py_unpack(wds) != st:
                raise LowerError("layout round-trip of an initial state failed")

    # expand()
    lw.begin_function()
    if next_e[0] == "id":
        nd, nctx = lw.named_def(next_e[1])
        start = [(nd.body, nctx, nd.module, {})]
    else:
        start = [(next_e, root, None, {})]
    lw.gen_next(start, {}, None)
    lw.end_unit()
    expand_prologue = list(lw.prologue)
    # One-phase form: consecutive units packed into groups of bounded size, one function each; expand() calls them
    # in order.  The host tests, the CPU baseline and the host-side shard stand-ins run it; the CUDA build skips
    # this section of the header (-DKMC_NO_ONE_PHASE) to keep nvcc time down.
    # A unit's one-phase text keeps its empty blocks; a split unit's is its pruned sub-units, one level shallower.
    # The body digest, which checkpoints are checked against, hashes this text.
    groups: list[list[str]] = []
    cur_lines: list[str] = []
    all_units: list[tuple[list, list[str]]] = []      # (pruned tree, one-phase text)
    for nodes in lw.units:
        pruned = _prune(nodes)
        if sum(isinstance(n, Block) for n in pruned) > 40:
            all_units.extend((sub, render(sub, 1)) for sub in _split_unit(pruned, 40))
        else:
            all_units.append((pruned, render(nodes, 2)))
    for _, lines in all_units:
        if cur_lines and len(cur_lines) + len(lines) > GROUP_LINES:
            groups.append(cur_lines)
            cur_lines = []
        cur_lines = cur_lines + ["  {"] + lines + ["  }"]
    if cur_lines or not groups:
        groups.append(cur_lines)
    expand_lines = [l for g in groups for l in g]
    # Two-phase form (what the CUDA expand kernel runs): every emit site becomes an item = (complete path
    # condition, straight-line body).  A site group = a run of consecutive sites (<= 64: one mask word; bounded
    # guard code so that the guard phase of a group stays in the instruction cache); a unit with more sites than
    # fit is covered by several windows of the same guard tree.
    unit_trees = [_unit_sites(nodes) for nodes, _ in all_units]
    site_bodies: list[list[str]] = []
    site_action: list[int] = []
    site_groups: list[dict] = []            # {"begin": first site, "count": n, "guard": lines}
    cur = {"begin": 0, "count": 0, "guard": []}
    for tree, sites in unit_trees:
        k = 0
        while k < len(sites):
            room = MAX_GROUP_SITES - cur["count"]
            if room == 0 or (cur["count"] and len(cur["guard"]) > GUARD_LINES):
                site_groups.append(cur)
                cur = {"begin": cur["begin"] + cur["count"], "count": 0, "guard": []}
                continue
            n = min(room, len(sites) - k)
            g = _render_guard(tree, k, k + n, cur["count"])
            cur["guard"] += ["  {"] + g + ["  }"]
            cur["count"] += n
            k += n
        site_action.extend(label for label, _ in sites)
        site_bodies.extend(body for _, body in sites)
    if cur["count"] or not site_groups:
        site_groups.append(cur)
    max_fanout = lw.emit_sites

    # invariants.  Each one ends in a top-level `return i` statement; violated_invariants() is the same tree with those
    # statements setting bit i instead, so that every invariant is evaluated.
    lw.begin_function()
    inv_exits: dict[int, str] = {}          # index in the body's children -> the statement of the mask form
    for i, inv in enumerate(cfg.invariants):
        idf, ictx = lw.named_def(inv)
        c = lw.ev_bool(idf.body, ictx, idf.module, {})
        if c is False:
            lw.cg.emit(f"return {i};")
            inv_exits[len(lw.cg.body.children) - 1] = f"m |= 1ull << {i};"
        elif c is not True:
            lw.cg.emit(f"if (!({c.s})) return {i};")
            inv_exits[len(lw.cg.body.children) - 1] = f"if (!({c.s})) m |= 1ull << {i};"
        if len(lw.cg.stack) != 1:
            raise LowerError(f"internal: invariant {inv} left a block open")
    inv_lines = lw.prologue + render(lw.cg.body.children, 1)
    mask_lines = lw.prologue + render([inv_exits.get(k, n) for k, n in enumerate(lw.cg.body.children)], 1)

    # constraints
    lw.begin_function()
    conds = []
    for con in cfg.constraints:
        cdf, cctx = lw.named_def(con)
        conds.append(lw.ev_bool(cdf.body, cctx, cdf.module, {}))
    c_all = lw.b_and(conds)
    con_lines = lw.prologue + render(lw.cg.body.children, 1) + [f"  return {lw.bstr(c_all)};"]

    # SYMMETRY: canonicalize(s) = lexicographically smallest packed image of s under the symmetry group
    sym_lines: list[str] = []
    n_perms = 0
    if cfg.symmetry:
        sdf, sctx = lw.named_def(cfg.symmetry)
        pv = lw.ev(sdf.body, sctx, sdf.module, {}, None)
        if not isinstance(pv, frozenset) or not all(isinstance(f, FnVal) for f in pv):
            raise LowerError("SYMMETRY must name a constant set of permutations (e.g. Permutations(Replicas))")
        lw.begin_function()
        for f in sorted(pv, key=sort_key):
            pmap = {k: x for k, x in f.items if k != x}
            if not pmap:
                continue
            n_perms += 1
            lw.cg.open()
            words = lw.gen_permuted_words(pmap)
            lw.cg.emit("State c;")
            for w, e in enumerate(words):
                lw.cg.emit(f"c.w[{w}] = {e};")
            lw.cg.emit("if (state_less(c, best)) best = c;")
            lw.cg.close()
        sym_lines = lw.prologue + render(lw.cg.body.children, 1)

    name = name or module
    if len(lw.actions) > 255:
        raise LowerError(f"{len(lw.actions)} sub-actions: the parent word holds the action id in 8 bits (<= 255)")
    # (the device form's code is part of what a checkpoint is checked against; a table model hashes what it always did)
    body_digest = hashlib.sha256(("\n".join(expand_lines + inv_lines + con_lines + sym_lines + init_lines) + cfg_text).encode()).hexdigest()[:16]
    unpack = lw.unpack_lines()

    parts = [HEADER_PROLOGUE.format(
        name=name, module=module, digest=body_digest, words=lay.words, bits=lay.bits,
        all_ones="true" if lay.all_ones_possible else "false",
        num_actions=max(1, len(lw.actions)), num_invariants=len(cfg.invariants),
        num_constraints=len(cfg.constraints), num_init=len(init_words), max_fanout=max(1, max_fanout),
        check_deadlock="true" if cfg.check_deadlock else "false")]
    if dev is not None:
        parts.extend(init_lines)
    else:
        parts.append("static const uint64_t INIT_STATES[NUM_INIT][W] = {")
        for wds in init_words:
            parts.append("  {" + ", ".join(f"0x{w:x}ull" for w in wds) + "},")
        parts.append("};")
    parts.append("/* successor enumeration: sink.emit(const State&, int action) per successor; sink.fail(code) on a layout trap.")
    parts.append("   Two equivalent forms (tests prove they enumerate the same multiset):")
    parts.append("   one-phase   expand() = expand_group<0..NUM_GROUPS-1> in order; a group is a slice of the Next disjuncts /")
    parts.append("               bindings small enough to stay in the instruction cache while it is swept over a tile of states;")
    parts.append("   two-phase   site_mask(SiteGroupTag<g>, s) = bit k set iff the COMPLETE path condition of emit site")
    parts.append("               SITE_GROUP_BEGIN[g] + k holds for s;  site_body(SiteTag<i>, s, sink) = the straight-line")
    parts.append("               successor construction of site i, run only for (state, site) pairs whose bit is set. */")
    parts.append("#ifndef KMC_NO_ONE_PHASE")
    parts.append(f"static constexpr int NUM_GROUPS = {len(groups)};")
    parts.append("template <int G> struct GroupTag {};")
    for gi, glines in enumerate(groups):
        parts.append(f"template <class Sink> KMC_HD void expand_group(GroupTag<{gi}>, const State& s, Sink& sink) {{")
        parts.extend(unpack)
        parts.extend(expand_prologue)
        parts.extend(glines)
        parts.append("}")
    parts.append("template <class Sink> KMC_HD void expand(const State& s, Sink& sink) {")
    for gi in range(len(groups)):
        parts.append(f"  expand_group(GroupTag<{gi}>{{}}, s, sink);")
    parts.append("}")
    parts.append("#endif  // KMC_NO_ONE_PHASE")
    n_sites = len(site_bodies)
    parts.append(f"static constexpr int NUM_SITES = {n_sites};")
    parts.append("/* action of every emit site (index into the model's actions; -1: the site only reports a layout trap) */")
    parts.append("static constexpr int SITE_ACTION[NUM_SITES > 0 ? NUM_SITES : 1] = {" +
                 (", ".join(str(a) for a in site_action) if site_action else "-1") + "};")
    parts.append(f"static constexpr int NUM_SITE_GROUPS = {len(site_groups)};")
    parts.append("static constexpr int SITE_GROUP_BEGIN[NUM_SITE_GROUPS + 1] = {" +
                 ", ".join(str(g["begin"]) for g in site_groups) + f", {n_sites}" + "};")
    parts.append("template <int G> struct SiteGroupTag {};")
    parts.append("template <int I> struct SiteTag {};")
    for gi, g in enumerate(site_groups):
        parts.append(f"KMC_HD uint64_t site_mask(SiteGroupTag<{gi}>, const State& s) {{")
        parts.extend(unpack)
        parts.extend(expand_prologue)
        parts.append("  uint64_t m = 0;")
        parts.extend(g["guard"])
        parts.append("  return m;")
        parts.append("}")
    for i, body in enumerate(site_bodies):
        parts.append(f"template <class Sink> KMC_HD void site_body(SiteTag<{i}>, const State& s, Sink& sink) {{")
        parts.extend(unpack)
        parts.extend(expand_prologue)
        parts.extend(body)
        parts.append("}")
    parts.append("/* expand() through the two-phase form (host-side tests prove both forms agree) */")
    parts.append("template <int I, int END> struct SiteLoop {")
    parts.append("  template <class Sink> static KMC_HD void run(uint64_t m, int bit, const State& s, Sink& sink) {")
    parts.append("    if ((m >> bit) & 1) site_body(SiteTag<I>{}, s, sink);")
    parts.append("    SiteLoop<I + 1, END>::run(m, bit + 1, s, sink);")
    parts.append("  }")
    parts.append("};")
    parts.append("template <int END> struct SiteLoop<END, END> {")
    parts.append("  template <class Sink> static KMC_HD void run(uint64_t, int, const State&, Sink&) {}")
    parts.append("};")
    parts.append("template <int G> struct SiteGroupLoop {")
    parts.append("  template <class Sink> static KMC_HD void run(const State& s, Sink& sink) {")
    parts.append("    SiteLoop<SITE_GROUP_BEGIN[G], SITE_GROUP_BEGIN[G + 1]>::run(site_mask(SiteGroupTag<G>{}, s), 0, s, sink);")
    parts.append("    SiteGroupLoop<G + 1>::run(s, sink);")
    parts.append("  }")
    parts.append("};")
    parts.append("template <> struct SiteGroupLoop<NUM_SITE_GROUPS> {")
    parts.append("  template <class Sink> static KMC_HD void run(const State&, Sink&) {}")
    parts.append("};")
    parts.append("template <class Sink> KMC_HD void expand_sites(const State& s, Sink& sink) { SiteGroupLoop<0>::run(s, sink); }")
    parts.append("/* index of the first violated INVARIANT of the cfg, or -1 */")
    parts.append("KMC_HD int first_violated_invariant(const State& s) {")
    parts.extend(unpack)
    parts.extend(inv_lines)
    parts.append("  return -1;")
    parts.append("}")
    parts.append("/* conjunction of the cfg's CONSTRAINTs */")
    parts.append("KMC_HD bool in_model(const State& s) {")
    parts.extend(unpack)
    parts.extend(con_lines)
    parts.append("}")
    parts.append(f"/* SYMMETRY: {n_perms} non-identity permutations; canonicalize = smallest packed image (identity if none) */")
    parts.append(f"static constexpr bool HAS_SYMMETRY = {'true' if n_perms else 'false'};")
    parts.append("KMC_HD bool state_less(const State& a, const State& b) {")
    parts.append("  for (int i = W - 1; i >= 0; --i) { if (a.w[i] != b.w[i]) return a.w[i] < b.w[i]; }")
    parts.append("  return false;")
    parts.append("}")
    parts.append("KMC_HD void canonicalize(const State& s, State& best) {")
    parts.append("  best = s;")
    if n_perms:
        parts.extend(unpack)
        parts.extend(sym_lines)
    parts.append("}")
    parts.append("}  // namespace kmc_model")
    header = "\n".join(parts) + "\n"

    # invariants.h, included after model.h: the invariants as a bit mask (up to 64 of them)
    if len(cfg.invariants) <= MAX_MASK_INVARIANTS:
        mask_fn = (["/* bit i set iff INVARIANT i of the cfg is false: first_violated_invariant with every invariant evaluated */",
                    "KMC_HD uint64_t violated_invariants(const State& s) {"] + unpack + ["  uint64_t m = 0;"] + mask_lines +
                   ["  return m;", "}"])
    else:
        mask_fn = [f"/* {len(cfg.invariants)} INVARIANTs do not fit a 64-bit mask: no per-invariant report for this model */",
                   "KMC_HD uint64_t violated_invariants(const State&) { return 0; }"]
    invariants_header = "\n".join([f"// generated by the lowering for {name}: the companion of model.h", "namespace kmc_model {",
                                   f"static constexpr bool HAS_INVARIANT_MASK = {'true' if len(cfg.invariants) <= MAX_MASK_INVARIANTS else 'false'};",
                                   *mask_fn, "}  // namespace kmc_model"]) + "\n"

    return LoweredModel(
        name=name, module=module, header=header, layout=lay.describe(), words=lay.words,
        state_bits=lay.bits, init_states=init_words, actions=lw.actions or [{"name": "Next", "module": module}],
        invariants=list(cfg.invariants), constraints=list(cfg.constraints),
        check_deadlock=cfg.check_deadlock, max_fanout=max(1, max_fanout), warnings=lw.warnings,
        digest=body_digest, lowerer=lw, variables=list(lw.variables),
        sites=[{"action": a} for a in site_action],
        init={**_init_info(lw, init_e, module), **(dev.describe() if dev is not None else {})},
        invariants_header=invariants_header)
