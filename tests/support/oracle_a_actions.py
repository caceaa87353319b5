"""Test support: Oracle A (oracle/tla_interp.py) with every successor labelled by its action.

TLC's rule for the action of a successor (the one its -coverage report and its error traces name): the first
user-defined operator applied below ``Next``.  ``run_bfs_by_action`` runs Oracle A's own BFS unchanged and counts,
per action, the successors generated -- duplicates and successors a CONSTRAINT discards included, exactly as
"generated" counts them.  The lowering labels its emit sites by the same rule in its own code path, so the two
agreeing checks the lowering's labels against an independent interpreter.  ``OracleA`` holds the labelled interpreter
of one registered model and replays the error traces of GPU runs through it.
"""
from __future__ import annotations

import os
import sys
from collections import Counter

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import tla_interp  # noqa: E402
from tla_interp import Closure, EvalError, set_elems, sort_key  # noqa: E402


class LabelledInterp(tla_interp.Interp):
    """Interp whose next_states() also counts the successors of every action in ``self.generated``."""

    def __init__(self, root, cfg):
        super().__init__(root, cfg)
        self.generated: Counter = Counter()

    def labelled_successors(self, next_expr, st: dict) -> list[tuple[dict, str]]:
        """The successors of `st` under Next, each with the name of the action that produced it."""
        start = (next_expr, self.root, None, {})
        if next_expr[0] == "id":
            # the body of Next: Next itself is not an action (the lowering starts at the same place)
            r = self.root.resolve(next_expr[1], None)
            if r is not None and r.kind == "def" and not r.defn.params:
                start = (r.defn.body, r.ctx, r.defn.module, {})
        out: list[tuple[dict, str]] = []
        self._next_l([start], st, {}, out, None)
        return out

    def next_states(self, next_expr, st: dict) -> list[dict]:
        out = self.labelled_successors(next_expr, st)
        for _, label in out:
            self.generated[label] += 1
        return [s1 for s1, _ in out]

    def _next_l(self, items, st, st1, out, label):
        """Interp._next with the action label carried along."""
        if not items:
            for v in self.variables:
                if v not in st1:
                    raise EvalError(f"successor leaves {v}' unassigned")
            out.append((st1, label or "Next"))
            return
        (e, ctx, fm, env), rest = items[0], items[1:]
        k = e[0]
        if k == "and":
            self._next_l([(x, ctx, fm, env) for x in e[1]] + rest, st, st1, out, label)
            return
        if k == "or":
            for x in e[1]:
                self._next_l([(x, ctx, fm, env)] + rest, st, st1, out, label)
            return
        if k == "quant" and e[1] == "E":
            for env2 in self.bindings(e[2], ctx, fm, env, st, st1):
                self._next_l([(e[3], ctx, fm, env2)] + rest, st, st1, out, label)
            return
        if k == "let":
            self._next_l([(e[2], ctx, fm, self.let_env(e[1], ctx, fm, env))] + rest, st, st1, out, label)
            return
        if k == "if":
            branch = e[2] if self.ev_bool(e[1], ctx, fm, env, st, st1) else e[3]
            self._next_l([(branch, ctx, fm, env)] + rest, st, st1, out, label)
            return
        if k in ("id", "app", "inst"):
            op = None
            if not (k == "id" and e[1] in env and not isinstance(env[e[1]], Closure)):
                op = self.find_operator(e, ctx, fm, env)
            if op is not None:
                target, defctx, args = op
                if label is None and not isinstance(target, Closure):
                    label = target.name
                body, c2, fm2, env2 = self.bind_call(target, defctx, args, ctx, fm, env)
                self._next_l([(body, c2, fm2, env2)] + rest, st, st1, out, label)
                return
        if k == "binop" and e[1] in ("=", "\\in") and e[2][0] == "prime":
            v = self.resolve_var(e[2][1], ctx, fm, env)
            if v is not None and v not in st1:
                rhs = self.ev(e[3], ctx, fm, env, st, st1)
                if e[1] == "=":
                    self._next_l(rest, st, {**st1, v: rhs}, out, label)
                else:
                    for x in sorted(set_elems(rhs), key=sort_key):
                        self._next_l(rest, st, {**st1, v: x}, out, label)
                return
        if k == "unchanged":
            new1 = st1
            for v in self.unchanged_vars(e[1], ctx, fm, env):
                if v in new1:
                    if new1[v] != st[v]:
                        return
                else:
                    new1 = {**new1, v: st[v]}
            self._next_l(rest, st, new1, out, label)
            return
        if self.ev_bool(e, ctx, fm, env, st, st1):
            self._next_l(rest, st, st1, out, label)


class OracleA:
    """Oracle A's interpreter for one registered model: initial states, labelled successors, predicates."""

    def __init__(self, name: str):
        from kafka_specification_b200.build import registry, tla_search_dirs
        from kafka_specification_b200.frontend.cfg import parse_cfg
        from kafka_specification_b200.frontend.modules import load_root
        spec = registry()[name]
        with open(os.path.join(ROOT, spec["cfg"])) as f:
            self.cfg = parse_cfg(f.read())
        root = load_root(spec["module"], tla_search_dirs())
        self.it = LabelledInterp(root, self.cfg)
        init_e, self.next_e = tla_interp.resolve_init_next(root, self.cfg)
        self.inits = self.it.init_states(init_e)

    def text(self, st: dict) -> str:
        from kafka_specification_b200.frontend.values import fmt
        return "\n".join(f"/\\ {v} = {fmt(st[v])}" for v in self.it.variables)

    def holds(self, name: str, st: dict) -> bool:
        return self.it.eval_named_predicate(name, st)

    def violated(self, st: dict) -> list[str]:
        return [inv for inv in self.cfg.invariants if not self.holds(inv, st)]

    def in_model(self, st: dict) -> bool:
        return all(self.holds(c, st) for c in self.cfg.constraints)

    def replay(self, trace: list[dict]) -> list[dict]:
        """The Oracle A states of an error trace (entries with "text" and "action"): the first one an initial state of
        that text, each next one a successor of its predecessor under the action the trace names, of that text."""
        assert trace[0]["action"] is None
        by_text = {self.text(s): s for s in self.inits}
        assert trace[0]["text"] in by_text, "the first state is not an initial state"
        states = [by_text[trace[0]["text"]]]
        for i, t in enumerate(trace[1:], start=1):
            nxt = [s1 for s1, label in self.it.labelled_successors(self.next_e, states[-1])
                   if label == t["action"]["name"] and self.text(s1) == t["text"]]
            assert nxt, f"trace state {i + 1} is not a {t['action']['name']} successor of state {i}:\n{t['text']}"
            states.append(nxt[0])
        return states


def run_bfs_by_action(module: str, search_dirs: list[str], cfg_text: str) -> dict:
    """Oracle A's full BFS (past violations, like -continue) plus ``per_action``: successors generated per action."""
    interps = []

    class Recording(LabelledInterp):
        def __init__(self, root, cfg):
            super().__init__(root, cfg)
            interps.append(self)

    saved = tla_interp.Interp
    tla_interp.Interp = Recording          # run_bfs builds its interpreter from the module's global
    try:
        res = tla_interp.run_bfs(module, search_dirs, cfg_text, stop_on_violation=False)
    finally:
        tla_interp.Interp = saved
    res["per_action"] = dict(interps[0].generated)
    return res
