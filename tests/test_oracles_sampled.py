"""Oracle A on the BIG models, by sampling.

The interpreter of the unchanged .tla text (Oracle A, ~400 states/s) can enumerate 10^4..10^6 states; the headline
model has 3.4e8, config #4 (5 brokers) and config #5 (AsyncIsr deep) more.  What it CAN do at any size is judge single
states: this test walks each big model's state graph from Init with the lowered Next (random successor, fixed seed)
and, AT EVERY STEP of every walk, compares for the current state

  * the multiset of successors (TLC's "states generated" multiplicity included), as canonical TLC text, and
  * the verdict of every configured invariant and constraint,

between Oracle A (evaluating the reference's text for this cfg) and the lowered model (the header the CUDA engine
compiles), in both forms of the lowered Next.  Every state visited is reachable by construction as long as all earlier
steps agreed -- and the first disagreement fails the test.  Walks are long enough to reach the deep levels (full logs,
maximal epochs) that a bounded BFS prefix never sees."""
import os
import random

import numpy as np
import pytest

from conftest import REFERENCE, ROOT, needs_reference
from hostmodel import HostModel, lower_model

DIRS = [REFERENCE, os.path.join(ROOT, "models"), os.path.join(ROOT, "tests", "specs")]

# (model, walks, steps per walk)
CASES = [("kip320_3x4_r4e3", 6, 45), ("trunchw_3x4_r3e3", 4, 40), ("kip101_3x4_r3e3", 3, 40), ("kip279_3x4_r3e3", 3, 40),
         ("firsttry_3x4_r3e3", 3, 40), ("kip320_with279_small", 3, 30), ("asyncisr_deep", 5, 45), ("kip320_5brokers", 3, 40)]


def _text(variables, st):
    from kafka_specification_b200.frontend.values import fmt
    return "\n".join(f"/\\ {v} = {fmt(st[v])}" for v in variables)


@needs_reference
@pytest.mark.parametrize("name,walks,steps", CASES)
def test_random_walks_agree_with_oracle_a_step_by_step(name, walks, steps, registry):
    import tla_interp
    from kafka_specification_b200.frontend.cfg import parse_cfg
    from kafka_specification_b200.frontend.modules import load_root
    spec = registry[name]
    cfg_text = open(os.path.join(ROOT, spec["cfg"])).read()
    m = lower_model(spec["module"], DIRS, cfg_text, name=name)
    hm = HostModel.from_lowered(m)

    cfg = parse_cfg(cfg_text)
    root = load_root(spec["module"], DIRS)
    it = tla_interp.Interp(root, cfg)
    it.check_assumes()
    init_e, next_e = tla_interp.resolve_init_next(root, cfg)
    variables = it.variables

    # Init: the same set of states on both sides
    a_inits = sorted(_text(variables, st) for st in it.init_states(init_e))
    l_inits = list(hm.init_states())
    assert sorted(m.state_text(w) for w in l_inits) == a_inits

    walks *= int(os.environ.get("KSPEC_WALK_SCALE", "1"))          # (a longer offline run: KSPEC_WALK_SCALE=10)
    kafka_b = None
    if spec.get("kso") and "replicaLog" in variables:
        import kso
        kafka_b = tuple(spec["kso"])
        replicas = sorted(m.decode_state(l_inits[0])["replicaLog"].domain(), key=str)
    rng = random.Random(20260923 + len(name))
    compared = deepest = 0
    for _ in range(walks):
        cur = l_inits[rng.randrange(len(l_inits))].copy()
        for step in range(steps):
            st = m.decode_state(cur)
            assert m.lowerer.layout.py_pack(st) == [int(x) for x in cur]        # decode/encode round trip
            # verdicts
            viol_a = next((i for i, inv in enumerate(cfg.invariants) if not it.eval_named_predicate(inv, st)), -1)
            assert hm.first_violated(cur) == viol_a, (name, step, m.state_text(cur))
            inmodel_a = all(it.eval_named_predicate(c, st) for c in cfg.constraints)
            assert hm.in_model(cur) == inmodel_a
            # successors: multiset of canonical texts, both forms of the lowered Next
            succ_a = it.next_states(next_e, st)
            want = sorted(_text(variables, s1) for s1 in succ_a)
            if kafka_b is not None:
                # three-way: Oracle B (the hand-written C restatement all the large goldens come from) enumerates the
                # same multiset of successors for this state and gives the same invariant verdicts as Oracle A
                model_b, params_b = kafka_b
                rec = kso.kstate_from_tla(st, replicas)
                assert sorted(kso.successors(model_b, params_b, rec)) == sorted(kso.kstate_from_tla(s1, replicas) for s1 in succ_a), \
                    (name, f"step {step}: Oracle B and Oracle A enumerate different successors for\n{m.state_text(cur)}")
                inv_b = [i for i in cfg.invariants if i in kso.INVARIANTS]
                assert set(kso.violated(model_b, params_b, rec, inv_b)) == {i for i in inv_b if not it.eval_named_predicate(i, st)}
            rows = None
            for items in (0, 1):
                rows, _ = hm.successors(cur, sites=bool(items))          # (a layout trap raises)
                got = sorted(m.state_text(r) for r in rows)
                assert got == want, (name, f"step {step}, form {items}: successors differ for\n{m.state_text(cur)}")
            compared += 1
            deepest = max(deepest, step + 1)
            # continue from a random in-model successor (out-of-model ones are not expanded by a checker)
            nxt = [r for r in rows if hm.in_model(r)]
            if not nxt:
                break
            cur = nxt[rng.randrange(len(nxt))].copy()
    assert compared >= walks * 5 and deepest >= min(steps, 12)
    print(f"[walks] {name}: {walks} walks, {compared} states compared step by step, deepest step {deepest}")


@needs_reference
@pytest.mark.parametrize("name,walks,steps", [("kip320sym_3x4_r4e3", 4, 40), ("kip320sym_5brokers", 2, 35)])
def test_canonicalize_is_an_orbit_invariant_on_deep_states(name, walks, steps, registry):
    """SYMMETRY at headline size (3! permutations) and for config #4 (5! = 120): on the states of random walks the lowered
    canonicalize() (what the GPU fingerprints) must be (a) the same for every permuted image of the state -- images
    built with Oracle A's permute_value on the decoded TLA values, packed by the layout --, (b) one of those images,
    (c) idempotent.  Together: it picks one representative per orbit, which is all TLC's symmetry reduction needs."""
    import itertools
    import tla_interp
    spec = registry[name]
    cfg_text = open(os.path.join(ROOT, spec["cfg"])).read()
    m = lower_model(spec["module"], DIRS, cfg_text, name=name)
    hm = HostModel.from_lowered(m)
    lay = m.lowerer.layout
    replicas = sorted(m.decode_state(np.array(m.init_states[0], dtype=np.uint64))["replicaLog"].domain(), key=str)
    perms = [dict(zip(replicas, p)) for p in itertools.permutations(replicas)]

    def canon(words):
        return tuple(int(x) for x in hm.canonicalize(np.array(words, dtype=np.uint64))[0])

    rng = random.Random(7 + len(name))
    checked = 0
    for _ in range(walks):
        cur = np.array(m.init_states[0], dtype=np.uint64)
        for step in range(steps):
            st = m.decode_state(cur)
            c0 = canon(cur)
            images = set()
            for pm in perms:
                img = {v: tla_interp.permute_value(st[v], pm) for v in m.variables}
                words = lay.py_pack(img)
                images.add(tuple(words))
                assert canon(words) == c0, (name, step, pm)
            assert c0 in images and canon(c0) == c0
            checked += 1
            out, _ = hm.successors(cur)                               # (a layout trap raises)
            if len(out) == 0:
                break
            cur = out[rng.randrange(len(out))].copy()
    assert checked >= walks * 10
