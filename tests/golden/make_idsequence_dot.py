"""Generates tests/golden/idsequence.dot -- the state graph `tlc2 -dump dot,actionlabels,colorize` writes for
models/IdSequence.cfg -- from the host side alone: the host BFS of the lowered model (tests/support/host_model.cpp),
the engine's fingerprint computed in numpy, and the state texts of model.json's layout.  Run after build()."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests", "support")]

from kafka_specification_b200 import dump  # noqa: E402
from kafka_specification_b200.runtime import EDGE_DTYPE, StateDecoder  # noqa: E402
from store_audit import AuditLib  # noqa: E402


def main():
    a = AuditLib.for_built_model("idsequence")
    meta = json.load(open(os.path.join(ROOT, "build", "models", "idsequence", "model.json")))
    st = a.host_bfs()
    states, widths = st["states"], st["widths"]
    fps, texts, first = [], [], 0
    dec = StateDecoder(meta)
    for w in widths:
        rows = dump.sorted_rows(states[first:first + w])
        fps.append(a.fingerprints(rows, a.symmetry))
        texts += dec.texts(rows)
        first += w
    edges = []
    for s in states:
        succ, act = a.successors(s)
        for t, ac in zip(succ, act):
            if a.in_model(t):
                edges.append((a.fingerprints(s[None], a.symmetry)[0], a.fingerprints(t[None], a.symmetry)[0], ac))
    e = np.zeros(len(edges), dtype=EDGE_DTYPE)
    for i, (s, d, ac) in enumerate(edges):
        e[i]["src_fp"], e[i]["dst_fp"], e[i]["action"] = s, d, ac
    with open(os.path.join(HERE, "idsequence.dot"), "w") as f:
        print(dump.write_dot(f, np.concatenate(fps), texts, widths[0], e, [x["name"] for x in meta["actions"]],
                             actionlabels=True, colorize=True))


if __name__ == "__main__":
    main()
