"""Writers of TLC's ``-dump`` files: the reachable states, or the state graph in GraphViz dot.

    -dump FILE                                      every stored state, ``State k:`` and its text (``FILE.dump``)
    -dump dot[,actionlabels][,colorize][,snapshot] FILE   the state graph (``FILE.dot``)

The layouts are reproduced from TLC's published behaviour (its ``-dump`` state file and its ``DotStateWriter``).  TLC
cannot be run here, so they are unverified, like the ``-tool`` message codes (DESIGN section 0).  Two differences are
deliberate:

* TLC numbers the states of ``-dump`` in the order its workers discover them.  Here the states are written level by
  level, and within a level by their packed words, so that a file does not depend on which insert won: without
  SYMMETRY it is byte-identical across runs and across ``spill`` / ``set_spill``.  Compared as sets, the two tools'
  files hold the same states.
* ``snapshot`` (TLC rewrites the dot file at every progress report) is accepted and ignored: the file is written once,
  at the end of the run.

Node ids of the dot file are the set-identity fingerprints of the states (``kmc_edge_t.src_fp``, under SYMMETRY that
of the orbit) as signed decimals.  Edges come from the expanded states only, so a stopped run shows the graph explored
so far, and an edge may point at a fingerprint that has no node (a successor of the last level of a stopped run).
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

DOT_OPTIONS = ("actionlabels", "colorize", "snapshot")
COLORS = 12          # GraphViz's "paired12" scheme: action a is drawn in colour a % 12 + 1


@dataclass
class DumpRequest:
    path: str
    dot: bool = False
    options: list[str] = field(default_factory=list)

    @property
    def actionlabels(self) -> bool:
        return "actionlabels" in self.options

    @property
    def colorize(self) -> bool:
        return "colorize" in self.options


def split_dump_args(argv: list[str]) -> tuple[list[str], DumpRequest | None]:
    """Takes ``-dump FILE`` or ``-dump dot[,OPTION...] FILE`` out of a TLC command line before the rest is parsed (the
    two-token form would otherwise swallow ``SPEC``).  The file gets ``.dot`` / ``.dump`` when its name lacks it.
    Raises ValueError on a missing file name or an unknown dot option."""
    if "-dump" not in argv:
        return list(argv), None
    i = argv.index("-dump")
    rest = argv[:i]
    tail = argv[i + 1:]
    if not tail:
        raise ValueError("-dump needs a file name")
    dot = tail[0] == "dot" or tail[0].startswith("dot,")
    if dot:
        options = [o for o in tail[0].split(",")[1:] if o]
        bad = [o for o in options if o not in DOT_OPTIONS]
        if bad:
            raise ValueError(f"-dump dot: unknown option {bad[0]!r} (known: {', '.join(DOT_OPTIONS)})")
        tail = tail[1:]
        if not tail:
            raise ValueError("-dump dot needs a file name")
    else:
        options = []
    path = tail[0]
    suffix = ".dot" if dot else ".dump"
    if not path.endswith(suffix):
        path += suffix
    rest2, again = split_dump_args(tail[1:])
    if again is not None:
        raise ValueError("-dump is given twice")
    return rest + rest2, DumpRequest(path, dot, options)


def row_order(rows: np.ndarray) -> np.ndarray:
    """The permutation that orders packed states by their words, word 0 first."""
    rows = np.asarray(rows, dtype=np.uint64)
    if rows.shape[0] == 0:
        return np.empty(0, dtype=np.int64)
    return np.lexsort(rows.T[::-1])


def sorted_rows(rows: np.ndarray) -> np.ndarray:
    return rows[row_order(rows)]


def write_states(f, texts: list[str], first_number: int) -> int:
    """``State k:`` blocks of TLC's ``-dump`` file, numbered from ``first_number``; returns how many were written."""
    f.write("".join(f"State {first_number + i}:\n{t}\n\n" for i, t in enumerate(texts)))
    return len(texts)


def escape(text: str) -> str:
    """A state's text as a dot label: backslashes and quotes escaped, lines joined by ``\\n``."""
    return text.replace("\\", "\\\\").replace('"', '\\"').strip().replace("\n", "\\n")


def signed(fp) -> int:
    return int(np.uint64(fp).astype(np.int64))


def distinct_edges(edges: np.ndarray) -> np.ndarray:
    """One row per distinct (src_fp, dst_fp, action), ordered by them."""
    if len(edges) == 0:
        return np.empty(0, dtype=[("src_fp", np.uint64), ("dst_fp", np.uint64), ("action", np.uint32)])
    keys = np.empty(len(edges), dtype=[("src_fp", np.uint64), ("dst_fp", np.uint64), ("action", np.uint32)])
    for k in ("src_fp", "dst_fp", "action"):
        keys[k] = edges[k]
    return np.unique(keys)


def write_dot(f, fps: np.ndarray, texts: list[str], n_init: int, edges: np.ndarray, actions: list[str], *,
              actionlabels: bool = False, colorize: bool = False) -> dict:
    """The state graph in TLC's DotStateWriter layout.  ``fps[i]`` / ``texts[i]``: node i (the first ``n_init`` are the
    initial states, drawn filled); ``edges``: records with ``src_fp``, ``dst_fp`` and ``action`` (duplicates allowed).
    Returns the node and edge counts written."""
    out = ["strict digraph DiskGraph {"]
    if colorize:
        out.append('edge [colorscheme="paired12"]')
    out += ["nodesep=0.35;", "subgraph cluster_graph {", 'color="white";']
    for i, (fp, text) in enumerate(zip(fps, texts)):
        style = ",style = filled" if i < n_init else ""
        out.append(f'{signed(fp)} [label="{escape(text)}"{style}]')
    uniq = distinct_edges(edges)
    for e in uniq:
        attrs = []
        a = int(e["action"])
        if actionlabels:
            attrs.append(f'label="{actions[a] if a < len(actions) else a}"')
        if colorize:
            attrs += [f'color="{a % COLORS + 1}"', f'fontcolor="{a % COLORS + 1}"']
        out.append(f'{signed(e["src_fp"])} -> {signed(e["dst_fp"])}' + (f' [{",".join(attrs)}]' if attrs else "") + ";")
    out.append("}")
    if colorize:
        out.append('subgraph cluster_legend {graph[style=bold];label = "Next State Actions" style="solid"')
        out.append('node [ labeljust="l",colorscheme="paired12",style=filled,shape=record ]')
        out += [f'{name} [label="{name}",fillcolor={a % COLORS + 1}]' for a, name in enumerate(actions)]
        out.append("}")
    out.append("}")
    f.write("\n".join(out) + "\n")
    return {"nodes": len(texts), "edges": len(uniq)}
