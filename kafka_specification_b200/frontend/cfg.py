"""Parser for TLC model configuration (``.cfg``) files.

The reference ships no ``.cfg`` (its ``.gitignore:1`` excludes the Toolbox model
directories), so the grammar here is the published TLC one, restricted to what a
safety run needs:

    CONSTANT[S]   name = value | name <- Operator       (any number, any order)
    INIT name / NEXT name / SPECIFICATION name
    INVARIANT[S] names...   CONSTRAINT[S] names...   ACTION_CONSTRAINT[S] names...
    CHECK_DEADLOCK TRUE|FALSE      SYMMETRY name      VIEW name      PROPERTY/PROPERTIES names

Values: integers, "strings", TRUE/FALSE, identifiers (model values) and ``{v, ...}`` sets.

Build-specific directives live in ``\\* kspec:`` comment lines so that the file stays a
valid TLC configuration:

    \\* kspec: LAYOUT LayoutOk                    operator whose conjuncts give each variable's type
    \\* kspec: CAPACITY leaderAndIsrRequests = MaxLeaderEpoch + 1
                                                  bound on the cardinality of a set variable stored as a sorted array, or
                                                  on the length of a `v \\in Seq(S)` variable (checked: a longer value traps)
    \\* kspec: TYPE leaderAndIsrRequests \\subseteq [leaderEpoch : 0 .. MaxLeaderEpoch, ...]
                                                  layout type of one variable, overriding the one inferred from the
                                                  type invariant (a checked hint: a value outside it traps)
    \\* kspec: KEYED leaderAndIsrRequests BY leaderEpoch
                                                  a set of records in which the field determines the record: stored as
                                                  one entry per key value (checked: a second record with the key traps)
    \\* kspec: PREFIX replicaLog records endOffset
                                                  in every record of the variable, `records[o]` is the Nil alternative
                                                  exactly for o >= `endOffset` (checked), so Nil needs no code of its own
    \\* kspec: INIT DEVICE                         enumerate Init on the GPU (lower/init_device.py) even when it has
                                                  fewer candidates than the threshold that selects that form by itself
"""
from __future__ import annotations

import re
from dataclasses import dataclass, field


class CfgError(Exception):
    pass


@dataclass(frozen=True)
class ModelValue:
    name: str

    def __repr__(self) -> str:
        return self.name

    def __lt__(self, other):
        return self.name < other.name


@dataclass
class Config:
    constants: dict[str, object] = field(default_factory=dict)       # name -> python value
    overrides: dict[str, str] = field(default_factory=dict)          # name -> operator name
    init: str | None = None
    next: str | None = None
    specification: str | None = None
    invariants: list[str] = field(default_factory=list)
    constraints: list[str] = field(default_factory=list)
    action_constraints: list[str] = field(default_factory=list)
    properties: list[str] = field(default_factory=list)
    symmetry: str | None = None
    view: str | None = None
    check_deadlock: bool = True
    layout: str | None = None                                        # kspec pragma
    capacities: dict[str, str] = field(default_factory=dict)         # var -> TLA+ expression text
    type_hints: dict[str, tuple] = field(default_factory=dict)       # var -> ("\\in" | "\\subseteq", TLA+ expression text)
    keyed: dict[str, str] = field(default_factory=dict)              # var -> key field
    prefix: dict[str, tuple] = field(default_factory=dict)           # var -> (array field, length field)
    init_device: bool = False                                        # kspec pragma INIT DEVICE: Init is enumerated on the GPU
    source: str = ""


_SECTION_WORDS = {
    "CONSTANT", "CONSTANTS", "INIT", "NEXT", "SPECIFICATION", "INVARIANT", "INVARIANTS",
    "CONSTRAINT", "CONSTRAINTS", "ACTION_CONSTRAINT", "ACTION_CONSTRAINTS", "PROPERTY",
    "PROPERTIES", "SYMMETRY", "VIEW", "CHECK_DEADLOCK", "ALIAS", "POSTCONDITION",
}

_TOK = re.compile(r'\s+|(?P<num>-?\d+)|(?P<str>"[^"]*")|(?P<id>[A-Za-z_][A-Za-z0-9_!]*)|(?P<op><-|=|\{|\}|,)')


def _strip_comments(text: str) -> tuple[str, list[str]]:
    pragmas: list[str] = []
    for m in re.finditer(r"\\\*\s*kspec:\s*(.*)", text):
        pragmas.append(m.group(1).strip())
    text = re.sub(r"\(\*.*?\*\)", " ", text, flags=re.S)
    text = re.sub(r"\\\*[^\n]*", " ", text)
    return text, pragmas


def parse_cfg(text: str) -> Config:
    cfg = Config(source=text)
    body, pragmas = _strip_comments(text)
    toks: list[tuple[str, str]] = []
    pos = 0
    while pos < len(body):
        m = _TOK.match(body, pos)
        if m is None:
            raise CfgError(f"cfg: unexpected character {body[pos]!r}")
        pos = m.end()
        if m.lastgroup:
            toks.append((m.lastgroup, m.group(m.lastgroup)))
    i = 0

    def value() -> object:
        nonlocal i
        k, t = toks[i]
        i += 1
        if k == "num":
            return int(t)
        if k == "str":
            return t[1:-1]
        if k == "id":
            if t == "TRUE":
                return True
            if t == "FALSE":
                return False
            return ModelValue(t)
        if k == "op" and t == "{":
            items = []
            if toks[i] == ("op", "}"):
                i += 1
                return frozenset()
            while True:
                items.append(value())
                k2, t2 = toks[i]
                i += 1
                if (k2, t2) == ("op", "}"):
                    return frozenset(items)
                if (k2, t2) != ("op", ","):
                    raise CfgError("cfg: expected , or } in set value")
        raise CfgError(f"cfg: bad value token {t!r}")

    section = None
    while i < len(toks):
        k, t = toks[i]
        if k == "id" and t in _SECTION_WORDS:
            section = t
            i += 1
            continue
        if section in ("CONSTANT", "CONSTANTS"):
            if k != "id":
                raise CfgError(f"cfg: expected constant name, got {t!r}")
            name = t
            i += 1
            if i >= len(toks) or toks[i][0] != "op":
                raise CfgError(f"cfg: expected = or <- after {name}")
            op = toks[i][1]
            i += 1
            if op == "=":
                cfg.constants[name] = value()
            elif op == "<-":
                if toks[i][0] != "id":
                    raise CfgError("cfg: expected operator name after <-")
                cfg.overrides[name] = toks[i][1]
                i += 1
            else:
                raise CfgError(f"cfg: expected = or <- after {name}")
            continue
        if k != "id":
            raise CfgError(f"cfg: unexpected token {t!r} in section {section}")
        i += 1
        if section == "INIT":
            cfg.init = t
        elif section == "NEXT":
            cfg.next = t
        elif section == "SPECIFICATION":
            cfg.specification = t
        elif section in ("INVARIANT", "INVARIANTS"):
            cfg.invariants.append(t)
        elif section in ("CONSTRAINT", "CONSTRAINTS"):
            cfg.constraints.append(t)
        elif section in ("ACTION_CONSTRAINT", "ACTION_CONSTRAINTS"):
            cfg.action_constraints.append(t)
        elif section in ("PROPERTY", "PROPERTIES"):
            cfg.properties.append(t)
        elif section == "SYMMETRY":
            cfg.symmetry = t
        elif section == "VIEW":
            cfg.view = t
        elif section == "CHECK_DEADLOCK":
            cfg.check_deadlock = (t == "TRUE")
        else:
            raise CfgError(f"cfg: token {t!r} outside any section")
    for p in pragmas:
        m = re.match(r"LAYOUT\s+(\w+)\s*$", p)
        if m:
            cfg.layout = m.group(1)
            continue
        m = re.match(r"CAPACITY\s+(\w+)\s*=\s*(.+)$", p)
        if m:
            cfg.capacities[m.group(1)] = m.group(2).strip()
            continue
        m = re.match(r"TYPE\s+(\w+)\s*(\\in|\\subseteq)\s+(.+)$", p)
        if m:
            cfg.type_hints[m.group(1)] = (m.group(2), m.group(3).strip())
            continue
        m = re.match(r"KEYED\s+(\w+)\s+BY\s+(\w+)\s*$", p)
        if m:
            cfg.keyed[m.group(1)] = m.group(2)
            continue
        if re.match(r"INIT\s+DEVICE\s*$", p):
            cfg.init_device = True
            continue
        m = re.match(r"PREFIX\s+(\w+)\s+(\w+)\s+(\w+)\s*$", p)
        if m:
            cfg.prefix[m.group(1)] = (m.group(2), m.group(3))
            continue
        raise CfgError(f"cfg: unknown kspec pragma {p!r}")
    return cfg


def load_cfg(path: str) -> Config:
    with open(path, "r", encoding="utf-8") as f:
        return parse_cfg(f.read())
