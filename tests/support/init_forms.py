"""Test support: the MiniDecode models (tests/specs/MiniDecode.tla) whose device Init has 2^32 candidates or more, too
many for the host to enumerate -- a plain mixed-radix decode of their generators and their solutions in closed form.

The decode is written from the spec, not from the lowering: the generators of a branch count in source order, the
first one least significant; x \\in a .. b is digit value - a; SUBSET Big has bit i for the i-th model value of Big in
name order.  Each model has one branch."""
from __future__ import annotations

# every variable's value where the model's Init fixes it, as TLC prints it
DEFAULTS = {"a": "0", "s": '"x"', "t": '<<0, FALSE, "x">>', "r": "[u |-> 0, v |-> 0]",
            "nest": "[k |-> (p1 :> 0 @@ p2 :> 0), p |-> [q |-> 0, w |-> FALSE]]", "u": "none",
            "x": "0", "y": "0", "z": "0", "sub": "{}"}
BIG = [f"b{i:02d}" for i in range(1, 35)]
SPACE = {"minidecode_ranges": 65536 * 65537 * 4, "minidecode_edge": 1 << 32, "minidecode_subsets": 1 << 34}
LARGE = list(SPACE)


def state_text(**values) -> str:
    return "\n".join(f"/\\ {v} = {values.get(v, d)}" for v, d in DEFAULTS.items())


def decode(name: str, idx: int) -> str | None:
    """The text of candidate idx of model `name` if it satisfies the branch's filters, else None."""
    assert 0 <= idx < SPACE[name]
    if name == "minidecode_ranges":            # x \in 0..65535, y \in 0..65536, z \in 0..3, x = y % 65536
        x, y, z = idx % 65536, idx // 65536 % 65537, idx // (65536 * 65537)
        return state_text(x=x, y=y, z=z) if x == y % 65536 else None
    if name == "minidecode_edge":              # x \in 0..65535, y \in 0..65535, x = y
        x, y = idx % 65536, idx // 65536
        return state_text(x=x, y=y) if x == y else None
    sub = [BIG[i] for i in range(34) if idx >> i & 1]    # sub \in SUBSET Big, Cardinality(sub) <= 1
    return state_text(sub="{" + ", ".join(sub) + "}") if len(sub) <= 1 else None


def solution_indices(name: str) -> list[int]:
    """The candidate index of every solution, in closed form (each solution is generated once)."""
    if name == "minidecode_ranges":
        return [y % 65536 + 65536 * (y + 65537 * z) for z in range(4) for y in range(65537)]
    if name == "minidecode_edge":
        return [x + 65536 * x for x in range(65536)]
    return [0] + [1 << i for i in range(34)]


def boundary_indices(name: str) -> list[int]:
    """0, 1, around 2^32, the last index and the solutions nearest above 2^32 -- where a 32-bit index would wrap."""
    last = SPACE[name] - 1
    out = {0, 1, (1 << 32) - 1, (1 << 32), (1 << 32) + 1, last, last - 1}
    out |= {i for i in solution_indices(name) if (1 << 32) - 70000 <= i <= (1 << 32) + 140000}
    return sorted(i for i in out if 0 <= i <= last)
