"""Test support: the whole-store audit of a GPU run (host_model.cpp) and a reference of the engine's fingerprints.

``audit_checker(ck, levels, distinct)`` reads every stored state and parent word of a finished or stopped run and checks them
against the lowered Next compiled for the host from the same ``model.h`` (init, edges, uniqueness, closure; see
audit_store in host_model.cpp), then compares the totals the audit recomputes from the stored states with the run's stats and
coverage, and the reported counterexample with the one ``build_trace``'s rule picks among the violators the engine
records: deadlocks first, then the smallest fingerprint, then the smallest parent word.

The reference fingerprints below are written from the definitions in kmc_engine.cu (fmix64, fingerprint, fmix64b,
key_of, bucket_of, owner_of), once over NumPy arrays and once over Python ints.
"""
from __future__ import annotations

import ctypes

import numpy as np

from hostmodel import HostModel

NO_PARENT = 0x0000FFFFFFFFFFFF
VIOL_RING = 1 << 16          # rows of the engine's violator ring; past it the reported pick is not deterministic
M64 = (1 << 64) - 1
GOLDEN_RATIO = 0x9E3779B97F4A7C15
KEY_SEED = 0xD6E8FEB86659FD93


class AuditError(AssertionError):
    """A failed audit; the message starts with the name of the check."""


# ------------------------------------------------------------------------------------------------ reference hashes
def fmix64_int(x: int) -> int:
    x ^= x >> 33
    x = (x * 0xFF51AFD7ED558CCD) & M64
    x ^= x >> 33
    x = (x * 0xC4CEB9FE1A85EC53) & M64
    return x ^ (x >> 33)


def fmix64b_int(x: int) -> int:
    x ^= x >> 30
    x = (x * 0xBF58476D1CE4E5B9) & M64
    x ^= x >> 27
    x = (x * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def fingerprint_int(words, state_bits: int) -> int:
    """64-bit fingerprint of one packed state: a bijection up to 63 bits, else a chain of fmix64 (never 0)."""
    if state_bits <= 63:
        return fmix64_int((words[0] + 1) & M64)
    h = fmix64_int((words[0] + GOLDEN_RATIO) & M64)
    for i in range(1, len(words)):
        h = fmix64_int(h ^ ((words[i] + GOLDEN_RATIO * (i + 1)) & M64))
    return h or 1


def key_of_int(words, fp: int, all_ones_possible: bool = False) -> tuple[int, int]:
    """128-bit set key: the two words themselves (two-word states that never pack to all-ones), else the fingerprint
    and an independent fmix64b chain, with the empty-slot pattern (all-ones) escaped."""
    if len(words) == 2 and not all_ones_possible:
        return words[0], words[1]
    h = fmix64b_int(words[0] ^ KEY_SEED)
    for w in words[1:]:
        h = fmix64b_int((((h << 7) | (h >> 57)) & M64) ^ w)
    if fp & h == M64:
        h ^= 1
    return fp, h


def bucket_of_int(fp: int, bucket_mask: int) -> int:
    return (fp ^ (fp >> 31)) & bucket_mask


def owner_of_int(fp: int, world: int) -> int:
    return ((fp >> 32) * world) >> 32


def _u64(x) -> np.uint64:
    return np.uint64(x)


def fmix64(x: np.ndarray) -> np.ndarray:
    x = x ^ (x >> _u64(33))
    x = x * _u64(0xFF51AFD7ED558CCD)
    x = x ^ (x >> _u64(33))
    x = x * _u64(0xC4CEB9FE1A85EC53)
    return x ^ (x >> _u64(33))


def fmix64b(x: np.ndarray) -> np.ndarray:
    x = x ^ (x >> _u64(30))
    x = x * _u64(0xBF58476D1CE4E5B9)
    x = x ^ (x >> _u64(27))
    x = x * _u64(0x94D049BB133111EB)
    return x ^ (x >> _u64(31))


def fingerprint(rows: np.ndarray, state_bits: int) -> np.ndarray:
    rows = np.asarray(rows, dtype=np.uint64)
    with np.errstate(over="ignore"):
        if state_bits <= 63:
            return fmix64(rows[:, 0] + _u64(1))
        h = fmix64(rows[:, 0] + _u64(GOLDEN_RATIO))
        for i in range(1, rows.shape[1]):
            h = fmix64(h ^ (rows[:, i] + _u64((GOLDEN_RATIO * (i + 1)) & M64)))
    return np.where(h == 0, _u64(1), h)


def key_of(rows: np.ndarray, fp: np.ndarray, all_ones_possible: bool = False) -> np.ndarray:
    """[n, 2] keys (lo, hi)."""
    rows = np.asarray(rows, dtype=np.uint64)
    if rows.shape[1] == 2 and not all_ones_possible:
        return rows.copy()
    with np.errstate(over="ignore"):
        h = fmix64b(rows[:, 0] ^ _u64(KEY_SEED))
        for i in range(1, rows.shape[1]):
            h = fmix64b(((h << _u64(7)) | (h >> _u64(57))) ^ rows[:, i])
    h = np.where((fp & h) == _u64(M64), h ^ _u64(1), h)
    return np.stack([fp, h], axis=1)


def bucket_of(fp: np.ndarray, bucket_mask: int) -> np.ndarray:
    return (fp ^ (fp >> _u64(31))) & _u64(bucket_mask)


def owner_of(fp: np.ndarray, world: int) -> np.ndarray:
    return ((fp >> _u64(32)) * _u64(world)) >> _u64(32)


# ------------------------------------------------------------------------------------------------ the host library
class AuditLib(HostModel):
    """host_model.cpp compiled against one model header, with the audit's entry points."""

    def fingerprints(self, rows: np.ndarray, canonical: np.ndarray | bool = False) -> np.ndarray:
        """The engine's fingerprint of each row, of its canonical form where `canonical` says so."""
        rows = np.ascontiguousarray(rows, dtype=np.uint64).reshape(-1, self.words)
        canonical = np.broadcast_to(np.asarray(canonical, dtype=bool), (len(rows),))
        src = rows.copy()
        if canonical.any():
            src[canonical] = self.canonicalize(rows[canonical])
        return fingerprint(src, self.state_bits)

    def host_bfs(self, stop_after: int = 0, sites: bool = False) -> dict:
        """Level-ordered host BFS that writes its store in the engine's format, through expand() or, with `sites`, the
        two-phase form (which orbit member is stored follows the order of the form); stops at the first level end that
        holds >= stop_after states (0: never)."""
        r = self.bfs(sites=sites, stop_at=stop_after)
        if r["fail"]:
            raise RuntimeError(f"{self.name}: host BFS trapped the layout (code {r['fail']})")
        return {"states": r["states"], "parents": r["parents"], "widths": r["widths"], "n_expanded": r["n_expanded"]}

    def check_store(self, states, parents, widths, n_expanded: int, *, check_deadlock: bool,
                    rank_widths: list[list[int]] | None = None, init_rows: np.ndarray | None = None) -> dict:
        """Init, edges, uniqueness and closure of a store; returns the recomputed totals and the violators of the first
        level end that has any.  `widths` are the level widths of one rank's store; for the union of several ranks'
        stores (concatenated in rank order) pass `rank_widths`, one list per rank.  `init_rows` are the generated
        initial states (duplicates included) when the audit is not to enumerate them itself: a device form of Init
        with more than 2^32 candidates, whose solutions the caller knows in closed form."""
        states = np.ascontiguousarray(states, dtype=np.uint64).reshape(-1, self.words)
        parents = np.ascontiguousarray(parents, dtype=np.uint64)
        per_rank = rank_widths if rank_widths is not None else [list(widths)]
        levels, offs = [], [0]
        for w in per_rank:
            levels.append(np.repeat(np.arange(1, len(w) + 1, dtype=np.uint32), np.asarray(w, dtype=np.int64)))
            offs.append(offs[-1] + int(sum(w)))
        level = np.ascontiguousarray(np.concatenate(levels) if levels else np.zeros(0, np.uint32))
        n = len(states)
        if len(parents) != n or offs[-1] != n:
            raise AuditError(f"levels: {n} states, {len(parents)} parent words, level widths summing to {offs[-1]}")
        rank_off = np.asarray(offs, dtype=np.uint64)
        totals = np.zeros(3, dtype=np.uint64)
        act_gen = np.zeros(max(self.num_actions, 1), dtype=np.uint64)
        site_gen = np.zeros(max(self.num_sites, 1), dtype=np.uint64)
        viol_counts = np.zeros(n_expanded + 1, dtype=np.uint64)
        msg = ctypes.create_string_buffer(1024)
        if init_rows is not None:
            init_rows = np.ascontiguousarray(init_rows, dtype=np.uint64).reshape(-1, self.words)
        rc = self.lib.audit_store(states.ctypes.data, parents.ctypes.data, level.ctypes.data, n, rank_off.ctypes.data,
                                  len(per_rank), n_expanded, 1 if check_deadlock else 0,
                                  None if init_rows is None else init_rows.ctypes.data,
                                  0 if init_rows is None else len(init_rows), totals.ctypes.data,
                                  act_gen.ctypes.data, site_gen.ctypes.data, viol_counts.ctypes.data, msg, len(msg))
        if rc != 0:
            raise AuditError(f"{msg.value.decode()}  [{self.name}]")
        n_rows = int(self.lib.audit_violator_rows(None, 0))
        rows = np.zeros((n_rows, self.words + 2), dtype=np.uint64)
        if n_rows:
            self.lib.audit_violator_rows(rows.ctypes.data, n_rows)
        return {"generated": int(totals[0]), "deadlocks": int(totals[1]), "out_of_model": int(totals[2]),
                "action_generated": [int(x) for x in act_gen[: self.num_actions]],
                "site_generated": [int(x) for x in site_gen[: self.num_sites]],
                "violators_per_level_end": [int(x) for x in viol_counts], "violators": rows}


# ------------------------------------------------------------------------------------------------ the audit proper
def expected_violation(a: AuditLib, found: dict) -> dict | None:
    """build_trace's pick among the violators of the first level end that has any: deadlocks first, then the smallest
    fingerprint, then the smallest parent word.  The engine fingerprints every violator, stored or discarded by a
    CONSTRAINT, by its canonical state (its set identity), so under SYMMETRY the pick does not depend on which member
    of an orbit was stored."""
    counts = found["violators_per_level_end"]
    ends = [e for e, c in enumerate(counts) if c]
    if not ends:
        return None
    rows = found["violators"]
    w = a.words
    fps = a.fingerprints(rows[:, :w], True)
    dead = rows[:, w + 1] == np.uint64(M64)
    order = np.lexsort((rows[:, w], fps, ~dead))          # last key first: deadlocks, fingerprint, parent word
    best = int(order[0])
    return {"level_end": ends[0], "count": int(counts[ends[0]]), "rows": rows, "fps": fps, "dead": dead,
            "kind": "deadlock" if dead[best] else "invariant", "invariant": None if dead[best] else int(rows[best, w + 1]),
            "level": ends[0] if dead[best] else ends[0] + 1, "fingerprint": int(fps[best]),
            "words": [int(x) for x in rows[best, :w]], "parent_word": int(rows[best, w])}


def compare(a: AuditLib, found: dict, *, stats: dict, coverage: dict | None, parents: np.ndarray,
            violation: dict | None, record, invariants: list[str]) -> dict | None:
    """The run's totals, coverage and counterexample against what the audit recomputed from the stored states."""
    for k in ("generated", "deadlocks", "out_of_model"):
        if stats[k] != found[k]:
            raise AuditError(f"totals: the run reports {k} = {stats[k]}, its stored states give {found[k]}  [{a.name}]")
    if coverage is not None:
        gen = [x["generated"] for x in coverage["actions"]]
        if gen != found["action_generated"]:
            raise AuditError(f"totals: generated per action {gen} != {found['action_generated']} from the stored states")
        if coverage["sites"] != found["site_generated"]:
            raise AuditError(f"totals: generated per site {coverage['sites']} != {found['site_generated']}")
        init = (parents & np.uint64(NO_PARENT)) == np.uint64(NO_PARENT)
        hist = np.bincount((parents[~init] >> np.uint64(56)).astype(np.int64), minlength=a.num_actions)
        dist = [x["distinct"] for x in coverage["actions"]]
        if dist != [int(x) for x in hist[: a.num_actions]]:
            raise AuditError(f"totals: distinct per action {dist} != the parent words' action ids {hist.tolist()}")
    want = expected_violation(a, found)
    if want is None:
        if violation is not None:
            raise AuditError(f"counterexample: the run reports {violation}, no stored state or successor violates anything")
        return None
    if violation is None:
        raise AuditError(f"counterexample: {want['count']} violators at the end of level {want['level_end']}, "
                         f"the run reports none")
    got_inv = None if violation["kind"] == "deadlock" else invariants.index(violation["invariant"])
    if want["count"] > VIOL_RING:
        # the ring kept an arbitrary VIOL_RING of them: the reported state must be one of the level's violators
        print(f"[audit] {a.name}: {want['count']} violators at the end of level {want['level_end']} exceed the "
              f"ring ({VIOL_RING}); the pick is not deterministic")
        w = a.words
        rows = want["rows"]
        hit = (want["fps"] == np.uint64(violation["fingerprint"])) & (want["dead"] == (violation["kind"] == "deadlock"))
        if got_inv is not None:
            hit &= rows[:, w + 1] == np.uint64(got_inv)
        if record is not None:
            hit &= np.all(rows[:, :w] == np.asarray(record[0], dtype=np.uint64), axis=1) & (rows[:, w] == np.uint64(record[1]))
        level = want["level_end"] + (0 if violation["kind"] == "deadlock" else 1)
        if not hit.any() or violation["level"] != level:
            raise AuditError(f"counterexample: the reported state is not a violator of level end {want['level_end']}")
        return want
    got = (violation["kind"], got_inv, violation["level"], violation["fingerprint"])
    exp = (want["kind"], want["invariant"], want["level"], want["fingerprint"])
    if got != exp:
        raise AuditError(f"counterexample: the run reports (kind, invariant, level, fingerprint) = {got}, build_trace's "
                         f"rule picks {exp} among {want['count']} violators  [{a.name}]")
    if record is not None:
        if (list(record[0]), record[1]) != (want["words"], want["parent_word"]):
            raise AuditError(f"counterexample: kmc_violation_record {record} is not the picked violator "
                             f"{(want['words'], want['parent_word'])}")
        fp = int(a.fingerprints(np.asarray([record[0]], dtype=np.uint64), True)[0])
        if fp != violation["fingerprint"]:
            raise AuditError(f"counterexample: the record's words hash to {fp:#x}, the run reports "
                             f"{violation['fingerprint']:#x}")
    return want


def copy_parents(ck, first: int, count: int) -> np.ndarray:
    buf = np.empty(count, dtype=np.uint64)
    if count:
        ck._check(ck.lib.kmc_copy_parents(ck.ctx, first, count, buf.ctypes.data))
    return buf


def audit_checker(ck, levels: list[int], distinct: int, *, check_deadlock: bool | None = None, audit: AuditLib | None = None,
                  init_rows: np.ndarray | None = None) -> dict:
    """Audit the store of a Checker after a run: `levels` are the widths of the levels the run expanded (RunResult /
    ShardedResult .levels), `distinct` the stored states; the states past the expanded levels are the queue.  The
    report holds the audit's totals and pick, the store and the run's kmc_violation_record (None without a violation).
    `init_rows` (see AuditLib.check_store) are the generated initial states of a device Init too large to enumerate."""
    a = audit or AuditLib.for_built_model(ck.meta["name"])
    if a.digest != ck.meta["digest"]:
        raise AuditError(f"digest: the audit's model.h ({a.digest}) is not the loaded library's ({ck.meta['digest']})")
    states = ck.copy_states(0, distinct)
    parents = copy_parents(ck, 0, distinct)
    widths = list(levels)
    if distinct > sum(widths):
        widths.append(distinct - sum(widths))
    cd = a.check_deadlock if check_deadlock is None else check_deadlock
    found = a.check_store(states, parents, widths, len(levels), check_deadlock=cd, init_rows=init_rows)
    record = ck.violation_record() if ck.violation() else None
    want = compare(a, found, stats=ck.stats(), coverage=ck.coverage(), parents=parents, violation=ck.violation(),
                   record=record, invariants=ck.meta["invariants"])
    return {"found": found, "violation": want, "states": states, "parents": parents, "widths": widths, "record": record}


def host_audit(name: str, sites: bool = True) -> tuple[AuditLib, dict, dict]:
    """The audit of the store that a host BFS of the registered model `name` writes: (AuditLib, the store, the audit's
    findings)."""
    a = AuditLib.for_registered(name)
    st = a.host_bfs(sites=sites)
    found = a.check_store(st["states"], st["parents"], st["widths"], st["n_expanded"], check_deadlock=a.check_deadlock)
    return a, st, found


def expected_orbit(a: AuditLib, found: dict) -> tuple[list[int], int]:
    """The counterexample the documented rule picks, as an orbit: (canonical words, fingerprint of the canonical form),
    computed from the violators alone -- whichever member of each orbit a store happens to hold."""
    w = a.words
    rows = found["violators"]
    dead = rows[:, w + 1] == np.uint64(M64)
    canon = a.canonicalize(rows[:, :w])
    fps = fingerprint(canon, a.state_bits)
    keys = [(0 if d else 1, int(f)) for d, f in zip(dead, fps)]
    best = min(range(len(rows)), key=lambda i: keys[i])
    return [int(x) for x in canon[best]], int(fps[best])
