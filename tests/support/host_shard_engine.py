"""CPU stand-in for one rank of the sharded engine (tests only), see the hs_* calls of host_model.cpp."""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from hostmodel import HostModel


class HostShardEngine:
    def __init__(self, name: str, rank: int, world: int, chunk_states: int = 1000):
        self.model = HostModel.for_built_model(name)
        self.lib = self.model.lib
        self.rank, self.world = rank, world
        self.h = self.lib.hs_create(rank, world)
        self.row_words = self.lib.hs_row_words()
        self.chunk_states = chunk_states
        self.device = torch.device("cpu")
        self._recv_rows = 0
        self._recv = None
        self._incoming_total = 0

    def begin(self):
        self.lib.hs_begin(self.h)

    def seed_init(self):
        self.lib.hs_seed_init(self.h)

    def expand(self, first, count):
        self.lib.hs_expand(self.h, first, count)

    def counts(self):
        buf = np.zeros(8, dtype=np.uint64)
        self.lib.hs_counts(self.h, buf.ctypes.data)
        self._recv = None
        return [int(buf[d]) for d in range(self.world)]

    def _view(self, ptr, nwords):
        if nwords == 0:
            return torch.empty(0, dtype=torch.int64)
        return torch.from_numpy(np.ctypeslib.as_array(ptr, shape=(nwords,)))

    def send_view(self, dest, rows):
        return self._view(self.lib.hs_send_ptr(self.h, dest), rows * self.row_words)

    def reserve_recv(self, rows):
        if self._recv is None or self._recv.numel() < rows * self.row_words:
            self._recv = torch.zeros(max(rows, 1024) * self.row_words, dtype=torch.int64)

    def recv_view(self, offset_rows, rows):
        return self._recv[offset_rows * self.row_words: (offset_rows + rows) * self.row_words]

    def insert_received(self, rows):
        buf = self._recv[: rows * self.row_words].contiguous().numpy()
        self.lib.hs_insert(self.h, buf.ctypes.data, rows)

    def insert_local(self, rows):
        ptr = self.lib.hs_send_ptr(self.h, 0)
        self.lib.hs_insert(self.h, ctypes.cast(ptr, ctypes.c_void_p), rows)

    def reset_cand(self):
        self.lib.hs_reset_cand(self.h)

    def level_done(self):
        a, b = ctypes.c_uint64(), ctypes.c_uint64()
        self.lib.hs_level_done(self.h, ctypes.byref(a), ctypes.byref(b))
        return int(a.value), int(b.value)

    def finish(self):
        pass

    def _raw(self):
        st = np.zeros(8, dtype=np.uint64)
        self.lib.hs_stats(self.h, st.ctypes.data)
        return st

    def stats(self):
        st = self._raw()
        return {"distinct": int(st[0]), "generated": int(st[1]), "deadlocks": int(st[2]), "fail": int(st[3])}

    def _record(self):
        out = np.zeros(self.row_words + 4, dtype=np.uint64)
        inv = self.lib.hs_violation_record(self.h, out.ctypes.data)
        return inv, out

    def violation(self):
        inv, out = self._record()
        if inv < 0:
            return None
        W = self.row_words - 1
        return {"kind": "invariant", "invariant": inv, "level": int(out[W + 2]), "fingerprint": int(out[W + 1])}

    def violation_record(self):
        inv, out = self._record()
        if inv < 0:
            return None
        W = self.row_words - 1
        return [int(x) for x in out[:W]], int(out[W])

    def state_and_parent(self, idx):
        out = np.zeros(self.row_words, dtype=np.uint64)
        self.lib.hs_state_and_parent(self.h, idx, out.ctypes.data)
        return [int(x) for x in out[:-1]], int(out[-1])

    def is_successor(self, a, b) -> int:
        """The action id of a successor of state a under expand() equal to b, or -1."""
        rows, actions = self.model.successors(a)
        hit = np.flatnonzero(np.all(rows == np.asarray(b, dtype=np.uint64), axis=1))
        return int(actions[hit[0]]) if len(hit) else -1

    def is_init(self, a) -> int:
        return int(bool(np.all(self.model.init_states() == np.asarray(a, dtype=np.uint64), axis=1).any()))
