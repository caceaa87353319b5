"""Test support: the fingerprint-sharded driver over the host stand-in engine, in `world` processes over gloo
(gloo_worker.py), on the CPU."""
import json
import os
import socket
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def gloo_run(name, world, chunk, tmp_path, extra=()):
    """Runs gloo_worker.py on `world` ranks (chunks of `chunk` states; `extra`: "cont", "board") and returns rank 0's
    result; skips when build() has not lowered the model."""
    if not os.path.exists(os.path.join(ROOT, "build", "models", name, "model.h")):
        pytest.skip(f"lowered model {name} not built")
    out = str(tmp_path / f"{name}_{world}.json")
    port = _free_port()
    procs = []
    for rank in range(world):
        env = dict(os.environ, RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, os.path.join(HERE, "gloo_worker.py"), name, out, str(chunk),
                                       *extra], env=env))
    for p in procs:
        assert p.wait(timeout=600) == 0
    return json.load(open(out))
