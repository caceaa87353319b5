"""Generates tests/golden/header_digests.json -- run after `make -C oracle` (needs oracle/_ref/spec), commit the output.

For every registered model (models/MODELS.json and the test-only tests/specs/MODELS.json) it records the sha256 of
the whole generated header and of its model.json metadata.  The body digest in body_digests.json covers only the
one-phase form of Next, the invariants, the constraints and the symmetry code; these pin everything else the
lowering emits: the two-phase site split the GPU runs, SITE_ACTION and the per-site action map of model.json.
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)


def header_digests(name: str, spec: dict) -> dict:
    from kafka_specification_b200.build import tla_search_dirs
    from kafka_specification_b200.lower.model import lower_model
    with open(os.path.join(ROOT, spec["cfg"])) as f:
        m = lower_model(spec["module"], tla_search_dirs(), f.read(), name=name)
    return {"header": hashlib.sha256(m.header.encode()).hexdigest(),
            "meta": hashlib.sha256(json.dumps(m.meta(), sort_keys=True).encode()).hexdigest()}


def main():
    from kafka_specification_b200.build import registry
    out = {name: header_digests(name, spec) for name, spec in registry().items()}
    with open(os.path.join(HERE, "header_digests.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
