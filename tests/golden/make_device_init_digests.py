"""Generates tests/golden/device_init_header_digests.json -- run after `make -C oracle` (needs oracle/_ref/spec), commit
the output.

The same record as header_digests.json (sha256 of the whole generated header and of its model.json metadata), for the
models that test the device form of Init (tests/specs/MODELS_device_init.json): a change of their generated code,
including init_candidate(), shows up as a changed digest.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from golden.make_header_digests import header_digests  # noqa: E402


def main():
    from kafka_specification_b200.build import device_init_registry
    out = {name: header_digests(name, spec) for name, spec in device_init_registry().items()}
    with open(os.path.join(HERE, "device_init_header_digests.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
