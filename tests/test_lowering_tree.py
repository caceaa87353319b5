"""Every generated header and model.json, byte for byte, against the digests recorded in tests/golden/header_digests.json.

The body digest (body_digests.json) covers only the one-phase form of Next; this also pins the two-phase form the GPU
runs (site_mask / site_body, the site groups), SITE_ACTION and the per-site action map of model.json.
"""
import json
import os

from conftest import ROOT, needs_reference
from golden.make_header_digests import header_digests


@needs_reference
def test_every_model_lowers_to_the_recorded_header_and_metadata():
    from kafka_specification_b200.build import registry
    with open(os.path.join(ROOT, "tests", "golden", "header_digests.json")) as f:
        golden = json.load(f)
    reg = registry()
    assert set(golden) == set(reg)
    changed = [name for name, spec in reg.items() if header_digests(name, spec) != golden[name]]
    assert not changed, f"generated header or model.json changed for {changed}"
