import json
import os
import sys

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

GOLDEN_DIR = os.path.join(REPO, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90) GPU (select with `-m gpu`)")


@pytest.fixture(scope="session")
def golden():
    data = np.load(os.path.join(GOLDEN_DIR, "reference_vectors.npz"))
    with open(os.path.join(GOLDEN_DIR, "reference_vectors.json")) as f:
        meta = json.load(f)
    return data, meta


def golden_cases():
    with open(os.path.join(GOLDEN_DIR, "reference_vectors.json")) as f:
        return json.load(f)["cases"]


def case_from_meta(c):
    """Regenerate the seeded inputs of a golden case (oracle.make_case) and verify their sha256."""
    import hashlib

    from oracle import aqlm_oracle as O

    case = O.make_case(c["seed"], c["in_features"], c["out_features"], c["num_codebooks"], c["nbits"],
                       c["in_group_size"], c["batch"], c["bias"])
    h = hashlib.sha256()
    for k in ("x", "codes", "codebooks", "scales", "bias"):
        if case[k] is not None:
            h.update(np.ascontiguousarray(case[k]).tobytes())
    assert h.hexdigest() == c["inputs_sha256"], f"input generator drifted for {c['name']}"
    return case
