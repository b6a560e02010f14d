import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "icassp2022-depression_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session", autouse=True)
def _built_library():
    """Every test run starts from a built C-ABI library (nvcc cross-compiles sm_90a without a GPU)."""
    # build() unconditionally (an incremental `make`: seconds when nothing changed), so the tests always run the
    # binary the tree's sources produce - never a stale pre-built one that merely travelled with the snapshot
    import __graft_entry__

    __graft_entry__.build()
    lib = os.path.join(PKG, "lib", "libb200rnn.so")
    assert os.path.exists(lib), "libb200rnn.so missing and build() did not produce it"
    yield


def load_golden(name):
    import json

    import numpy as np

    data = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(bytes(data["__meta__"]).decode("utf-8"))
    arrays = {}
    for k in data.files:
        if k == "__meta__":
            continue
        if "::" in k:
            a, b = k.split("::")
            arrays.setdefault(a, {})[b] = data[k]
        else:
            arrays[k] = data[k]
    return arrays, meta
