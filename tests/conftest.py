import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def load_golden(name):
    """-> {case: {key: array}} from tests/golden/<name>.npz and its parts <name>.<case>.npz (files stay under 1 MB)"""
    cases = {}
    for f in sorted(os.listdir(GOLDEN)):
        if f == name + ".npz" or (f.startswith(name + ".") and f.endswith(".npz")):
            z = np.load(os.path.join(GOLDEN, f))
            for full in z.files:
                case, key = full.split("/", 1)
                cases.setdefault(case, {})[key] = z[full]
    return cases


@pytest.fixture(scope="session")
def oracle_lib():
    import oracle.oracle as orc
    orc.build()          # gcc is in the image on both boxes; _ref only where the reference exists
    return orc.Oracle()


@pytest.fixture(scope="session")
def ref_lib():
    import oracle.oracle as orc
    if not orc.have_ref():
        pytest.skip("oracle/_ref not built (needs /root/reference)")
    return orc.Ref(threads=1)
