import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def golden():
    import numpy as np

    def load(name):
        # a fixture may be stored in parts below 1 MB each: name.npz, name.1.npz, name.2.npz, ...
        arrays, part = {}, 0
        path = os.path.join(GOLDEN, name + ".npz")
        while os.path.exists(path):
            with np.load(path) as z:
                arrays.update((k, z[k]) for k in z.files)
            part += 1
            path = os.path.join(GOLDEN, "%s.%d.npz" % (name, part))
        if not arrays:
            raise FileNotFoundError(os.path.join(GOLDEN, name + ".npz"))
        return arrays
    return load
