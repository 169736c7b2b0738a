import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")
    # The C-ABI library is a build artefact (git-ignored).  In a fresh checkout build it before the
    # first test needs it (nvcc cross-compiles for sm_90a without a GPU); an existing library is never rebuilt here.
    lib = os.path.join(ROOT, "torchcde_b200", "csrc", "libtcde_b200.so")
    if not os.path.isfile(lib):
        import shutil
        import subprocess
        if shutil.which("nvcc") and shutil.which("make"):
            subprocess.run(["make", "-C", os.path.join(ROOT, "torchcde_b200", "csrc"), "-j8"], check=False,
                           capture_output=True)


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available() or os.environ.get("TCDE_TRICKS_ON_REFERENCE"):
        return              # (the second case: tests/test_gpu_tricks.py self-checking its logic on the CPU reference)
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


class Golden:
    """Thin reader for the committed reference fixtures (tests/golden/*.npz)."""

    def __init__(self, name):
        self.z = np.load(os.path.join(GOLDEN, name + ".npz"))
        self.count = int(self.z["count"])

    def has(self, key):
        return key in self.z.files

    def t(self, key):
        return torch.from_numpy(self.z[key])

    def s(self, key):
        return str(self.z[key])

    def f(self, key):
        return float(self.z[key])


@pytest.fixture(scope="session")
def golden():
    return Golden


def same(a, b):
    """Bit-level equality that treats NaN == NaN (and +0 == -0, like torch.equal)."""
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    return bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())
