import os
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def asset_root():
    """Materialised assets/ tree (synthetic FLAME model + shipped topology); cwd is set to it because
    the reference-compatible constructors use the reference's relative paths."""
    from smirk_b200 import synth_assets
    root = synth_assets.materialize(os.path.join(tempfile.gettempdir(), "smk_assets_tests_%d" % os.getuid()))
    old = os.getcwd()
    os.chdir(root)
    yield root
    os.chdir(old)


@pytest.fixture(scope="session")
def native_lib():
    from smirk_b200 import build, _lib
    build.build()
    return _lib.lib()


@pytest.fixture(scope="session")
def golden():
    import numpy as np

    def load(name):
        z = np.load(os.path.join(GOLD, name + ".npz"))
        return {k: z[k] for k in z.files}
    return load
