import importlib
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def pkg():
    p = importlib.import_module("rwkv-cpp-accelerated_b200")
    p.build.build_all(force=False)
    return p


@pytest.fixture(scope="session")
def model_dir(tmp_path_factory):
    base = os.environ.get("RWKV_B200_TEST_DIR")
    if base:
        os.makedirs(base, exist_ok=True)
        return base
    return str(tmp_path_factory.mktemp("models"))


@pytest.fixture(scope="session")
def make_model(pkg, model_dir):
    """make_model(L, E, seed) -> path of a cached synthetic reference-format .bin"""
    def _make(L, E, seed=20240924):
        path = os.path.join(model_dir, "syn_L%d_E%d_s%d.bin" % (L, E, seed))
        if not os.path.exists(path):
            pkg.build.genmodel(L, E, seed, path)
        return path
    return _make
