import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import __graft_entry__ as ge  # noqa: E402


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an NVIDIA H100 (sm_90a); select with -m gpu")


@pytest.fixture(scope="session")
def pkg():
    return ge.import_package()


@pytest.fixture(scope="session")
def orc():
    o = ge.import_oracle()
    o.build()
    return o


@pytest.fixture(scope="session")
def model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("models")


@pytest.fixture(scope="session")
def make_model(pkg, model_dir):
    """make_model(shape_name, quant, ctx, seed) -> loader.Model (cached GGUF on disk)."""
    cache = {}

    def _make(shape_name, quant, ctx=64, seed=1234):
        key = (shape_name, quant, seed)
        if key not in cache:
            path = os.path.join(model_dir, f"{shape_name}-{quant}-{seed}.gguf")
            pkg.synth.write_model(path, shape_name, quant, seed=seed)
            cache[key] = path
        return pkg.load_model(cache[key], ctx)

    return _make
