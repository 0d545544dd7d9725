import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a GPU machine)")
    config.addinivalue_line("markers", "slow: multi-GB allocations (full llama2-7B shape)")


@pytest.fixture(scope="session")
def stories15m(tmp_path_factory, oracle):
    """Path of a stories15M-shaped checkpoint file with seeded synthetic weights
    (oracle_lib.write_stories15m_checkpoint; the golden fixtures are computed on it)."""
    return oracle.write_stories15m_checkpoint(str(tmp_path_factory.mktemp("ckpt") / "stories15M.bin"))


@pytest.fixture(scope="session")
def oracle():
    import oracle_lib
    oracle_lib.build_oracle()
    return oracle_lib


@pytest.fixture(scope="session")
def l2b():
    import llama2_zig_b200
    return llama2_zig_b200
