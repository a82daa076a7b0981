import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    # The library continues a Yinyang run with Lloyd passes once a Yinyang iteration proves slower than a Lloyd
    # iteration of the same run (identical results).  The tests that exercise the Yinyang kernels need them to run:
    # the switch is off for the suite and on in the one test that checks it.
    os.environ.setdefault("KMCUDA_B200_YY_ADAPTIVE", "0")


def pytest_collection_modifyitems(config, items):
    # A GPU test that hangs (a kernel waiting on something that never comes) must end the run loudly, not sit there until
    # the caller's limit: with pytest-timeout present every GPU test gets 7 minutes (the slowest takes ~20 s), enforced by
    # the watchdog thread (a signal cannot interrupt a thread blocked inside cudaStreamSynchronize).
    if not config.pluginmanager.hasplugin("timeout"):
        return
    for item in items:
        if item.get_closest_marker("gpu") and not item.get_closest_marker("timeout"):
            item.add_marker(pytest.mark.timeout(int(os.environ.get("KMB_TEST_TIMEOUT", "420")), method="thread"))


@pytest.fixture(scope="session", autouse=True)
def _built():
    """The product library and the C oracle must exist before any test imports them."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("kmcuda_b200_build", os.path.join(ROOT, "kmcuda_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build()
    from oracle import oracle as O
    O.build()
    yield
