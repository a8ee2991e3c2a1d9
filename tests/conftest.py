import os
import sys

import pytest

import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
# the dataset layer's binary cache (modules/load/fast.py) must not land in the user's ~/.cache during test runs
os.environ.setdefault("OEA_CACHE_DIR", os.path.join(tempfile.gettempdir(), "oea_dataset_cache_tests_%d" % os.getpid()))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device, an H100 (select with -m gpu)")
    config.addinivalue_line("markers", "first_hw_run: exercises code that has not yet executed on a GPU; collected last, strict "
                                       "(OEA_QUARANTINE=1 opts into xfail reporting)")


def pytest_collection_modifyitems(config, items):
    """Tests of code that has never executed on a GPU (`first_hw_run`) are collected LAST, so that under `-x` a fault in
    brand-new code cannot cut the hardware-verified tests short, and get a 10-minute timeout (a stuck kernel ends the
    process instead of holding the GPU box).  They are ORDINARY, strict tests: a failure is a failure.
    OEA_QUARANTINE=1 (opt-in, builder's own exploratory runs only) additionally reports their failures as xfailed and
    lists them in the terminal summary.  The marker is removed after the first green run on hardware."""
    late = [it for it in items if it.get_closest_marker("first_hw_run")]
    if late:
        items[:] = [it for it in items if not it.get_closest_marker("first_hw_run")] + late
    for it in late:
        if config.pluginmanager.hasplugin("timeout"):
            it.add_marker(pytest.mark.timeout(600, method="thread"))
        if os.environ.get("OEA_QUARANTINE") == "1":
            it.add_marker(pytest.mark.xfail(strict=False, reason="first run on hardware (quarantined, see tests/conftest.py)"))


def pytest_terminal_summary(terminalreporter, exitstatus, config):
    xfailed = [r for r in terminalreporter.stats.get("xfailed", []) if "first run on hardware" in str(getattr(r, "wasxfail", ""))]
    xpassed = [r for r in terminalreporter.stats.get("xpassed", [])]
    if not xfailed and not xpassed:
        return
    terminalreporter.section("first hardware runs (quarantined)")
    terminalreporter.write_line("%d passed on their first hardware run, %d FAILED:" % (len(xpassed), len(xfailed)))
    for r in xfailed:
        crash = getattr(r.longrepr, "reprcrash", None)
        text = str(r.longrepr).strip().splitlines()
        where = "%s:%s: %s" % (os.path.basename(crash.path), crash.lineno, crash.message.splitlines()[0]) if crash else \
            (text[-1] if text else "")
        terminalreporter.write_line("  FAILED %s :: %s" % (r.nodeid, where[:300]))


@pytest.fixture(scope="session")
def cuda_device():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")
