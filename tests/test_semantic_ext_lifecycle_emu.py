"""CPU: set_args / set_kgs / init / run / test / save of RotatE, HolE and BootEA_RotatE on the micro synthetic dataset,
through tests/emu/fake_cuda.py (torch's CUDA surface faked, liboea's entry points on the warp emulator).  BootEA_RotatE
additionally runs with bootstrapping from the first iteration and ε-truncated negatives, so that its alignment loss,
reference-entity similarity and neighbour refresh on re + im execute too."""
import os
import subprocess
import sys

import pytest

from tests.emu import build_emu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUNNER = os.path.join(ROOT, "tests", "emu", "fake_cuda.py")

# the runner's lifecycle with a preset override (one-epoch iterations, bootstrapping and truncated negatives from the start)
BOOTSTRAPPING = """
import sys
sys.path.insert(0, {root!r})
from tests.emu import fake_cuda
fake_cuda.install()
from openea_b200 import presets
base = presets.bootea_rotate
def patched(scale="15K"):
    a = base(scale)
    a.sub_epoch, a.start_bp, a.neg_sampling, a.sim_th, a.min_iter = 1, 1, "truncated", 0.0, 1
    return a
presets.bootea_rotate = patched
fake_cuda.lifecycle("BootEA_RotatE", {folder!r})
"""


def _run(cmd, name):
    if build_emu.build() is None:
        pytest.skip("no CUDA headers for the emulator build")
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert res.returncode == 0, res.stdout[-1500:] + res.stderr[-2500:]
    assert "lifecycle ok: " + name in res.stdout
    return res.stdout


@pytest.mark.parametrize("name", ["RotatE", "HolE", "BootEA_RotatE"])
def test_semantic_ext_lifecycle_on_the_emulator(tmp_path, name):
    out = _run([sys.executable, RUNNER, "lifecycle", name, str(tmp_path)], name)
    if name != "BootEA_RotatE":          # (sub_epoch 10 > the runner's two epochs: BootEA_RotatE only initialises here)
        assert "avg. triple loss" in out and "Training ends" in out


def test_bootea_rotate_bootstraps_on_the_emulator(tmp_path):
    out = _run([sys.executable, "-c", BOOTSTRAPPING.format(root=ROOT, folder=str(tmp_path))], "BootEA_RotatE")
    for line in ("avg. triple loss", "bootstrapping", "generating neighbors of", "Training ends"):
        assert line in out, line
