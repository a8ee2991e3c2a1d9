"""CPU: set_args / set_kgs / init / run / test / save of TransR on the micro synthetic dataset, through
tests/emu/fake_cuda.py (torch's CUDA surface faked, liboea's entry points on the warp emulator library of
tests/emu/build_emu_transr.py), with presets.transr —
the values of the reference's run/args/transr_args_15K.json."""
import os
import subprocess
import sys

import pytest

from openea_b200 import presets
from tests.emu import build_emu_transr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUNNER = os.path.join(ROOT, "tests", "emu", "fake_cuda.py")


def test_transr_preset_is_the_shipped_configuration():
    a = presets.transr()
    assert (a.embedding_module, a.alignment_module, a.loss, a.loss_norm, a.margin) == ("TransR", "sharing", "margin-based", "L2", 1.5)
    assert (a.optimizer, a.learning_rate, a.batch_size, a.neg_sampling, a.neg_triple_num) == ("Adagrad", 0.01, 5000, "uniform", 1)
    assert (a.dim, a.init, a.ent_l2_norm, a.rel_l2_norm, a.eval_metric, a.eval_norm) == (100, "normal", True, True, "inner", False)


def test_transr_lifecycle_on_the_emulator(tmp_path):
    lib = build_emu_transr.build()
    if lib is None:
        pytest.skip("no CUDA headers for the emulator build")
    env = dict(os.environ, OEA_EMU_LIB=lib)           # the runner's emulated library, with the TransR entry points
    res = subprocess.run([sys.executable, RUNNER, "lifecycle", "TransR", str(tmp_path)], capture_output=True, text=True,
                         timeout=900, cwd=ROOT, env=env)
    assert res.returncode == 0, res.stdout[-1500:] + res.stderr[-2500:]
    assert "lifecycle ok: TransR" in res.stdout
    assert "avg. triple loss" in res.stdout and "Training ends" in res.stdout
