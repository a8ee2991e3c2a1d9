"""CPU: the flagged-row optimiser (rowopt_flagged_body in oea_rowopt.cuh) on the warp emulator, driven through
oea_rowopt_apply_pair and through the one-launch fed step (duo and grouped scorers), with row flags and gradients placed
before the call.  The cooperative launch runs as one block here, so each warp walks many 32-quad windows.

Flagged rows must equal a NumPy float32 restatement of TF1 Adagrad / SGD; unflagged rows keep their weight, slot and
gradient bit for bit; afterwards every flag and every flagged gradient row is zero and padding columns are unchanged
(tests/rowopt_flag_cases.py has the patterns)."""
import ctypes as C

import numpy as np
import pytest

from tests.rowopt_flag_cases import PATTERNS, LR, check_update, expect_update, place, run_fed_step, seed_of

DIMS = (4, 75, 100, 128)          # pitches 4, 76, 100, 128
BASE_A, BASE_B = 1200, 17         # one block of 4 (duo) or 8 (grouped) warps: 75 or 38 quads of A per warp


@pytest.fixture()
def emu_engine(monkeypatch):
    from openea_b200 import engine as eng
    from openea_b200 import lib as L
    from tests.emu import build_emu
    so = build_emu.build()
    if so is None:
        pytest.skip("no CUDA headers for the emulator build")
    lib = C.CDLL(so)
    for name, (res, args) in L.SIGNATURES.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    monkeypatch.setattr(L, "load", lambda: lib)
    monkeypatch.setattr(eng, "_stream_ptr", lambda: C.c_void_p(0))
    return eng


@pytest.mark.parametrize("opt", ["Adagrad", "SGD"])
@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("pattern", sorted(PATTERNS))
def test_emulated_pair_optimiser_updates_exactly_the_flagged_rows(emu_engine, pattern, dim, opt):
    trainer, before = place(emu_engine, np.random.default_rng(seed_of(pattern, dim, opt)), pattern, dim, opt, "cpu",
                            BASE_A, BASE_B)
    trainer.apply()
    check_update(trainer, expect_update(before, opt, LR))


@pytest.mark.parametrize("k", [3, 17])
@pytest.mark.parametrize("opt", ["Adagrad", "SGD"])
@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("pattern", sorted(PATTERNS))
def test_emulated_one_launch_fed_step_updates_placed_and_batch_rows(emu_engine, pattern, dim, opt, k):
    """k_step_fed_duo (k <= 16) and k_step_fed_grouped (k = 17): the placed rows are updated together with the rows
    the step's own batch flags."""
    seed = seed_of(pattern, dim, opt, k)
    trainer, _ = place(emu_engine, np.random.default_rng(seed), pattern, dim, opt, "cpu", BASE_A, BASE_B)
    run_fed_step(emu_engine, trainer, pattern, dim, opt, "cpu", BASE_A, BASE_B, seed, n_pos=24, k=k)
