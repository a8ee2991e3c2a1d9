"""GPU: the flagged-row optimiser (rowopt_flagged_body) on the device at the bench's row space, 200 000 entity rows and
600 relation rows (tests/rowopt_flag_cases.py has the patterns and the float32 restatement).  It runs through
oea_rowopt_apply_pair and through the one-launch fed step: with 20 000 positives the step's grid is one resident wave,
as in the bench, and each warp has one window; with 64 positives the grid is small and each warp walks many windows."""
import numpy as np
import pytest
import torch

from tests.rowopt_flag_cases import PATTERNS, LR, check_update, expect_update, place, run_fed_step, seed_of

pytestmark = pytest.mark.gpu

DIMS = (75, 100)                  # pitch 76 (padding columns) and the bench's 100
BASE_A, BASE_B = 200000, 600


@pytest.fixture(scope="module")
def gpu_engine():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openea_b200 import engine as eng
    return eng


@pytest.mark.parametrize("opt", ["Adagrad", "SGD"])
@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("pattern", sorted(PATTERNS))
def test_pair_optimiser_updates_exactly_the_flagged_rows_on_the_device(gpu_engine, pattern, dim, opt):
    trainer, before = place(gpu_engine, np.random.default_rng(seed_of(pattern, dim, opt)), pattern, dim, opt, "cuda",
                            BASE_A, BASE_B)
    trainer.apply()
    torch.cuda.synchronize()
    check_update(trainer, expect_update(before, opt, LR))


@pytest.mark.parametrize("n_pos", [20000, 64])
@pytest.mark.parametrize("opt", ["Adagrad", "SGD"])
@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("pattern", sorted(PATTERNS))
def test_one_launch_fed_step_updates_placed_and_batch_rows_on_the_device(gpu_engine, pattern, dim, opt, n_pos):
    seed = seed_of(pattern, dim, opt, n_pos)
    trainer, _ = place(gpu_engine, np.random.default_rng(seed), pattern, dim, opt, "cuda", BASE_A, BASE_B)
    run_fed_step(gpu_engine, trainer, pattern, dim, opt, "cuda", BASE_A, BASE_B, seed, n_pos=n_pos)
