"""GPU: the edge cases of tests/test_emu_gnn_edges.py on the device, plus what the emulator cannot reach: SpMM over more
than four resident waves of the H100 (multi_processor_count × 64 warps) so that the grid-stride loop runs, SpMM
determinism on real-valued data with hub rows, the edge softmax against the documented error of __expf at logit spreads
up to ~80 and beyond, and the alignment loss at t = 100 000 with one hub entity in 10 % of the negatives."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from tests import gnn_edge_cases as gc

pytestmark = pytest.mark.gpu


@pytest.fixture()
def dev(cuda_device):
    return cuda_device


def _wave(dev):
    """Warps in one resident wave: 64 per SM."""
    return torch.cuda.get_device_properties(dev).multi_processor_count * 64


@pytest.mark.parametrize("i,d", list(enumerate(gc.SPMM_DIMS)))
def test_spmm_exact_at_every_row_length_and_width(dev, i, d):
    gc.case_spmm_widths(dev, i, d)


@pytest.mark.parametrize("d", [4, 132, 388, 512])
def test_spmm_real_valued_within_the_fp32_bound(dev, d):
    gc.case_spmm_bound(dev, d)


def test_spmm_substituted_values_and_transpose_with_hub_columns(dev):
    gc.case_spmm_vals_and_transpose(dev)


def test_spmm_empty_matrix_and_one_row_matrices(dev):
    gc.case_spmm_empty_and_one_row(dev)


def test_spmm_without_hub_plan_computes_every_row(dev):
    gc.case_spmm_no_hub_plan(dev)


def test_spmm_rejects_bad_widths_and_unaligned_x(dev):
    gc.case_spmm_rejections(dev)


def _many_rows(rng, n_rows, n_cols):
    """n_rows short rows (0 … 40 non-zeros, integer values) with the ROW_LENGTHS rows spread among them."""
    lengths = rng.integers(0, 41, n_rows)
    hub_at = rng.choice(n_rows, len(gc.ROW_LENGTHS), replace=False)
    lengths[hub_at] = gc.ROW_LENGTHS
    indptr = np.concatenate([[0], np.cumsum(lengths)])
    cols = np.empty(int(indptr[-1]), np.int64)
    for r in np.flatnonzero(lengths > 40):
        cols[indptr[r]:indptr[r + 1]] = np.sort(rng.choice(n_cols, lengths[r], replace=False))
    short = np.flatnonzero((lengths > 0) & (lengths <= 40))
    for r in short:                                        # 41 distinct columns from a random window: no duplicates
        s0 = rng.integers(0, n_cols - 41)
        cols[indptr[r]:indptr[r + 1]] = s0 + np.sort(rng.choice(41, lengths[r], replace=False))
    return sp.csr_matrix((gc.nonzero_ints(rng, cols.size), cols, indptr), shape=(n_rows, n_cols))


@pytest.mark.parametrize("d", [4, 256, 512])
def test_spmm_over_four_resident_waves(dev, d):
    """More rows than 4 × (SMs × 64) warps, hub rows among them: every row once, whatever pass of the grid-stride loop
    reaches it, bit for bit in exact mode, strided with all three epilogues."""
    rng = np.random.default_rng(d)
    n_rows = 4 * _wave(dev) + 77
    a = _many_rows(rng, n_rows, 4200)
    DA = gc.gnn.DeviceCsr(a, dev)
    assert DA.long_rows.numel() == 10
    X = gc.ints(rng, (a.shape[1], d))
    gc.check_spmm_exact(dev, DA, a, X)
    gc.check_spmm_exact(dev, DA, a, X, ldx=d + 4, ldy=d + 8, relu=True, mask=gc.ints(rng, (n_rows, d), -1, 1), beta=0.5,
                        y_old=gc.ints(rng, (n_rows, d)))


def test_spmm_is_deterministic_with_hub_rows(dev):
    """'No atomics, deterministic': two calls on real-valued data with hub rows give the same bits."""
    rng = np.random.default_rng(11)
    a = gc.csr_rows(rng, rng.permutation(gc.ROW_LENGTHS * 4), 4200, "real")
    DA = gc.gnn.DeviceCsr(a, dev)
    for d in (132, 512):
        X = torch.from_numpy(rng.standard_normal((a.shape[1], d)).astype(np.float32)).to(dev)
        y1, y2 = gc.gnn.spmm(DA, X).cpu().numpy(), gc.gnn.spmm(DA, X).cpu().numpy()
        assert np.array_equal(y1.view(np.int32), y2.view(np.int32))


@pytest.mark.parametrize("edge_mode", [False, True])
def test_edge_softmax_exact_on_equal_logits(dev, edge_mode):
    gc.case_softmax_exact_fwd(dev, edge_mode)


@pytest.mark.parametrize("spread", [40.0, 100.0, 320.0, 400.0])
@pytest.mark.parametrize("edge_mode", [False, True])
def test_edge_softmax_within_the_expf_bound(dev, edge_mode, spread):
    """__expf's documented 2 + floor(1.173·|x|) ulp, with exponent arguments up to ~80 inside the rows (and far below,
    where the exponential underflows).  The worst err / bound is printed."""
    worst = 0.0
    for seed in range(3):
        worst = max(worst, gc.case_softmax_bound(dev, edge_mode, gc.expf_ulps_device, seed=seed, spread=spread)[-1])
    print("edge softmax edge_mode=%s spread=%g: max err/bound %.4g" % (edge_mode, spread, worst))


@pytest.mark.parametrize("edge_mode", [False, True])
def test_edge_softmax_backward_exact_on_the_kink(dev, edge_mode):
    gc.case_softmax_bwd_exact(dev, edge_mode)


@pytest.mark.parametrize("edge_mode", [False, True])
def test_edge_softmax_backward_within_the_fp32_bound(dev, edge_mode):
    gc.case_softmax_bwd_bound(dev, edge_mode, gc.expf_ulps_device)


@pytest.mark.parametrize("d", gc.SDDMM_DIMS)
def test_sddmm_with_strides(dev, d):
    gc.case_sddmm(dev, d, exact=True)
    gc.case_sddmm(dev, d, exact=False)


def test_edge_softmax_and_sddmm_argument_checks(dev):
    gc.case_softmax_arguments(dev)


def test_transpose_perm_with_duplicated_entries(dev):
    gc.case_transpose_perm(dev)


@pytest.mark.parametrize("edge_mode", [False, True])
def test_aggregate_functions_forward_and_backward(dev, edge_mode):
    gc.case_aggregate_fn(dev, edge_mode, gc.expf_ulps_device)


@pytest.mark.parametrize("dim", gc.LOSS_DIMS)
def test_align_loss_exact_with_degenerate_pairs(dev, dim):
    for t, k in ((1, 1), (16, 2), (4, 8), (1024, 4)):
        gc.case_align_exact(dev, dim, t, k, seed=t)


def test_align_loss_real_valued_within_the_fp32_bound(dev):
    gc.case_align_bound(dev, 33, 7, 25)
    gc.case_align_bound(dev, 300, 40, 3, hub=True)


def test_align_loss_at_100k_pairs_with_a_hub_entity(dev):
    gc.case_align_bound(dev, 100, 100_000, 5, hub=True, ref_device=dev)


def test_align_loss_rejects_empty_batches(dev):
    gc.case_align_rejections(dev)
