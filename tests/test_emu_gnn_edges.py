"""CPU: the path-(ii) kernels at their edges — every SpMM row length class (gather tails, hub threshold, segment and
per-warp share edges), every VEC bucket, strides and the fused epilogues in their documented order, the hub plan's
absence, the edge softmax on equal, widely spread and huge logits in node and edge-logit mode with its backward on the
leaky kink, SDDMM with strides, transpose_perm with duplicated entries, and the L1 alignment loss on its degenerate
pairs — executed from the product's kernel source on the warp emulator (tests/emu) through the product's host layer and
the raw C-ABI, against the float64 references of tests/gnn_edge_cases.py.  tests/test_zz_gnn_edges_gpu.py runs the same
cases on the GPU."""
import ctypes as C

import pytest
import torch

from tests import gnn_edge_cases as gc
from tests.emu import build_emu


@pytest.fixture()
def dev(monkeypatch):
    lib = build_emu.load()
    build_emu.patch_engine(monkeypatch, lib)
    d = C.c_int(0)
    assert lib.cudaGetDevice(C.byref(d)) != 0, "a CUDA device is visible: the grid would not be sized by the fallback"
    return torch.device("cpu")


@pytest.mark.parametrize("i,d", list(enumerate(gc.SPMM_DIMS)))
def test_emulated_spmm_exact_at_every_row_length_and_width(dev, i, d):
    gc.case_spmm_widths(dev, i, d)


@pytest.mark.parametrize("d", [4, 132, 388, 512])
def test_emulated_spmm_real_valued_within_the_fp32_bound(dev, d):
    gc.case_spmm_bound(dev, d)


def test_emulated_spmm_substituted_values_and_transpose_with_hub_columns(dev):
    gc.case_spmm_vals_and_transpose(dev)


def test_emulated_spmm_empty_matrix_and_one_row_matrices(dev):
    gc.case_spmm_empty_and_one_row(dev)


def test_emulated_spmm_without_hub_plan_computes_every_row(dev):
    gc.case_spmm_no_hub_plan(dev)


def test_emulated_spmm_rejects_bad_widths_and_unaligned_x(dev):
    gc.case_spmm_rejections(dev)


@pytest.mark.parametrize("edge_mode", [False, True])
def test_emulated_edge_softmax_exact_on_equal_logits(dev, edge_mode):
    gc.case_softmax_exact_fwd(dev, edge_mode)


@pytest.mark.parametrize("edge_mode", [False, True])
def test_emulated_edge_softmax_within_the_expf_bound(dev, edge_mode):
    gc.case_softmax_bound(dev, edge_mode, gc.expf_ulps_host)


@pytest.mark.parametrize("edge_mode", [False, True])
def test_emulated_edge_softmax_backward_exact_on_the_kink(dev, edge_mode):
    gc.case_softmax_bwd_exact(dev, edge_mode)


@pytest.mark.parametrize("edge_mode", [False, True])
def test_emulated_edge_softmax_backward_within_the_fp32_bound(dev, edge_mode):
    gc.case_softmax_bwd_bound(dev, edge_mode, gc.expf_ulps_host)


@pytest.mark.parametrize("d", gc.SDDMM_DIMS)
def test_emulated_sddmm_with_strides(dev, d):
    gc.case_sddmm(dev, d, exact=True)
    gc.case_sddmm(dev, d, exact=False)


def test_emulated_edge_softmax_and_sddmm_argument_checks(dev):
    gc.case_softmax_arguments(dev)


def test_emulated_transpose_perm_with_duplicated_entries(dev):
    gc.case_transpose_perm(dev)


@pytest.mark.parametrize("edge_mode", [False, True])
def test_emulated_aggregate_functions_forward_and_backward(dev, edge_mode):
    gc.case_aggregate_fn(dev, edge_mode, gc.expf_ulps_host)


@pytest.mark.parametrize("dim", gc.LOSS_DIMS)
def test_emulated_align_loss_exact_with_degenerate_pairs(dev, dim):
    for t, k in ((1, 1), (16, 2), (4, 8)):
        gc.case_align_exact(dev, dim, t, k, seed=t)


def test_emulated_align_loss_real_valued_within_the_fp32_bound(dev):
    gc.case_align_bound(dev, 33, 7, 25)
    gc.case_align_bound(dev, 300, 40, 3, hub=True)


def test_emulated_align_loss_rejects_empty_batches(dev):
    gc.case_align_rejections(dev)
