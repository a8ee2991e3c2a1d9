"""CPU: the kernels of path (ii) (openea_b200/csrc/oea_spmm.cu: warp-per-row SpMM with fused epilogues, hub-row segments +
ordered finalize, edge softmax forward / backward, SDDMM, L1 alignment loss) on the warp emulator of tests/emu against
SciPy / torch-autograd statements of the same operations."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from openea_b200 import lib as L
from tests.emu import build_emu


@pytest.fixture(scope="module")
def emu():
    return build_emu.load()


class HostCsr:
    """oea_csr + oea_spmm_hubs over NumPy buffers, hub segmentation as openea_b200.gnn.DeviceCsr does it."""

    def __init__(self, emu, mat):
        m = sp.csr_matrix(mat, dtype=np.float32)
        m.sort_indices()
        self.m = m
        self.rowptr, self.col, self.val = m.indptr.astype(np.int32), m.indices.astype(np.int32), m.data.astype(np.float32)
        thr, seg = emu.oea_spmm_long_row_threshold(), emu.oea_spmm_segment_nnz()
        nnz_row = np.diff(m.indptr)
        self.long_rows = np.flatnonzero(nnz_row > thr).astype(np.int32)
        n_seg_row = -(-nnz_row[self.long_rows] // seg)
        self.seg_ptr = np.concatenate([[0], np.cumsum(n_seg_row)]).astype(np.int32)
        self.seg_row = np.repeat(np.arange(len(self.long_rows)), n_seg_row).astype(np.int32)
        within = np.arange(int(self.seg_ptr[-1])) - self.seg_ptr[self.seg_row] if len(self.long_rows) else np.zeros(0, np.int64)
        self.seg_start = (m.indptr[self.long_rows][self.seg_row] + within * seg).astype(np.int32) if len(self.long_rows) \
            else np.zeros(0, np.int32)
        self.n_seg = int(self.seg_ptr[-1])

    def csr(self, vals=None):
        v = self.val if vals is None else vals
        return L.Csr(self.rowptr.ctypes.data, self.col.ctypes.data, v.ctypes.data, self.m.shape[0], self.m.shape[1], self.m.nnz)

    def hubs(self):
        p = lambda a: a.ctypes.data if a.size else 0
        return L.SpmmHubs(p(self.long_rows), p(self.seg_ptr), p(self.seg_row), p(self.seg_start), len(self.long_rows), self.n_seg)


def _spmm(emu, A, X, relu=0, mask=None, beta=0.0, Y=None, vals=None):
    d = X.shape[1]
    Y = np.zeros((A.m.shape[0], d), dtype=np.float32) if Y is None else Y
    nbytes = emu.oea_spmm_workspace_bytes(A.n_seg, d)
    ws = np.zeros(max(4, nbytes // 4), dtype=np.float32)
    cs, hb = A.csr(vals), A.hubs()
    rc = emu.oea_spmm_csr(C.byref(cs), C.byref(hb), X.ctypes.data, X.shape[1], Y.ctypes.data, d, d, relu,
                          None if mask is None else mask.ctypes.data, beta, ws.ctypes.data, nbytes, None)
    assert rc == 0
    return Y


@pytest.mark.parametrize("d", [4, 100, 132, 300])
def test_emulated_spmm_with_hub_rows_and_epilogues(emu, d):
    rng = np.random.default_rng(d)
    n, m = 70, 600
    a = sp.random(n, m, density=0.03, random_state=1, format="lil", dtype=np.float32)
    a[3, :] = 0
    a[5, rng.choice(m, 300, replace=False)] = rng.standard_normal(300)          # one hub row: > 256 non-zeros → segments
    a[9, rng.choice(m, 580, replace=False)] = rng.standard_normal(580)          # two segments
    A = HostCsr(emu, a.tocsr())
    assert len(A.long_rows) == 2 and A.n_seg == 3
    X = rng.standard_normal((m, d)).astype(np.float32)
    want = A.m @ X
    np.testing.assert_allclose(_spmm(emu, A, X), want, rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(_spmm(emu, A, X, relu=1), np.maximum(want, 0), rtol=1e-4, atol=1e-4)
    mask = rng.standard_normal((n, d)).astype(np.float32)
    np.testing.assert_allclose(_spmm(emu, A, X, mask=mask), want * (mask > 0), rtol=1e-4, atol=1e-4)
    y0 = rng.standard_normal((n, d)).astype(np.float32)
    np.testing.assert_allclose(_spmm(emu, A, X, beta=0.5, Y=y0.copy()), want + 0.5 * y0, rtol=1e-4, atol=1e-4)
    assert not _spmm(emu, A, X)[3].any()                                         # an empty row gives zeros


@pytest.mark.parametrize("edge_mode", [False, True])
def test_emulated_edge_softmax_sddmm_forward_and_backward(emu, edge_mode):
    rng = np.random.default_rng(3)
    n_r, n_c, d, slope = 37, 45, 8, 0.2                                          # rectangular: a row block of a sharded graph
    a = sp.random(n_r, n_c, density=0.15, random_state=2, format="csr", dtype=np.float32)
    a.data[:] = rng.random(a.nnz).astype(np.float32) + 0.5
    A = HostCsr(emu, a)
    row = torch.as_tensor(np.repeat(np.arange(n_r), np.diff(A.rowptr)), dtype=torch.long)
    col = torch.as_tensor(A.col, dtype=torch.long)
    s1 = torch.tensor(rng.standard_normal(n_r), dtype=torch.float32, requires_grad=True)
    s2 = torch.tensor(rng.standard_normal(n_c), dtype=torch.float32, requires_grad=True)
    ev = torch.tensor(rng.standard_normal(a.nnz), dtype=torch.float32, requires_grad=True)    # per-edge logits
    M = torch.tensor(rng.standard_normal((n_c, d)), dtype=torch.float32, requires_grad=True)
    pre = ev if edge_mode else torch.as_tensor(A.val) * (s1[row] + s2[col])
    logit = torch.nn.functional.leaky_relu(pre, slope)
    mx = torch.full((n_r,), -1e30).scatter_reduce(0, row, logit, "amax")
    ex = torch.exp(logit - mx[row])
    alpha_t = ex / torch.zeros(n_r).index_add(0, row, ex)[row]
    out_t = torch.zeros(n_r, d).index_add(0, row, alpha_t[:, None] * M[col])
    G = torch.tensor(rng.standard_normal((n_r, d)), dtype=torch.float32)
    (out_t * G).sum().backward()

    vals = ev.detach().numpy().copy() if edge_mode else None
    cs = A.csr(vals)
    alpha = np.zeros(a.nnz, dtype=np.float32)
    p = lambda t: None if t is None else t.ctypes.data
    s1n, s2n = (None, None) if edge_mode else (s1.detach().numpy().copy(), s2.detach().numpy().copy())
    assert emu.oea_edge_softmax_fwd(C.byref(cs), p(s1n), p(s2n), slope, alpha.ctypes.data, None) == 0
    np.testing.assert_allclose(alpha, alpha_t.detach().numpy(), rtol=1e-5, atol=1e-7)
    Mn, Gn = M.detach().numpy().copy(), G.numpy().copy()
    np.testing.assert_allclose(_spmm(emu, A, Mn, vals=alpha), out_t.detach().numpy(), rtol=1e-4, atol=1e-5)
    dalpha = np.zeros(a.nnz, dtype=np.float32)
    assert emu.oea_sddmm(C.byref(cs), Gn.ctypes.data, d, Mn.ctypes.data, d, d, dalpha.ctypes.data, None) == 0
    np.testing.assert_allclose(dalpha, (G[row] * M.detach()[col]).sum(1).numpy(), rtol=1e-5, atol=1e-6)
    ds1 = np.zeros(a.nnz if edge_mode else n_r, dtype=np.float32)
    ds2 = np.zeros(n_c, dtype=np.float32)
    assert emu.oea_edge_softmax_bwd(C.byref(cs), p(s1n), p(s2n), slope, alpha.ctypes.data, dalpha.ctypes.data,
                                    ds1.ctypes.data, None if edge_mode else ds2.ctypes.data, None) == 0
    if edge_mode:
        np.testing.assert_allclose(ds1, ev.grad.numpy(), rtol=1e-4, atol=1e-6)
    else:
        np.testing.assert_allclose(ds1, s1.grad.numpy(), rtol=1e-4, atol=1e-6)
        np.testing.assert_allclose(ds2, s2.grad.numpy(), rtol=1e-4, atol=1e-6)


def test_emulated_align_loss_l1_forward_and_backward(emu):
    from oracle.gnn import align_loss
    rng = np.random.default_rng(6)
    n, d, t, k = 60, 12, 19, 3
    x = torch.tensor(rng.standard_normal((n, d)), dtype=torch.float32, requires_grad=True)
    ill = np.stack([rng.permutation(n)[:t], rng.permutation(n)[:t]], 1)
    negs = [np.repeat(ill[:, 0], k), rng.integers(0, n, t * k), rng.integers(0, n, t * k), np.repeat(ill[:, 1], k)]
    want = align_loss(x, ill, 1.5, k, *negs)
    want.backward()
    xn = x.detach().numpy().copy()
    grad = np.zeros_like(xn)
    loss = np.zeros(1, dtype=np.float64)
    i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)
    arrs = [i32(ill[:, 0]), i32(ill[:, 1])] + [i32(a) for a in negs]
    rc = emu.oea_align_loss_l1(xn.ctypes.data, d, d, arrs[0].ctypes.data, arrs[1].ctypes.data, t, k, arrs[2].ctypes.data,
                               arrs[3].ctypes.data, arrs[4].ctypes.data, arrs[5].ctypes.data, 1.5, loss.ctypes.data,
                               grad.ctypes.data, None)
    assert rc == 0
    assert float(loss[0]) == pytest.approx(float(want.detach()), rel=1e-5)
    bad = np.abs(grad - x.grad.numpy()) > 1e-5                     # sign(0) cases of the L1 distance: none expected
    assert bad.mean() < 1e-3
