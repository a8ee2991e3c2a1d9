"""Host side of path (ii): device CSR matrices, the SpMM wrapper, adjacency builders of GCN-Align.

Adjacency construction is host-side SciPy (one-off, like the reference); the per-epoch work (A·X forward,
Aᵀ·dY backward, L1 alignment loss) runs in liboea.so kernels.
"""
import ctypes as C

import numpy as np
import scipy.sparse as sp
import torch

from . import lib as L
from .engine import _ptr, _stream_ptr


class DeviceCsr:
    """A sparse matrix on the device in CSR (int32 / fp32) plus, lazily, its transpose (for the backward)."""

    def __init__(self, mat, device="cuda", keep_duplicates=False):
        m = sp.csr_matrix(mat, dtype=np.float32)
        if not keep_duplicates:          # RDGCN's r_mat keeps one entry per triple, duplicates of (h, t) included
            m.sum_duplicates()
        m.sort_indices()
        self._keep_dup = keep_duplicates
        self.shape = m.shape
        self.nnz = int(m.nnz)
        self.device = torch.device(device)
        self._host = m
        self.rowptr = torch.from_numpy(m.indptr.astype(np.int32)).to(self.device)
        self.col = torch.from_numpy(m.indices.astype(np.int32)).to(self.device)
        self.val = torch.from_numpy(m.data.astype(np.float32)).to(self.device)
        lib = L.load()
        thr, seg = lib.oea_spmm_long_row_threshold(), lib.oea_spmm_segment_nnz()
        nnz_row = np.diff(m.indptr)
        long_rows = np.flatnonzero(nnz_row > thr).astype(np.int32)
        n_seg_row = -(-nnz_row[long_rows] // seg)
        seg_ptr = np.concatenate([[0], np.cumsum(n_seg_row)]).astype(np.int32)
        seg_row = np.repeat(np.arange(len(long_rows)), n_seg_row).astype(np.int32)
        within = np.arange(int(seg_ptr[-1])) - seg_ptr[seg_row] if len(long_rows) else np.zeros(0, dtype=np.int64)
        seg_start = (m.indptr[long_rows][seg_row] + within * seg).astype(np.int32) if len(long_rows) else np.zeros(0, np.int32)
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.device)
        self.long_rows, self.seg_ptr, self.seg_row, self.seg_start = up(long_rows), up(seg_ptr), up(seg_row), up(seg_start)
        self.n_seg = int(seg_ptr[-1])
        self._ws = None
        self._t = None

    def transpose(self):
        if self._t is None:
            self._t = DeviceCsr(self._host.T.tocsr(), self.device, keep_duplicates=self._keep_dup)
            self._t._t = self
        return self._t

    def transpose_perm(self):
        """perm [nnz] (int64 CUDA tensor): position e of the TRANSPOSE's CSR order holds edge perm[e] of this matrix,
        so `vals[perm]` are per-edge values re-ordered for the transposed pattern (backward of a weighted SpMM)."""
        if getattr(self, "_perm", None) is None:
            m = self._host
            ids = sp.csr_matrix((np.arange(1, m.nnz + 1, dtype=np.float64), m.indices, m.indptr), shape=m.shape)
            t = ids.T.tocsr()
            t.sort_indices()
            self._perm = torch.from_numpy((t.data - 1).astype(np.int64)).to(self.device)
        return self._perm

    def hubs_struct(self):
        return L.SpmmHubs(self.long_rows.data_ptr(), self.seg_ptr.data_ptr(), self.seg_row.data_ptr(),
                          self.seg_start.data_ptr(), self.long_rows.numel(), self.n_seg)

    def workspace(self, d):
        need = L.load().oea_spmm_workspace_bytes(self.n_seg, d)
        if self._ws is None or self._ws.numel() * 4 < need:
            self._ws = torch.empty(max(1, need // 4), dtype=torch.float32, device=self.device)
        return self._ws, need

    def c_struct(self, vals=None):
        v = self.val if vals is None else vals
        return L.Csr(self.rowptr.data_ptr(), self.col.data_ptr(), v.data_ptr(), self.shape[0], self.shape[1], self.nnz)


def spmm(A, X, out=None, relu=False, mask_src=None, beta=0.0, vals=None):
    """Y = A·X (fp32, X row-major with X.shape[1] % 4 == 0), optional fused relu / relu-backward mask.
    `vals` [nnz] replaces A's values (same pattern), e.g. attention coefficients."""
    lib = L.load()
    assert X.device == A.rowptr.device and X.dtype == torch.float32 and X.stride(1) == 1
    d = X.shape[1]
    if out is None:
        out = torch.empty(A.shape[0], d, dtype=torch.float32, device=X.device)
    cs, hubs = A.c_struct(vals), A.hubs_struct()
    ws, ws_bytes = A.workspace(d)
    L.check(lib.oea_spmm_csr(C.byref(cs), C.byref(hubs), _ptr(X), X.stride(0), _ptr(out), out.stride(0), d, int(relu),
                             _ptr(mask_src), float(beta), _ptr(ws), ws_bytes, _stream_ptr()), "oea_spmm_csr")
    return out


class SpmmFn(torch.autograd.Function):
    """Y = A·X for autograd graphs (A constant): backward is the same kernel on Aᵀ."""

    @staticmethod
    def forward(ctx, X, A):
        ctx.A = A
        return spmm(A, X.contiguous())

    @staticmethod
    def backward(ctx, gY):
        return spmm(ctx.A.transpose(), gY.contiguous()), None


def tc_gemm_nt(A, B):
    """C = A·Bᵀ for row-major fp32 A [m, k], B [n, k] (k % 4 == 0) on the tensor cores: the 3xTF32 wgmma kernel of path
    (iii) (oea_sim_matrix_tc) used as a GEMM-NT; values agree with an FP32 GEMM to fp32 round-off.  Returns [m, n]."""
    lib = L.load()
    m, k = A.shape
    n = B.shape[0]
    assert B.shape[1] == k and k % 4 == 0 and A.is_contiguous() and B.is_contiguous()
    ld = (n + 3) // 4 * 4
    out = torch.empty(m, ld, dtype=torch.float32, device=A.device)
    cfg = L.SimCfg(L.METRIC_INNER, m, n, k, k, k, 0, 0, 0, 0)
    L.check(lib.oea_sim_matrix_tc(C.byref(cfg), _ptr(A), _ptr(B), None, None, _ptr(out), ld, _stream_ptr()), "oea_sim_matrix_tc")
    return out if ld == n else out[:, :n]


class TcMatmulFn(torch.autograd.Function):
    """Y = X·W for the dense products of AliNet / RDGCN (alinet.py:574-590 `tf.matmul(inputs, kernel)`) on our tensor-core
    kernel: forward and dX are GEMM-NTs of the 3xTF32 kernel; dW = Xᵀ·dY has a contraction length of N entities and a tiny
    output (it would need split-K on that kernel) and stays a library GEMM."""

    @staticmethod
    def forward(ctx, X, W):
        ctx.save_for_backward(X, W)
        return tc_gemm_nt(X.contiguous(), W.t().contiguous())

    @staticmethod
    def backward(ctx, gY):
        X, W = ctx.saved_tensors
        gX = tc_gemm_nt(gY.contiguous(), W.contiguous()) if ctx.needs_input_grad[0] else None
        gW = X.t() @ gY if ctx.needs_input_grad[1] else None
        return gX, gW


def dense_matmul(X, W):
    """X·W: the tensor-core kernel for CUDA fp32 operands whose inner and output widths are multiples of 4 (every layer of
    the shipped configs), a library GEMM otherwise.  OEA_GNN_TC=0 keeps the library GEMM everywhere (A/B, parity checks)."""
    import os
    if (X.is_cuda and X.dtype == torch.float32 and W.dtype == torch.float32 and X.dim() == 2 and W.dim() == 2
            and X.shape[1] % 4 == 0 and W.shape[1] % 4 == 0 and X.shape[0] >= 128 and os.environ.get("OEA_GNN_TC", "1") != "0"):
        return TcMatmulFn.apply(X, W)
    return X @ W


class GatAggregateFn(torch.autograd.Function):
    """out_i = Σ_j softmax_j(leaky_relu(a_ij·(s1_i + s2_j)))·M_j over the non-zeros of A (alinet.py:656-677)."""

    @staticmethod
    def forward(ctx, s1, s2, M, A, slope):
        lib = L.load()
        s1, s2, M = s1.contiguous(), s2.contiguous(), M.contiguous()
        alpha = torch.empty(A.nnz, dtype=torch.float32, device=M.device)
        cs = A.c_struct()
        L.check(lib.oea_edge_softmax_fwd(C.byref(cs), _ptr(s1), _ptr(s2), float(slope), _ptr(alpha), _stream_ptr()),
                "oea_edge_softmax_fwd")
        ctx.A, ctx.slope = A, float(slope)
        ctx.save_for_backward(s1, s2, M, alpha)
        return spmm(A, M, vals=alpha)

    @staticmethod
    def backward(ctx, gOut):
        lib = L.load()
        s1, s2, M, alpha = ctx.saved_tensors
        A = ctx.A
        gOut = gOut.contiguous()
        cs = A.c_struct()
        dalpha = torch.empty_like(alpha)
        L.check(lib.oea_sddmm(C.byref(cs), _ptr(gOut), gOut.stride(0), _ptr(M), M.stride(0), M.shape[1], _ptr(dalpha),
                              _stream_ptr()), "oea_sddmm")
        ds1 = torch.empty_like(s1)
        ds2 = torch.zeros_like(s2)
        L.check(lib.oea_edge_softmax_bwd(C.byref(cs), _ptr(s1), _ptr(s2), ctx.slope, _ptr(alpha), _ptr(dalpha), _ptr(ds1),
                                         _ptr(ds2), _stream_ptr()), "oea_edge_softmax_bwd")
        dM = spmm(A.transpose(), gOut, vals=alpha.index_select(0, A.transpose_perm()))
        return ds1, ds2, dM, None, None


class EdgeLogitAggregateFn(torch.autograd.Function):
    """out_i = Σ_e softmax over row i of leaky_relu(logit_e) · X[col e] with per-EDGE logits (rdgcn.py:202-215)."""

    @staticmethod
    def forward(ctx, edge_logits, X, A, slope):
        lib = L.load()
        edge_logits, X = edge_logits.contiguous(), X.contiguous()
        alpha = torch.empty(A.nnz, dtype=torch.float32, device=X.device)
        cs = A.c_struct(edge_logits)
        L.check(lib.oea_edge_softmax_fwd(C.byref(cs), None, None, float(slope), _ptr(alpha), _stream_ptr()),
                "oea_edge_softmax_fwd")
        ctx.A, ctx.slope = A, float(slope)
        ctx.save_for_backward(edge_logits, X, alpha)
        return spmm(A, X, vals=alpha)

    @staticmethod
    def backward(ctx, gOut):
        lib = L.load()
        edge_logits, X, alpha = ctx.saved_tensors
        A = ctx.A
        gOut = gOut.contiguous()
        cs = A.c_struct(edge_logits)
        dalpha = torch.empty_like(alpha)
        L.check(lib.oea_sddmm(C.byref(cs), _ptr(gOut), gOut.stride(0), _ptr(X), X.stride(0), X.shape[1], _ptr(dalpha),
                              _stream_ptr()), "oea_sddmm")
        dlogit = torch.empty_like(alpha)
        L.check(lib.oea_edge_softmax_bwd(C.byref(cs), None, None, ctx.slope, _ptr(alpha), _ptr(dalpha), _ptr(dlogit),
                                         None, _stream_ptr()), "oea_edge_softmax_bwd")
        dX = spmm(A.transpose(), gOut, vals=alpha.index_select(0, A.transpose_perm()))
        return dlogit, dX, None, None


class AlignLossL1Fn(torch.autograd.Function):
    """align_loss / get_loss (gcn_align.py:298-320, rdgcn.py:293-315) for autograd graphs: forward+backward in one
    kernel launch; the gradient is kept for backward()."""

    @staticmethod
    def forward(ctx, x, left, right, k, negs, gamma):
        x = x.contiguous()
        grad = torch.zeros_like(x)
        loss = torch.zeros(1, dtype=torch.float64, device=x.device)
        align_loss_l1(x, x.shape[1], left, right, k, negs[0], negs[1], negs[2], negs[3], gamma, grad, loss)
        ctx.save_for_backward(grad)
        return loss.to(torch.float32).reshape(())

    @staticmethod
    def backward(ctx, gout):
        (grad,) = ctx.saved_tensors
        return grad * gout, None, None, None, None, None


def align_loss_l1(x, dim, left, right, k, neg_left, neg_right, neg2_left, neg2_right, gamma, grad, loss_out):
    lib = L.load()
    L.check(lib.oea_align_loss_l1(_ptr(x), x.stride(0), dim, _ptr(left), _ptr(right), left.numel(), k,
                                  _ptr(neg_left), _ptr(neg_right), _ptr(neg2_left), _ptr(neg2_right), float(gamma),
                                  _ptr(loss_out), _ptr(grad), _stream_ptr()), "oea_align_loss_l1")


# ---- adjacency builders of GCN-Align (approaches/gcn_align.py:566-578,610-664) ---------------------------
def relation_functionality(triples):
    """r2f[r] = #distinct heads / #triples of r ; r2if[r] = #distinct tails / #triples of r (gcn_align.py:610-640)."""
    tri = np.asarray(triples, dtype=np.int64).reshape(-1, 3)
    rels, inv, cnt = np.unique(tri[:, 1], return_inverse=True, return_counts=True)
    n_heads = np.bincount(np.unique(np.stack([inv, tri[:, 0]], 1), axis=0)[:, 0], minlength=len(rels))
    n_tails = np.bincount(np.unique(np.stack([inv, tri[:, 2]], 1), axis=0)[:, 0], minlength=len(rels))
    r2f = dict(zip(rels.tolist(), (n_heads / cnt).tolist()))
    r2if = dict(zip(rels.tolist(), (n_tails / cnt).tolist()))
    return r2f, r2if


def weighted_adjacency(n_ent, triples):
    """get_weighted_adj (gcn_align.py:642-664): for every triple with h ≠ t,
    M[(h,t)] += max(r2if[r], .3) and M[(t,h)] += max(r2f[r], .3); the COO entry of key (a, b) sits at
    (row = b, col = a)."""
    tri = np.asarray(triples, dtype=np.int64).reshape(-1, 3)
    r2f, r2if = relation_functionality(tri)
    keep = tri[:, 0] != tri[:, 2]
    h, r, t = tri[keep, 0], tri[keep, 1], tri[keep, 2]
    w_if = np.maximum(np.array([r2if[x] for x in r.tolist()]), 0.3)
    w_f = np.maximum(np.array([r2f[x] for x in r.tolist()]), 0.3)
    rows = np.concatenate([t, h])     # key (h,t) → row t, col h ; key (t,h) → row h, col t
    cols = np.concatenate([h, t])
    data = np.concatenate([w_if, w_f])
    return sp.coo_matrix((data, (rows, cols)), shape=(n_ent, n_ent)).tocsr()   # duplicates sum, as M[...] += does


def normalize_adj(adj):
    """D^-½ · adjᵀ · D^-½ with D = diag(row sums of adj) (gcn_align.py:566-573; the transpose is real for the
    asymmetric weighted adjacency)."""
    adj = sp.coo_matrix(adj)
    rowsum = np.asarray(adj.sum(1)).flatten()
    with np.errstate(divide="ignore"):
        d_inv_sqrt = np.power(rowsum, -0.5)
    d_inv_sqrt[np.isinf(d_inv_sqrt)] = 0.0
    dm = sp.diags(d_inv_sqrt)
    return adj.dot(dm).transpose().dot(dm).tocoo()


def preprocess_adj(adj):
    return normalize_adj(adj + sp.eye(adj.shape[0]))


def attribute_features(n_ent, entity_attributes_dict):
    """load_attr (gcn_align.py:89-111): 0/1 entity × attribute matrix over the 70 % most frequent attributes
    (ties in frequency keep first-seen order, as sorted(cnt, key=cnt.get, reverse=True) does)."""
    cnt = {}
    for _, attrs in entity_attributes_dict.items():
        for a in attrs:
            cnt[a] = cnt.get(a, 0) + 1
    ranked = sorted(cnt, key=cnt.get, reverse=True)
    num = int(0.7 * len(cnt))
    attr2id = {a: i for i, a in enumerate(ranked[:num])}
    rows, cols = [], []
    for ent, attrs in entity_attributes_dict.items():
        for a in attrs:
            if a in attr2id:
                rows.append(ent)
                cols.append(attr2id[a])
    data = np.ones(len(rows), dtype=np.float32)
    m = sp.coo_matrix((data, (rows, cols)), shape=(n_ent, max(num, 1))).tocsr()
    m.data[:] = 1.0   # attr[ent][id] = 1.0 is an assignment, not an accumulation
    return m
