"""Path (ii) at its edges: the warp-per-row SpMM with its hub segments and fused epilogues, the edge softmax forward and
backward, SDDMM and the L1 alignment loss (openea_b200/csrc/oea_spmm.cu), driven through the product's host layer
(openea_b200.gnn) wherever one exists, against float64 references.  tests/test_emu_gnn_edges.py runs these cases on the
warp emulator, tests/test_zz_gnn_edges_gpu.py on the GPU.

Two reference modes:

* Exact mode.  Inputs are small integers or dyadic values (quarters, eighths), chosen so that every sum the kernel forms
  is an exact fp32 dyadic below 2^24 whatever the summation order: values and X of SpMM and SDDMM in [-3, 3], integer
  embeddings and margins of the alignment loss with t·k a power of two (1/(2kt) exact), dyadic alpha / dalpha / slope
  in the softmax backward.  The edge-softmax forward is exact on rows of equal logits: every exponent is exp(0) = 1 and
  alpha must be fl(1/n).  Outputs must be bit-identical to float64 rounded to fp32.
* Bound mode.  Real-valued inputs.  Every output entry is compared with float64 within a first-order fp32 error bound,
  derived next to the function that computes it.  Backward kernels are checked as functions of their own fp32 inputs
  (the kernel's alpha and dalpha are fed to the float64 formula), so the reference does not inherit forward error.

Every output buffer a kernel should overwrite is pre-filled with NaN, and padding columns of strided inputs hold NaN,
so a skipped row or an over-read column cannot pass by accident.
"""
import ctypes as C

import numpy as np
import scipy.sparse as sp
import torch

from openea_b200 import gnn
from openea_b200 import lib as L
from openea_b200.engine import _ptr
from oracle import gnn as org

F32 = np.float32
U = float(np.finfo(np.float32).eps) / 2          # unit round-off of fp32
FLT_MIN = float(np.finfo(np.float32).tiny)       # smallest normal fp32: what a flushed exponential can lose
OK, ERR_NULL, ERR_DIM, ERR_ALIGN, ERR_SHAPE = 0, 1, 2, 3, 5
SENTINEL = 7.25                                  # columns >= d of a strided output: must stay untouched

# SpMM row lengths: empty, the gather tails of U = 8 / 4 / 2 (1…9), one chunk of 32 ± 1, the hub threshold (256 runs
# warp-per-row, 257 is a hub), the 512-non-zero segment edges, the 64-non-zero per-warp shares of a last segment
# (575 / 576 / 577 leave 63 / 64 / 65 non-zeros), two-segment edges and a row of nine segments
ROW_LENGTHS = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 31, 32, 33, 255, 256, 257, 511, 512, 513, 575, 576, 577, 1024, 1025, 4100]
# the VEC = 1 / 2 / 3 / 4 buckets of the SpMM at and around each edge
SPMM_DIMS = [4, 124, 128, 132, 252, 256, 260, 380, 384, 388, 508, 512]
# edge softmax: one lane pass ± 1, two lane passes ± 1, and a hub row
SOFTMAX_LENGTHS = [0, 1, 31, 32, 33, 64, 65, 650]
SDDMM_DIMS = [4, 128, 132, 512, 600]
LOSS_DIMS = [1, 31, 32, 33, 300, 600]
SLOPE = float(F32(0.2))                          # the fp32 value the kernels receive


def gamma(n):
    return n * U / (1 - n * U)


def host(t):
    return t.detach().cpu().numpy()


def dev_t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def ints(rng, shape, lo=-3, hi=3):
    return rng.integers(lo, hi + 1, shape).astype(F32)


def nonzero_ints(rng, n):
    return (rng.integers(1, 4, n) * rng.choice([-1, 1], n)).astype(F32)


def csr_rows(rng, lengths, n_cols, values):
    """CSR matrix whose rows have exactly `lengths` non-zeros (distinct, sorted columns); values 'int' (non-zero
    integers in [-3, 3]) or 'real' (standard normal)."""
    lengths = np.asarray(lengths, dtype=np.int64)
    indptr = np.concatenate([[0], np.cumsum(lengths)])
    cols = [np.sort(rng.choice(n_cols, n, replace=False)) for n in lengths]
    idx = np.concatenate(cols) if len(cols) else np.zeros(0, np.int64)
    nnz = int(indptr[-1])
    val = nonzero_ints(rng, nnz) if values == "int" else rng.standard_normal(nnz).astype(F32)
    return sp.csr_matrix((val, idx, indptr), shape=(len(lengths), n_cols))


def padded(x, ld, dev, fill=np.nan):
    """A [rows, ld] device buffer holding x in its first columns and `fill` in the rest; returns (buffer, view)."""
    buf = torch.full((x.shape[0], ld), fill, dtype=torch.float32, device=dev)
    buf[:, :x.shape[1]] = torch.from_numpy(np.ascontiguousarray(x, dtype=F32)).to(dev)
    return buf, buf[:, :x.shape[1]]


# ---- SpMM ---------------------------------------------------------------------------------------------------------
def spmm_epilogue(want, beta=0.0, y_old=None, relu=False, mask=None):
    """The documented epilogue order of oea_spmm_csr: beta·Y_old is added first, then relu, then the mask."""
    v = want + (beta * y_old.astype(np.float64) if beta else 0.0)
    if relu:
        v = np.maximum(v, 0.0)
    if mask is not None:
        v = np.where(mask > 0, v, 0.0)
    return v


def run_spmm(dev, DA, X, *, ldx=None, ldy=None, relu=False, mask=None, beta=0.0, y_old=None, vals=None):
    """gnn.spmm on strided views: X in a [n_cols, ldx] buffer whose padding is NaN, Y a view of an [n_rows, ldy] buffer
    (NaN in columns < d unless beta needs Y_old, SENTINEL beyond), mask_src an [n_rows, ldy] buffer as the kernel reads
    it at Y's stride.  Returns Y [n_rows, d] as NumPy after checking that the padding of Y was not written."""
    d = X.shape[1]
    ldx, ldy = ldx or d, ldy or d
    _, Xv = padded(X, ldx, dev)
    ybuf = torch.full((DA.shape[0], ldy), SENTINEL, dtype=torch.float32, device=dev)
    ybuf[:, :d] = float("nan") if y_old is None else torch.from_numpy(np.ascontiguousarray(y_old, dtype=F32)).to(dev)
    mbuf = None
    if mask is not None:
        mbuf = torch.full((DA.shape[0], ldy), -1.0, dtype=torch.float32, device=dev)
        mbuf[:, d:] = 1.0                      # read at stride d, row r > 0 would pick these up
        mbuf[:, :d] = torch.from_numpy(np.ascontiguousarray(mask, dtype=F32)).to(dev)
    v = None if vals is None else dev_t(np.asarray(vals, dtype=F32), dev)
    out = gnn.spmm(DA, Xv, out=ybuf[:, :d], relu=relu, mask_src=mbuf, beta=beta, vals=v)
    assert out.data_ptr() == ybuf.data_ptr()
    yb = host(ybuf)
    assert np.all(yb[:, d:] == F32(SENTINEL)), "columns >= d of Y were written"
    return yb[:, :d]


def check_spmm_exact(dev, DA, a, X, **kw):
    """Bit-identical to float64: `a` the scipy matrix (its values, or kw['vals']), X integer-valued."""
    vals = kw.get("vals")
    m = sp.csr_matrix((np.asarray(vals, np.float64), a.indices, a.indptr), shape=a.shape) if vals is not None else a
    want = m.astype(np.float64) @ X.astype(np.float64)
    ref = spmm_epilogue(want, kw.get("beta", 0.0), kw.get("y_old"), kw.get("relu", False), kw.get("mask")).astype(F32)
    got = run_spmm(dev, DA, X, **kw)
    bad = ~(got == ref)
    assert not bad.any(), "rows %s differ (first: got %r, want %r)" % (
        np.unique(np.nonzero(bad)[0])[:10], got[bad][:3], ref[bad][:3])
    return want


def check_spmm_bound(dev, DA, a, X, **kw):
    """Real-valued SpMM.  Row i sums nnz_i products with fmaf, split over lanes, warps and 512-non-zero segments and
    added in any tree: |fl(Σ) − Σ| ≤ γ_{nnz_i}·Σ_j |a_ij·x_jc| (Higham, Thm 3.5, for any summation order).  The beta
    epilogue is one more fma: + u·|v| with |v| ≤ Σ|a x| + |β y_old|.  Relu and the mask are 1-Lipschitz / selections
    and add nothing.  Bound: γ_{nnz_i + 2}·(Σ_j |a_ij x_jc| + |β·y_old|)."""
    a64 = a.astype(np.float64)
    X64 = X.astype(np.float64)
    beta, y_old = kw.get("beta", 0.0), kw.get("y_old")
    want = a64 @ X64
    absw = abs(a64) @ np.abs(X64) + (abs(beta) * np.abs(y_old.astype(np.float64)) if beta else 0.0)
    nnz = np.diff(a.indptr)[:, None]
    bound = gamma(nnz + 2) * absw
    ref = spmm_epilogue(want, beta, y_old, kw.get("relu", False), kw.get("mask"))
    got = run_spmm(dev, DA, X, **kw)
    err = np.abs(got - ref)
    assert np.all(err <= bound), "max err/bound %.3g at %s" % (np.max(err / np.maximum(bound, 1e-300)),
                                                               np.unravel_index(np.argmax(err - bound), err.shape))
    return float(np.max(err / np.maximum(bound, 1e-300)))


def raw_spmm(DA, X, d=None, hubs="plan", x_offset=0):
    """oea_spmm_csr through the C-ABI, for what gnn.spmm cannot express: no hub plan and bad arguments.  X is a
    contiguous [n_cols, ld] device tensor, ldx = ldy = ld; hubs is 'plan' (DeviceCsr's), None (a NULL pointer) or
    'empty' (n_long = 0); x_offset shifts the X pointer by that many bytes.  Returns (rc, Y) with Y pre-filled with NaN."""
    lib = L.load()
    ld = X.shape[1]
    d = ld if d is None else d
    Y = torch.full((DA.shape[0], ld), float("nan"), dtype=torch.float32, device=X.device)
    cs = DA.c_struct()
    hb = DA.hubs_struct() if hubs == "plan" else L.SpmmHubs(0, 0, 0, 0, 0, 0)
    ws, nbytes = DA.workspace(ld) if hubs == "plan" else (None, 0)
    rc = lib.oea_spmm_csr(C.byref(cs), None if hubs is None else C.byref(hb), C.c_void_p(X.data_ptr() + x_offset), ld,
                          _ptr(Y), ld, d, 0, None, 0.0, _ptr(ws), nbytes, gnn._stream_ptr())
    return rc, Y


# ---- edge softmax ----------------------------------------------------------------------------------------------------
def softmax_fwd(dev, DA, s1=None, s2=None, edge_logits=None, slope=SLOPE):
    """oea_edge_softmax_fwd as GatAggregateFn / EdgeLogitAggregateFn call it: node mode (s1, s2) or edge-logit mode
    (the logits replace A's values).  alpha is pre-filled with NaN."""
    lib = L.load()
    alpha = torch.full((DA.nnz,), float("nan"), dtype=torch.float32, device=dev)
    if edge_logits is None:
        s1t, s2t = dev_t(s1.astype(F32), dev), dev_t(s2.astype(F32), dev)
        cs = DA.c_struct()
        L.check(lib.oea_edge_softmax_fwd(C.byref(cs), _ptr(s1t), _ptr(s2t), slope, _ptr(alpha), gnn._stream_ptr()))
    else:
        lt = dev_t(edge_logits.astype(F32), dev)
        cs = DA.c_struct(lt)
        L.check(lib.oea_edge_softmax_fwd(C.byref(cs), None, None, slope, _ptr(alpha), gnn._stream_ptr()))
    return host(alpha)


def pre_activation(a, s1=None, s2=None, edge_logits=None):
    """float64 pre-activation logits of every edge in CSR order (from the fp32 inputs)."""
    if edge_logits is not None:
        return edge_logits.astype(np.float64)
    row = np.repeat(np.arange(a.shape[0]), np.diff(a.indptr))
    return a.data.astype(np.float64) * (s1.astype(np.float64)[row] + s2.astype(np.float64)[a.indices])


def softmax_ref(a, s1=None, s2=None, edge_logits=None, slope=SLOPE):
    """float64 alpha of oracle/gnn.py's edge_softmax, in CSR order."""
    t = lambda x: None if x is None else torch.as_tensor(x.astype(np.float64))
    return org.edge_softmax(a, t(s1), t(s2), slope, t(edge_logits), torch.float64).numpy()


def softmax_bound(a, alpha64, pre, slope, node_mode, exp_ulps):
    """Bound on |alpha_fp32 − alpha64| per edge.

    Logit l = leaky(pre): node mode rounds s1 + s2 and a·(…) (γ_2), the slope product one more: |Δl| ≤ γ_3·|l|.
    Exponent argument x = fl(l − mx), mx the row's largest fp32 logit: |Δx| ≤ |Δl| + |Δmx| + u·|l − mx|
    ≤ γ_4·(|l| + |mx|).  The exponential adds its own error, exp_ulps(x) ulp (≤ 2u relative each), plus at most
    FLT_MIN absolute where the result underflows (flushed on the GPU).  So e = E·(1 + η) with
    |η| ≤ expm1(|Δx|) + 2u·ulps(x)·(1 + expm1(|Δx|)).  The row sum of the positive e's is within η_max + γ_n of Σ E
    (relative), the reciprocal and the product round once each:
        |Δalpha| ≤ alpha·((1 + η_e)(1 + u)² / ((1 − η_max)(1 − γ_n)) − 1) + (n + 1)·FLT_MIN."""
    l = np.where(pre > 0, pre, slope * pre)
    row = np.repeat(np.arange(a.shape[0]), np.diff(a.indptr))
    n_row = np.diff(a.indptr)
    mx = np.full(a.shape[0], -np.inf)
    np.maximum.at(mx, row, l)
    dx = gamma(4 if node_mode else 3) * (np.abs(l) + np.abs(mx[row]))
    x = l - mx[row]
    ulps = exp_ulps(np.abs(x) + dx)
    eta = np.expm1(dx) + 2 * U * ulps * (1 + np.expm1(dx))
    eta_max = np.zeros(a.shape[0])
    np.maximum.at(eta_max, row, eta)
    n = n_row[row]
    rel = (1 + eta) * (1 + U) ** 2 / ((1 - eta_max[row]) * (1 - gamma(n))) - 1
    return alpha64 * rel + (n + 1) * FLT_MIN


def expf_ulps_host(x):
    """The emulator's expf (glibc): below 1 ulp."""
    return np.ones_like(x)


def expf_ulps_device(x):
    """CUDA's __expf: at most 2 + floor(1.173·|x|) ulp (CUDA C Programming Guide, intrinsic functions)."""
    return 2 + np.floor(1.173 * np.abs(x))


def check_softmax_bound(dev, DA, a, exp_ulps, s1=None, s2=None, edge_logits=None, slope=SLOPE):
    pre = pre_activation(a, s1, s2, edge_logits)
    got = softmax_fwd(dev, DA, s1, s2, edge_logits, slope)
    want = softmax_ref(a, s1, s2, edge_logits, slope)
    bound = softmax_bound(a, want, pre, slope, edge_logits is None, exp_ulps)
    err = np.abs(got.astype(np.float64) - want)
    ratio = err / bound
    assert np.all(err <= bound), "alpha err/bound %.3g at edge %d (alpha %r, want %r)" % (
        ratio.max(), int(np.argmax(ratio)), got[np.argmax(ratio)], want[np.argmax(ratio)])
    return got, float(ratio.max()) if ratio.size else 0.0


def softmax_bwd(dev, DA, alpha, dalpha, s1=None, s2=None, edge_logits=None, slope=SLOPE, ds2_fill=None):
    """oea_edge_softmax_bwd: node mode returns (ds1 [n_rows], ds2 [n_cols]) with ds2 accumulated into ds2_fill;
    edge-logit mode returns (dlogit [nnz], None) with a NULL ds2.  ds1 / dlogit are pre-filled with NaN."""
    lib = L.load()
    at, dat = dev_t(alpha.astype(F32), dev), dev_t(dalpha.astype(F32), dev)
    if edge_logits is None:
        s1t, s2t = dev_t(s1.astype(F32), dev), dev_t(s2.astype(F32), dev)
        ds1 = torch.full((DA.shape[0],), float("nan"), dtype=torch.float32, device=dev)
        ds2 = dev_t(ds2_fill.astype(F32), dev)
        cs = DA.c_struct()
        L.check(lib.oea_edge_softmax_bwd(C.byref(cs), _ptr(s1t), _ptr(s2t), slope, _ptr(at), _ptr(dat), _ptr(ds1),
                                         _ptr(ds2), gnn._stream_ptr()))
        return host(ds1), host(ds2)
    lt = dev_t(edge_logits.astype(F32), dev)
    ds1 = torch.full((DA.nnz,), float("nan"), dtype=torch.float32, device=dev)
    cs = DA.c_struct(lt)
    L.check(lib.oea_edge_softmax_bwd(C.byref(cs), None, None, slope, _ptr(at), _ptr(dat), _ptr(ds1), None,
                                     gnn._stream_ptr()))
    return host(ds1), None


def softmax_bwd_ref(a, alpha, dalpha, pre, slope, node_mode, ds2_fill=None, dalpha_err=None):
    """float64 backward of the softmax and the leaky relu as a function of the kernel's alpha and dalpha:
        dl_e = alpha_e·(dalpha_e − Σ_row alpha·dalpha)·(pre_e > 0 ? 1 : slope)·(a_e in node mode)
    (torch's leaky_relu takes the slope branch at pre = 0 too); ds1_i = Σ_row dl, ds2_c = fill_c + Σ_col dl.

    Bound.  dotp = fl(Σ alpha·dalpha) over n terms: γ_n·S, S = Σ|alpha·dalpha|.  r = fl(dalpha − dotp) adds u·|r|.
    The products alpha·r, ·s', ·a round k = 2 (edge) or 3 (node) times:
        |Δdl_e| ≤ |alpha_e s'_e a_e|·(Δr + γ_k·(|r| + Δr)),  Δr = γ_n·S + u·(|r| + γ_n·S).
    ds1_i sums n of them in a warp tree, ds2_c takes m_c atomic adds onto its fill, in any order:
        |Δds1_i| ≤ Σ|Δdl| + γ_n·Σ(|dl| + |Δdl|),  |Δds2_c| ≤ Σ|Δdl| + γ_{m_c}·(|fill| + Σ(|dl| + |Δdl|)).
    When dalpha itself carries an error ≤ dalpha_err (the SDDMM's, in the autograd tests), dl_e moves by at most
    |alpha_e s'_e a_e|·(dalpha_err_e + Σ_row alpha·dalpha_err) more."""
    n_rows = a.shape[0]
    row = np.repeat(np.arange(n_rows), np.diff(a.indptr))
    al, da = alpha.astype(np.float64), dalpha.astype(np.float64)
    dotp = np.bincount(row, al * da, minlength=n_rows)
    S = np.bincount(row, np.abs(al * da), minlength=n_rows)
    n = np.diff(a.indptr)[row]
    r = da - dotp[row]
    w = al * np.where(pre > 0, 1.0, slope) * (a.data.astype(np.float64) if node_mode else 1.0)
    dl = w * r
    dr = gamma(n) * S[row] + U * (np.abs(r) + gamma(n) * S[row])
    if dalpha_err is not None:
        dr = dr + dalpha_err + np.bincount(row, al * dalpha_err, minlength=n_rows)[row]
    ddl = np.abs(w) * (dr + gamma(3 if node_mode else 2) * (np.abs(r) + dr))
    if not node_mode:
        return dl, ddl, None, None, None, None
    nr = np.diff(a.indptr)
    ds1 = np.bincount(row, dl, minlength=n_rows)
    b1 = np.bincount(row, ddl, minlength=n_rows) + gamma(nr) * np.bincount(row, np.abs(dl) + ddl, minlength=n_rows)
    n_cols = a.shape[1]
    fill = ds2_fill.astype(np.float64)
    ds2 = fill + np.bincount(a.indices, dl, minlength=n_cols)
    m = np.bincount(a.indices, minlength=n_cols)
    b2 = np.bincount(a.indices, ddl, minlength=n_cols) + gamma(m) * (np.abs(fill) + np.bincount(
        a.indices, np.abs(dl) + ddl, minlength=n_cols))
    return ds1, b1, ds2, b2, dl, ddl


def assert_within(got, want, bound, what):
    err = np.abs(got.astype(np.float64) - want)
    ok = err <= bound
    assert ok.all(), "%s: %d entries outside the bound, worst err/bound %.3g at %d (got %r, want %r)" % (
        what, int((~ok).sum()), np.max(err / np.maximum(bound, 1e-300)), int(np.argmax(err - bound)),
        got.reshape(-1)[np.argmax(err - bound)], want.reshape(-1)[np.argmax(err - bound)])


def assert_exact(got, want, what):
    w = np.asarray(want).astype(F32)
    bad = ~(got == w)
    assert not bad.any(), "%s: %d entries differ, first at %s (got %r, want %r)" % (
        what, int(bad.sum()), np.argwhere(bad)[0], got[bad][:3], w[bad][:3])


# ---- SDDMM -----------------------------------------------------------------------------------------------------------
def sddmm(dev, DA, G, M, ldg, ldm):
    """oea_sddmm through the C-ABI with G, M in [·, ldg] / [·, ldm] buffers whose padding is NaN (the host layer only
    passes contiguous operands).  out is pre-filled with NaN."""
    lib = L.load()
    gb, _ = padded(G, ldg, dev)
    mb, _ = padded(M, ldm, dev)
    out = torch.full((DA.nnz,), float("nan"), dtype=torch.float32, device=dev)
    cs = DA.c_struct()
    L.check(lib.oea_sddmm(C.byref(cs), _ptr(gb), ldg, _ptr(mb), ldm, G.shape[1], _ptr(out), gnn._stream_ptr()))
    return host(out)


def sddmm_ref(a, G, M):
    """float64 <G[row e], M[col e]> and its bound γ_d·Σ|g·m| (d products summed with fmaf in any order)."""
    row = np.repeat(np.arange(a.shape[0]), np.diff(a.indptr))
    g, m = G.astype(np.float64)[row], M.astype(np.float64)[a.indices]
    return (g * m).sum(1), gamma(G.shape[1]) * np.abs(g * m).sum(1)


# ---- L1 alignment loss -----------------------------------------------------------------------------------------------
def align_case(rng, n, t, k):
    """Seed pairs and the k negatives per side: (l, random) and (random, r), as gcn_align.py draws them."""
    left, right = rng.integers(0, n, t), rng.integers(0, n, t)
    negs = [np.repeat(left, k), rng.integers(0, n, t * k), rng.integers(0, n, t * k), np.repeat(right, k)]
    return left, right, [np.asarray(x) for x in negs]


def run_align(dev, x, ld, left, right, k, negs, gamma_, grad_fill, loss_fill):
    """gnn.align_loss_l1 on an [N, ld] embedding buffer (padding NaN) with grad an [N, ld] buffer: grad_fill in its first
    dim columns (accumulated into), SENTINEL beyond (must stay); loss accumulated into loss_fill."""
    dim = x.shape[1]
    _, xv = padded(x, ld, dev)
    grad = torch.full((x.shape[0], ld), SENTINEL, dtype=torch.float32, device=dev)
    grad[:, :dim] = torch.from_numpy(np.ascontiguousarray(grad_fill, dtype=F32)).to(dev)
    loss = torch.full((1,), loss_fill, dtype=torch.float64, device=dev)
    i32 = lambda a: dev_t(np.asarray(a, dtype=np.int32), dev)
    gnn.align_loss_l1(xv, dim, i32(left), i32(right), k, *[i32(v) for v in negs], gamma_, grad, loss)
    g = host(grad)
    assert np.all(g[:, dim:] == F32(SENTINEL)), "grad columns >= dim were written"
    return float(loss.item()), g[:, :dim]


def align_ref(x, left, right, k, negs, gamma_, device="cpu"):
    """float64 loss and gradient of oracle/gnn.py's align_loss (autograd: d|u|/du = sgn(u) with sgn(0) = 0, and no
    gradient through relu at 0), plus every hinge term v = A + γ − B [t, 2k]."""
    xt = torch.tensor(x, dtype=torch.float64, device=device, requires_grad=True)
    ill = np.stack([left, right], 1)
    loss = org.align_loss(xt, ill, gamma_, k, *negs)
    loss.backward()
    with torch.no_grad():
        li = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.long, device=device)
        A = (xt[li(left)] - xt[li(right)]).abs().sum(1)
        B1 = (xt[li(negs[0])] - xt[li(negs[1])]).abs().sum(1).reshape(len(left), k)
        B2 = (xt[li(negs[2])] - xt[li(negs[3])]).abs().sum(1).reshape(len(left), k)
        v = (A[:, None] + gamma_) - torch.cat([B1, B2], 1)
        ab = torch.cat([A[:, None].expand(-1, 2 * k), torch.cat([B1, B2], 1)], 1)
    return float(loss.detach()), host(xt.grad), host(v), host(ab)


def align_bound(x, left, right, k, negs, gamma_, v, ab, loss64, grad_fill):
    """Bound mode of the alignment loss.

    Loss: A and B each sum dim rounded |differences| (γ_{dim+1}), then fl(A + γ) and fl(dplus − B) round once each:
    |Δv| ≤ γ_{dim+3}·(A + γ + B).  A warp (one per pair: the grid covers t) adds its ≤ 2k active v's in fp32 (γ_{2k}),
    the CTA sum and the atomic add are in double, and the scale fl(1/(2kt)) is within u of 1/(2kt):
        |Δloss| ≤ scale·(Σ_{v > −Δv} Δv + γ_{2k}·Σ_{v > 0} v) + 2u·|loss|.
    A hinge with |v| ≤ Δv may flip either way and add up to 2Δv.  Real-valued coordinates never tie at 0 unless
    l == r, where both sides give sgn = 0.
    Grad: every contribution is ±scale or ±scale·active (≤ 2k), one rounding each, and entity e receives at most
    cnt_e = (appearances as l or r)·1 + (appearances as a negative) atomic adds of |·| ≤ 2k·scale onto its fill:
        |Δgrad_e| ≤ γ_{cnt_e + 2}·(|fill| + 2k·scale·cnt_e)."""
    t = len(left)
    dim = x.shape[1]
    scale = 1.0 / (2.0 * k * t)
    A, B = ab[:, :2 * k], ab[:, 2 * k:]
    dv = gamma(dim + 3) * (A + gamma_ + B)
    amb = np.abs(v) <= dv
    lb = scale * (2 * dv[v > -dv].sum() + gamma(2 * k) * (v + dv)[v > -dv].sum()) + 2 * U * abs(loss64)
    cnt = np.bincount(np.concatenate([left, right] + list(negs)), minlength=x.shape[0]).astype(np.float64)[:, None]
    gb = gamma(cnt + 2) * (np.abs(grad_fill.astype(np.float64)) + 2 * k * scale * cnt)
    # a hinge within Δv of 0 may be active in fp32 and not in float64 (or the reverse): that moves each coordinate of
    # its four entities by scale (l and r through the active count, nl and nr through their own term)
    if amb.any():
        i, j = np.nonzero(amb)
        side = j >= k
        idx = i * k + np.where(side, j - k, j)
        ents = np.concatenate([left[i], right[i], np.where(side, negs[2][idx], negs[0][idx]),
                               np.where(side, negs[3][idx], negs[1][idx])])
        gb = gb + scale * np.bincount(ents, minlength=x.shape[0])[:, None]
    return lb, gb


def raw_align(dev, t, k, dim=4, ld=4):
    """oea_align_loss_l1 through the C-ABI with valid buffers and the given t, k (the host layer derives t from the
    pair arrays and cannot pass t <= 0 with a non-NULL pointer)."""
    lib = L.load()
    x = torch.zeros(8, ld, dtype=torch.float32, device=dev)
    ids = torch.zeros(8, dtype=torch.int32, device=dev)
    grad = torch.zeros_like(x)
    loss = torch.zeros(1, dtype=torch.float64, device=dev)
    p = _ptr(ids)
    return lib.oea_align_loss_l1(_ptr(x), ld, dim, p, p, t, k, p, p, p, p, 1.0, _ptr(loss), _ptr(grad), gnn._stream_ptr())


# ======================================================================================================================
# The cases, shared by the emulator and the GPU tests.  `dev` is the device the host layer runs on.
# ======================================================================================================================
EPILOGUES = ["relu", "mask", "beta", "all"]


def case_spmm_widths(dev, i, d):
    """Every row length of ROW_LENGTHS at width d, exact: once contiguous, once with ldx, ldy > d and one epilogue
    variant (relu / mask / beta / all three, by i).  Ten hub rows, so k_spmm_finalize runs two CTAs."""
    rng = np.random.default_rng(1000 + d)
    a = csr_rows(rng, rng.permutation(ROW_LENGTHS), 4200, "int")
    DA = gnn.DeviceCsr(a, dev)
    assert DA.long_rows.numel() == 10 and DA.n_seg == 1 + 1 + 1 + 2 + 2 + 2 + 2 + 2 + 3 + 9
    X = ints(rng, (a.shape[1], d))
    want = check_spmm_exact(dev, DA, a, X)
    kind = EPILOGUES[i % 4]
    kw = dict(ldx=d + 4 * (1 + i % 3), ldy=d + 4 * (1 + (i + 1) % 3))
    if kind in ("relu", "all"):
        kw["relu"] = True
    if kind in ("mask", "all"):
        kw["mask"] = ints(rng, (a.shape[0], d), -1, 1)
    if kind in ("beta", "all"):
        kw["beta"], kw["y_old"] = (-2.0 if kind == "beta" else 0.5), ints(rng, (a.shape[0], d))
        flips = np.sign(want) * np.sign(want + kw["beta"] * kw["y_old"]) < 0
        assert flips.sum() > 4, "beta must flip signs for the epilogue order to be observable"
    check_spmm_exact(dev, DA, a, X, **kw)


def case_spmm_bound(dev, d, n_short=0, seed=0):
    """Real-valued values and X with hub rows (and n_short extra short rows), beta + relu on strided buffers."""
    rng = np.random.default_rng(2000 + d + seed)
    lengths = list(ROW_LENGTHS) + list(rng.integers(0, 40, n_short))
    a = csr_rows(rng, rng.permutation(lengths), 4200, "real")
    DA = gnn.DeviceCsr(a, dev)
    X = rng.standard_normal((a.shape[1], d)).astype(F32)
    y_old = rng.standard_normal((a.shape[0], d)).astype(F32)
    r1 = check_spmm_bound(dev, DA, a, X)
    r2 = check_spmm_bound(dev, DA, a, X, ldx=d + 8, ldy=d + 4, relu=True, beta=0.75, y_old=y_old)
    return max(r1, r2)


def hub_column_matrix(rng, values="int"):
    """700 × 700 with three non-zeros per row, column 3 in every row and column 9 in 260 rows (hub rows of the
    transpose), and row 11 with 600 non-zeros (a hub row)."""
    n = 700
    dense = np.zeros((n, n), dtype=bool)
    for r in range(n):
        dense[r, rng.choice(n, 3, replace=False)] = True
    dense[:, 3] = True
    dense[rng.choice(n, 260, replace=False), 9] = True
    dense[11, rng.choice(n, 600, replace=False)] = True
    r, c = np.nonzero(dense)
    v = nonzero_ints(rng, r.size) if values == "int" else (rng.random(r.size) + 0.25).astype(F32)
    return sp.csr_matrix((v, (r, c)), shape=(n, n))


def case_spmm_vals_and_transpose(dev, d=132):
    rng = np.random.default_rng(3)
    a = hub_column_matrix(rng)
    DA = gnn.DeviceCsr(a, dev)
    assert DA.long_rows.numel() == 1
    X = ints(rng, (a.shape[1], d))
    check_spmm_exact(dev, DA, a, X, vals=nonzero_ints(rng, a.nnz))          # values substituted on the hub row too
    T = DA.transpose()
    assert T.long_rows.numel() == 2 and T.transpose() is DA
    G = ints(rng, (a.shape[0], d))
    check_spmm_exact(dev, T, sp.csr_matrix(a.T), G)


def case_spmm_empty_and_one_row(dev):
    rng = np.random.default_rng(4)
    empty = sp.csr_matrix((5, 7), dtype=np.float32)
    DA = gnn.DeviceCsr(empty, dev)
    assert DA.nnz == 0
    got = run_spmm(dev, DA, ints(rng, (7, 8)), ldy=12)
    assert np.array_equal(got, np.zeros((5, 8), F32)), "an empty matrix must give zeros"
    for n in (0, 1, 300, 1025):
        a = csr_rows(rng, [n], 1100, "int")
        check_spmm_exact(dev, gnn.DeviceCsr(a, dev), a, ints(rng, (1100, 36)), relu=True)


def case_spmm_no_hub_plan(dev):
    """Without a hub plan (a NULL pointer or n_long = 0) the warp-per-row kernel must take every row, however long."""
    rng = np.random.default_rng(5)
    a = csr_rows(rng, [0, 3, 257, 600, 1024, 40, 1025], 1100, "int")
    DA = gnn.DeviceCsr(a, dev)
    for d in (4, 132):
        X = ints(rng, (a.shape[1], d))
        want = (a.astype(np.float64) @ X.astype(np.float64)).astype(F32)
        for hubs in (None, "empty", "plan"):
            rc, Y = raw_spmm(DA, dev_t(X, dev), hubs=hubs)
            assert rc == OK
            got = host(Y)
            bad = np.unique(np.nonzero(~(got == want))[0])
            assert bad.size == 0, "hubs=%r, d=%d: rows %s (lengths %s) not computed" % (
                hubs, d, bad, np.diff(a.indptr)[bad])


def case_spmm_rejections(dev):
    rng = np.random.default_rng(6)
    a = csr_rows(rng, [3, 0, 5], 16, "int")
    DA = gnn.DeviceCsr(a, dev)
    for d, width, rc_want in ((0, 4, ERR_DIM), (2, 4, ERR_DIM), (516, 516, ERR_DIM), (6, 8, ERR_DIM)):
        rc, Y = raw_spmm(DA, dev_t(ints(rng, (16, width)), dev), d=d)
        assert rc == rc_want, (d, rc)
        assert torch.isnan(Y).all()
    X = dev_t(ints(rng, (17, 8)), dev)
    rc, Y = raw_spmm(DA, X, x_offset=4)                                    # X not 16-byte aligned
    assert rc == ERR_ALIGN and torch.isnan(Y).all()


# ---- edge softmax cases ----------------------------------------------------------------------------------------------
def softmax_matrix(rng, values, n_hub_col=120, reps=2):
    """Rows of every SOFTMAX_LENGTHS length (reps times), then n_hub_col rows of three non-zeros that all hold column
    0 (one column taking many atomic adds in the backward).  values: 'one', 'real' (in [0.5, 1.5] with some exact
    zeros) or 'int' (in {-1, 0, 1})."""
    n_var = len(SOFTMAX_LENGTHS) * reps
    a = csr_rows(rng, rng.permutation(list(SOFTMAX_LENGTHS) * reps).tolist() + [3] * n_hub_col, 700, "int")
    a.indices[a.indptr[n_var:-1]] = 0                        # a hub row's smallest column becomes 0: still sorted
    if values == "one":
        a.data[:] = 1.0
    elif values == "real":
        a.data[:] = (rng.random(a.nnz) + 0.5).astype(F32)
        a.data[rng.random(a.nnz) < 0.1] = 0.0
    else:
        a.data[:] = rng.integers(-1, 2, a.nnz).astype(F32)
    return a


def case_softmax_exact_fwd(dev, edge_mode):
    """Rows of equal logits: every exponent is exactly 1 and alpha must be fl(1/n); a single edge gives 1.  Node mode
    holds s2 constant and a = 1 (or a = 0 on some rows: every logit 0); edge mode gives each row one logit, some of
    them ±1e4 or −88.25."""
    rng = np.random.default_rng(7 + edge_mode)
    a = softmax_matrix(rng, "one")
    DA = gnn.DeviceCsr(a, dev)
    n_row = np.diff(a.indptr)
    row = np.repeat(np.arange(a.shape[0]), n_row)
    if edge_mode:
        per_row = rng.choice([1e4, -1e4, 3.5, 0.0, -88.25, 60.0], a.shape[0]).astype(F32)
        got = softmax_fwd(dev, DA, edge_logits=per_row[row])
    else:
        a.data[row % 5 == 2] = 0.0
        DA = gnn.DeviceCsr(a, dev)
        s1 = (rng.integers(-8, 9, a.shape[0]) / 4).astype(F32)
        got = softmax_fwd(dev, DA, s1=s1, s2=np.full(a.shape[1], 0.75, F32))
    want = F32(1) / n_row[row].astype(F32)
    assert_exact(got, want, "alpha on equal logits")
    assert np.all(got[n_row[row] == 1] == 1.0)


def node_scores(rng, n_r, n_c, spread):
    """s1 = ±[1.5, 3], s2 in [−0.5, 0.5] with 5 % of the columns at up to ±spread: |s1 + s2| ≥ 1 off those columns, so
    a·(s1 + s2) is either exactly 0 (a = 0) or far from the leaky kink."""
    s1 = (rng.uniform(1.5, 3.0, n_r) * rng.choice([-1, 1], n_r)).astype(F32)
    s2 = rng.uniform(-0.5, 0.5, n_c).astype(F32)
    wide = rng.random(n_c) < (0.05 if spread else 0.0)
    s2[wide] = rng.uniform(-spread, spread, wide.sum()).astype(F32)
    return dict(s1=s1, s2=s2)


def case_softmax_bound(dev, edge_mode, exp_ulps, seed=0, spread=400.0):
    """Real-valued logits against float64 within softmax_bound.  Node mode: a in [0.5, 1.5] with some exact zeros,
    s1, s2 from node_scores; edge mode: rows of N(0, 3) logits, of uniform logits over
    [−spread/4, spread/4], around +1e4 and around −1e4.  Returns (DA, a, inputs, alpha, max err/bound)."""
    rng = np.random.default_rng(20 + seed + 10 * edge_mode)
    a = softmax_matrix(rng, "real")
    DA = gnn.DeviceCsr(a, dev)
    row = np.repeat(np.arange(a.shape[0]), np.diff(a.indptr))
    if edge_mode:
        kind = rng.integers(0, 4, a.shape[0])[row]
        logit = np.select([kind == 0, kind == 1, kind == 2],
                          [3 * rng.standard_normal(a.nnz), rng.uniform(-spread / 4, spread / 4, a.nnz),
                           1e4 + 3 * rng.standard_normal(a.nnz)], -1e4 + 3 * rng.standard_normal(a.nnz)).astype(F32)
        inputs = dict(edge_logits=logit)
    else:
        inputs = node_scores(rng, a.shape[0], a.shape[1], spread)
    pre = pre_activation(a, **inputs)
    l = np.where(pre > 0, pre, SLOPE * pre)
    lo, hi = np.full(a.shape[0], np.inf), np.full(a.shape[0], -np.inf)
    np.minimum.at(lo, row, l)
    np.maximum.at(hi, row, l)
    assert spread < 300 or (hi - lo).max() > 88, "no row spreads its logits over more than 88"
    got, ratio = check_softmax_bound(dev, DA, a, exp_ulps, **inputs)
    return DA, a, inputs, got, ratio


def case_softmax_bwd_bound(dev, edge_mode, exp_ulps):
    """The backward as a function of the kernel's alpha and a real dalpha, ds2 accumulated into a real fill."""
    DA, a, inputs, alpha, _ = case_softmax_bound(dev, edge_mode, exp_ulps, seed=5, spread=40.0)
    rng = np.random.default_rng(30 + edge_mode)
    dalpha = rng.standard_normal(a.nnz).astype(F32)
    pre = pre_activation(a, **inputs)
    assert not np.any((pre != 0) & (np.abs(pre) < 1e-3)), "a logit sits at the leaky kink: pick other data"
    fill = rng.standard_normal(a.shape[1]).astype(F32)
    ds1, ds2 = softmax_bwd(dev, DA, alpha, dalpha, **inputs, ds2_fill=fill)
    ref = softmax_bwd_ref(a, alpha, dalpha, pre, SLOPE, not edge_mode, fill)
    if edge_mode:
        assert_within(ds1, ref[0], ref[1], "dlogit")
    else:
        assert_within(ds1, ref[0], ref[1], "ds1")
        assert_within(ds2, ref[2], ref[3], "ds2")


def case_softmax_bwd_exact(dev, edge_mode):
    """Dyadic alpha in {0, 1/16, 1/8}, dalpha in {0, ±1/2, ±1}, slope 1/4; node-mode a in {-1, 0, 1} and s1, s2 in
    quarters, so that pre is exactly 0 on many edges (the slope branch, as torch takes it); ds2 accumulated into a
    quarter-valued fill, column 0 taking more than a hundred atomic adds; ds1 of empty rows overwritten with 0.
    Every partial sum is a multiple of 2^-11 below 2^13: exact in fp32 in any order."""
    rng = np.random.default_rng(40 + edge_mode)
    a = softmax_matrix(rng, "int")
    DA = gnn.DeviceCsr(a, dev)
    slope = 0.25
    alpha = (rng.integers(0, 3, a.nnz) / 16).astype(F32)
    dalpha = (rng.integers(-2, 3, a.nnz) / 2).astype(F32)
    if edge_mode:
        inputs = dict(edge_logits=(rng.integers(-2, 3, a.nnz) / 2).astype(F32))
    else:
        inputs = dict(s1=(rng.integers(-4, 5, a.shape[0]) / 4).astype(F32), s2=(rng.integers(-4, 5, a.shape[1]) / 4).astype(F32))
    pre = pre_activation(a, **inputs)
    fill = (rng.integers(-8, 9, a.shape[1]) / 4).astype(F32)
    ds1, ds2 = softmax_bwd(dev, DA, alpha, dalpha, **inputs, slope=slope, ds2_fill=fill)
    ref = softmax_bwd_ref(a, alpha, dalpha, pre, slope, not edge_mode, fill)
    dl = ref[0] if edge_mode else ref[4]
    w = alpha.astype(np.float64) * (a.data if not edge_mode else 1.0)
    on_kink = (pre == 0) & (dl != 0) if not edge_mode else (pre == 0) & (w != 0) & (dl != 0)
    assert on_kink.sum() > 10, "the slope branch at pre = 0 must be observable"
    if edge_mode:
        assert_exact(ds1, ref[0], "dlogit")
    else:
        assert_exact(ds1, ref[0], "ds1")
        assert_exact(ds2, ref[2], "ds2")
        assert np.bincount(a.indices)[0] > 100
        assert np.all(ds1[np.diff(a.indptr) == 0] == 0)


def case_sddmm(dev, d, exact):
    rng = np.random.default_rng(50 + d)
    a = softmax_matrix(rng, "one", n_hub_col=8, reps=1)
    DA = gnn.DeviceCsr(a, dev)
    if exact:
        G, M = ints(rng, (a.shape[0], d)), ints(rng, (a.shape[1], d))
    else:
        G, M = rng.standard_normal((a.shape[0], d)).astype(F32), rng.standard_normal((a.shape[1], d)).astype(F32)
    got = sddmm(dev, DA, G, M, d + 4, d + 8)
    want, bound = sddmm_ref(a, G, M)
    if exact:
        assert_exact(got, want, "sddmm d=%d" % d)
    else:
        assert_within(got, want, bound, "sddmm d=%d" % d)


def case_softmax_arguments(dev):
    """A NULL ds2 is accepted in edge-logit mode and refused in node mode; mixed s1 / s2 are refused."""
    lib = L.load()
    a = csr_rows(np.random.default_rng(8), [2, 0, 3], 5, "int")
    DA = gnn.DeviceCsr(a, dev)
    v = torch.ones(8, dtype=torch.float32, device=dev)
    out = torch.zeros(8, dtype=torch.float32, device=dev)
    cs = DA.c_struct()
    st = gnn._stream_ptr()
    assert lib.oea_edge_softmax_bwd(C.byref(cs), None, None, SLOPE, _ptr(v), _ptr(v), _ptr(out), None, st) == OK
    assert lib.oea_edge_softmax_bwd(C.byref(cs), _ptr(v), _ptr(v), SLOPE, _ptr(v), _ptr(v), _ptr(out), None, st) == ERR_NULL
    assert lib.oea_edge_softmax_fwd(C.byref(cs), _ptr(v), None, SLOPE, _ptr(out), st) == ERR_NULL
    assert lib.oea_sddmm(C.byref(cs), _ptr(v), 4, _ptr(v), 4, 2, _ptr(out), st) == ERR_DIM


def duplicate_matrix(rng, n=300):
    """RDGCN's r_mat shape: one entry per triple, duplicated (h, t) pairs kept as separate entries (CSR built by hand,
    as the COO conversion would sum them); rows 0 and 1 are hub rows, column 2 a hub column."""
    h = np.concatenate([rng.integers(0, n, 4 * n), np.zeros(400, np.int64), np.ones(300, np.int64),
                        rng.integers(0, n, 280)])
    t = np.concatenate([rng.integers(0, n, 4 * n), rng.integers(0, n, 400), rng.integers(0, 40, 300),
                        np.full(280, 2)])
    order = np.lexsort((t, h))
    indptr = np.concatenate([[0], np.cumsum(np.bincount(h, minlength=n))])
    return sp.csr_matrix((np.ones(h.size, np.float64), t[order], indptr), shape=(n, n))


def case_transpose_perm(dev):
    """transpose_perm maps every edge of the transpose's CSR order to its edge in the matrix, duplicates included."""
    rng = np.random.default_rng(9)
    a = duplicate_matrix(rng)
    DA = gnn.DeviceCsr(a, dev, keep_duplicates=True)
    assert DA.nnz == a.nnz
    T = DA.transpose()
    perm = host(DA.transpose_perm())
    assert np.array_equal(np.sort(perm), np.arange(a.nnz)), "transpose_perm is not a permutation"
    rows = np.repeat(np.arange(a.shape[0]), np.diff(a.indptr))
    t_rows = np.repeat(np.arange(T.shape[0]), np.diff(host(T.rowptr)))
    assert np.array_equal(t_rows, host(DA.col)[perm]) and np.array_equal(host(T.col), rows[perm])
    b = sp.random(50, 60, density=0.2, random_state=1, format="csr", dtype=np.float32)
    DB = gnn.DeviceCsr(b, dev)
    assert np.array_equal(host(DB.val)[host(DB.transpose_perm())], host(DB.transpose().val))


def case_aggregate_fn(dev, edge_mode, exp_ulps):
    """GatAggregateFn (node mode, on a matrix with a hub row and hub columns) and EdgeLogitAggregateFn (edge mode, on a
    matrix with duplicated (h, t) entries whose logits differ), forward and autograd backward, against float64:
      alpha (the kernel's, read from the autograd context) within softmax_bound of oracle/gnn.py's;
      out within γ_{n+2}·Σ|alpha M| of Σ alpha·M (float64, the kernel's alpha);
      dM = Aᵀ-aggregation of gOut with the kernel's alpha moved by transpose_perm, within γ_{m+2}·Σ|alpha g|;
      ds1 / ds2 / dlogit within softmax_bwd_ref's bound around the float64 backward of the kernel's alpha and the
      float64 dalpha = <gOut_i, M_j>, whose SDDMM error γ_d·Σ|g m| is carried through."""
    rng = np.random.default_rng(60 + edge_mode)
    a = duplicate_matrix(rng) if edge_mode else hub_column_matrix(rng, "real")
    DA = gnn.DeviceCsr(a, dev, keep_duplicates=edge_mode)
    d = 36
    n_r, n_c = a.shape
    row = np.repeat(np.arange(n_r), np.diff(a.indptr))
    M = rng.standard_normal((n_c, d)).astype(F32)
    G = rng.standard_normal((n_r, d)).astype(F32)
    Mt = dev_t(M, dev).requires_grad_(True)
    if edge_mode:
        logit = (3 * rng.standard_normal(a.nnz)).astype(F32)
        dup = np.flatnonzero((np.diff(row) == 0) & (np.diff(a.indices) == 0))
        assert dup.size > 10 and np.all(logit[dup] != logit[dup + 1]), "duplicates must carry different logits"
        inputs = dict(edge_logits=logit)
        lt = dev_t(logit, dev).requires_grad_(True)
        out = gnn.EdgeLogitAggregateFn.apply(lt, Mt, DA, SLOPE)
    else:
        inputs = node_scores(rng, n_r, n_c, 0.0)
        s1t, s2t = dev_t(inputs["s1"], dev).requires_grad_(True), dev_t(inputs["s2"], dev).requires_grad_(True)
        out = gnn.GatAggregateFn.apply(s1t, s2t, Mt, DA, SLOPE)
    alpha = host(out.grad_fn.saved_tensors[-1])
    pre = pre_activation(a, **inputs)
    want_alpha = softmax_ref(a, **inputs)
    assert_within(alpha, want_alpha, softmax_bound(a, want_alpha, pre, SLOPE, not edge_mode, exp_ulps), "alpha")
    al = alpha.astype(np.float64)
    Aal = sp.csr_matrix((al, a.indices, a.indptr), shape=a.shape)
    absA = sp.csr_matrix((np.abs(al), a.indices, a.indptr), shape=a.shape)
    n_row = np.diff(a.indptr)[:, None]
    assert_within(host(out), Aal @ M.astype(np.float64), gamma(n_row + 2) * (absA @ np.abs(M.astype(np.float64))), "out")
    (out * dev_t(G, dev)).sum().backward()
    m_col = np.bincount(a.indices, minlength=n_c)[:, None]
    assert_within(host(Mt.grad), Aal.T @ G.astype(np.float64), gamma(m_col + 2) * (absA.T @ np.abs(G.astype(np.float64))),
                  "dM")
    dalpha, dalpha_err = sddmm_ref(a, G, M)
    ref = softmax_bwd_ref(a, alpha, dalpha, pre, SLOPE, not edge_mode, np.zeros(n_c, F32), dalpha_err)
    assert not np.any((pre != 0) & (np.abs(pre) < 1e-3)), "a logit sits at the leaky kink: pick other data"
    if edge_mode:
        assert_within(host(lt.grad), ref[0], ref[1], "dlogit")
    else:
        assert_within(host(s1t.grad), ref[0], ref[1], "ds1")
        assert_within(host(s2t.grad), ref[2], ref[3], "ds2")


# ---- alignment loss cases --------------------------------------------------------------------------------------------
def case_align_exact(dev, dim, t, k, seed=0):
    """Integer embeddings, integer γ, t·k a power of two: loss and gradient bit-identical to float64, both accumulated
    into non-zero fills, with ld > dim.  With t >= 4 the pairs also hold l == r (A = 0), a negative with nl == nr
    (B = 0), a negative equal to its positive pair, a hinge of exactly zero (B = A + γ: no gradient), and one entity
    in a third of the pairs; sgn(0) ties occur on every seventh coordinate."""
    assert t * k & (t * k - 1) == 0
    rng = np.random.default_rng(70 + dim + seed)
    n, gamma_ = 40, 3.0
    x = ints(rng, (n, dim))
    left, right, negs = align_case(rng, n - 2, t, k)
    zero_hinge = False
    if t >= 4:
        right[0] = left[0]                                  # A = 0
        negs[1][k] = left[1]                                # (l, l): B = 0
        negs[2][k] = left[1]                                # (l, r): a negative equal to its positive pair
        left[3::3] = 5                                      # one entity in a third of the pairs
        z1, z2 = n - 2, n - 1                               # right-side negative of pair 2 with B = A + γ
        x[z1] = 0
        x[z2] = 0
        x[z2, 0] = np.abs(x[left[2]] - x[right[2]]).sum() + gamma_
        negs[2][2 * k], negs[3][2 * k] = z1, z2
        zero_hinge = True
    grad_fill = (ints(rng, (n, dim)) / 2).astype(F32)
    loss, grad = run_align(dev, x, dim + 3, left, right, k, negs, gamma_, grad_fill, 1.25)
    loss64, grad64, v, _ = align_ref(x, left, right, k, negs, gamma_)
    if zero_hinge:
        assert v[2, k] == 0.0
    assert loss == 1.25 + loss64, (loss, 1.25 + loss64)
    assert_exact(grad, grad_fill.astype(np.float64) + grad64, "grad")


def case_align_bound(dev, dim, t, k, hub=False, seed=0, ref_device="cpu"):
    """Real-valued embeddings within align_bound; with hub=True one entity fills 10 % of the negative slots."""
    rng = np.random.default_rng(80 + dim + seed)
    n, gamma_ = max(64, t // 4), 1.5
    x = rng.standard_normal((n, dim)).astype(F32)
    left, right, negs = align_case(rng, n, t, k)
    if hub:
        for j in (1, 2):
            negs[j][rng.random(t * k) < 0.1] = 7
    grad_fill = rng.standard_normal((n, dim)).astype(F32)
    loss, grad = run_align(dev, x, dim + 5, left, right, k, negs, gamma_, grad_fill, -0.5)
    loss64, grad64, v, ab = align_ref(x, left, right, k, negs, gamma_, ref_device)
    lb, gb = align_bound(x, left, right, k, negs, gamma_, v, ab, loss64, grad_fill)
    assert abs(loss - (-0.5 + loss64)) <= lb + 2 * U * 0.5, (loss, -0.5 + loss64, lb)
    assert_within(grad, grad_fill.astype(np.float64) + grad64, gb, "grad")


def case_align_rejections(dev):
    for t, k in ((0, 1), (-1, 1), (1, 0), (4, -2)):
        assert raw_align(dev, t, k) == ERR_SHAPE, (t, k)
    assert raw_align(dev, 1, 1, dim=5, ld=4) == ERR_SHAPE
    assert raw_align(dev, 1, 1) == OK
