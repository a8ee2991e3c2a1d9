"""Path (iii) at its edges: the similarity tile kernel with its top-k / rank / store epilogues, the short-contraction
store kernel, the split merge, the stored-matrix CSLS kernels, the radix selection with its gather-sort and the row
normaliser (openea_b200/csrc/oea_sim.cu, oea_match.cu), against float64 references.  tests/test_emu_sim_edges.py runs
these cases on the warp emulator, tests/test_zz_sim_edges_gpu.py on the GPU.

Two reference modes:

* Exact mode.  Entries are small integers in [-3, 3].  Every inner and L1 contraction, and the L2 accumulator, is then
  an integer below 2^24, exact in fp32 and float64 whatever the summation order.  The reference applies the kernels'
  fp32 operation sequence to it in NumPy float32 (each NumPy float32 operation is correctly rounded, and the kernels
  are built without fast math): 1 − acc, 1 − sqrtf(acc), the CSLS means fl32(Σ)/fl32(k) where Σ is an exact integer for
  inner and L1, and (2·s − r) − c.  Every output must be bit-identical: values, means, top-k indices, top-1, ranks and
  selected sets, huge tie classes included.
* Bound mode.  Real-valued entries.  Values are compared with float64 within a first-order fp32 error bound δ per
  entry (derived at `bound_matrix`), index outputs by intervals that no near-tie can break:
  rank[i] ∈ [#{s64 > g64 + 2δ}, #{s64 ≥ g64 − 2δ}], s64[top1] ≥ max s64 − 2δ, every top-k index has
  s64 ≥ (k-th s64) − 2δ with no duplicates, and the top-k values lie within δ of float64's sorted top-k.
"""
import ctypes as C

import numpy as np
import torch

from openea_b200 import lib as L
from openea_b200.engine import _ptr

F32 = np.float32
U = float(np.finfo(np.float32).eps) / 2          # unit round-off of fp32
TILE = 128                                       # the tile kernel's TM = TN
# contraction lengths: one and two 16-wide K chunks (fewer than the 3 pipeline stages), each tail length (4, 8, 12),
# the short-K limit 104 and its first pitch above, and long ones
PITCHES = [4, 8, 12, 16, 20, 32, 36, 100, 104, 108, 300, 512]
KS = [1, 7, 8, 9, 16, 17, 31, 32]                # every kcap bucket edge of the tile kernel's list (8 / 16 / 32)


def gamma(n):
    return n * U / (1 - n * U)


def ints(rng, n, d, lo=-3, hi=3):
    return rng.integers(lo, hi + 1, (n, d)).astype(F32)


def host(t):
    return t.detach().cpu().numpy()


def dev_rows(F, x):
    """Rows on the engine's device, zero-padded to the kernels' pitch (no normalisation)."""
    return F.to_device_rows(np.ascontiguousarray(x, dtype=F32), False)[0]


# ---- exact-mode references ---------------------------------------------------------------------------------------
def exact_sim(e1, e2, metric):
    """fp32 similarity of integer rows: the contraction is exact, then the kernels' fp32 epilogue."""
    a, b = e1.astype(np.float64), e2.astype(np.float64)
    if metric == "inner":
        return (a @ b.T).astype(F32)
    out = np.empty((a.shape[0], b.shape[0]), dtype=F32)
    for r0 in range(0, a.shape[0], 64):
        dlt = a[r0:r0 + 64, None, :] - b[None, :, :]
        if metric == "manhattan":
            out[r0:r0 + 64] = F32(1) - np.abs(dlt).sum(2).astype(F32)
        else:
            out[r0:r0 + 64] = F32(1) - np.sqrt((dlt * dlt).sum(2).astype(F32))
    return out


def exact_means(s, k):
    """calculate_nearest_k of an integer-valued fp32 matrix: the sum of the k largest is an exact integer."""
    top = -np.sort(-s.astype(np.float64), axis=1)[:, :k]
    return top.sum(1).astype(F32) / F32(k)


def csls(s, r, c):
    return (F32(2) * s - r[:, None]) - c[None, :]


def order_desc(s):
    """Column order of each row by (value descending, index ascending)."""
    cols = np.broadcast_to(np.arange(s.shape[1]), s.shape)
    return np.lexsort((cols, -s.astype(np.float64)), axis=1)


def topk_ref(s, k):
    o = order_desc(s)[:, :k]
    return np.take_along_axis(s, o, 1), o.astype(np.int32)


def rank_ref(s, gold):
    n = s.shape[0]
    g = s[np.arange(n), gold][:, None]
    cols = np.arange(s.shape[1])[None, :]
    rk = (s > g).sum(1) + ((s == g) & (cols < gold[:, None])).sum(1)
    return s.argmax(1).astype(np.int32), rk.astype(np.int32)


# ---- bound-mode references ---------------------------------------------------------------------------------------
def bound_matrix(a, b, metric, d, normalised_on_device=False):
    """float64 similarity S64 and a bound δ ≥ |fl32(S) − S64| per entry, from float32 operands a, b (torch float64 here).

    inner:  fl(Σ a_k b_k) with fmaf, d terms: |err| ≤ γ_d·Σ|a_k b_k| (Higham, Thm 3.5).  When the rows were normalised
            on the device (cosine), each operand entry carries the normaliser's relative error, at most
            γ_d/2 (the fp32 sum of squares under the square root) + 3u (sqrt, reciprocal, product); that adds
            (γ_d + 6u)·Σ|a_k b_k| against the float64 cosine.
    L1:     each |a_k − b_k| carries one rounding, the sum d more: |acc err| ≤ γ_{d+1}·acc; 1 − acc adds u·|S|.
    L2:     (a_k − b_k)² by a rounded difference and an fma, then d sums: |acc err| ≤ γ_{d+2}·acc; sqrt(acc(1+θ))
            is within θ/2 of sqrt(acc) relatively, plus its own rounding u: |dist err| ≤ (γ_{d+2}/2 + u)·dist;
            1 − dist adds u·|S|.
    The padding columns are zero on both sides and add nothing."""
    if metric in ("inner", "cosine"):
        s = a @ b.T
        w = a.abs() @ b.abs().T
        g = gamma(d) * (2.0 if normalised_on_device else 1.0) + (6 * U if normalised_on_device else 0.0)
        return s, g * w
    if metric == "manhattan":
        acc = torch.cdist(a, b, p=1)
        s = 1 - acc
        return s, gamma(d + 1) * acc + U * s.abs()
    dist = torch.cdist(a, b, p=2, compute_mode="donot_use_mm_for_euclid_dist")
    s = 1 - dist
    return s, (gamma(d + 2) / 2 + U) * dist + U * s.abs()


def bound_means(s, dl, k):
    """Mean of the k largest of each row and its bound.  The fp32 top-k values are the k largest of a matrix within δ of
    s, so each sorted value is within max_row δ of float64's; the fp32 sum of k of them adds γ_{k-1}·Σ|v|, the division
    u·|mean|."""
    top = torch.topk(s, k, dim=1).values
    m = top.mean(1)
    dm = dl.max(1).values + gamma(max(k - 1, 0)) * (top.abs().mean(1) + dl.max(1).values) + U * m.abs()
    return m, dm


def bound_csls(s, dl, r, dr, c, dc):
    """(2·s − r) − c in fp32 from values carrying δ, δ_r, δ_c: 2δ + δ_r + δ_c, plus the two roundings."""
    t = 2 * s - r[:, None]
    out = t - c[None, :]
    return out, 2 * dl + dr[:, None] + dc[None, :] + U * (t.abs() + out.abs())


def check_values_bound(got, s64, dl, what):
    got = torch.as_tensor(got, dtype=torch.float64, device=s64.device)
    err = (got - s64).abs() - dl
    assert float(err.max()) <= 0.0, "%s: %.3g beyond the fp32 bound" % (what, float(err.max()))


def check_rank_interval(top1, rk, s64, dl, gold, what):
    """The interval rule on the rows given (s64, dl [rows, n2]; top1, rk, gold [rows])."""
    dev = s64.device
    top1 = torch.as_tensor(top1, dtype=torch.long, device=dev)
    rk = torch.as_tensor(rk, dtype=torch.long, device=dev)
    gold = torch.as_tensor(gold, dtype=torch.long, device=dev)
    rows = torch.arange(s64.shape[0], device=dev)
    d2 = 2 * dl.max(1).values[:, None]
    g = s64[rows, gold][:, None]
    lo = (s64 > g + d2).sum(1)
    hi = (s64 >= g - d2).sum(1)
    assert bool(((rk >= lo) & (rk <= hi)).all()), "%s: rank outside its interval" % what
    assert bool((top1 >= 0).all()) and bool((top1 < s64.shape[1]).all()), what
    assert bool((s64[rows, top1][:, None] >= s64.max(1).values[:, None] - d2).all()), "%s: top-1 not a maximum" % what


def check_topk_interval(val, idx, s64, dl, k, what):
    dev = s64.device
    idx = torch.as_tensor(idx, dtype=torch.long, device=dev)
    val = torch.as_tensor(val, dtype=torch.float64, device=dev)
    d = dl.max(1).values[:, None]
    top = torch.topk(s64, k, dim=1).values
    assert bool((idx >= 0).all()) and bool((idx < s64.shape[1]).all()), what
    srt = idx.sort(1).values
    assert bool((srt[:, 1:] != srt[:, :-1]).all()), "%s: duplicate top-k index" % what
    assert bool((s64.gather(1, idx) >= top[:, -1:] - 2 * d).all()), "%s: a top-k index below the k-th value" % what
    assert bool(((val - top).abs() <= d).all()), "%s: top-k values off float64's" % what
    assert bool(((val - s64.gather(1, idx)).abs() <= d).all()), "%s: value and index disagree" % what


# ---- split bookkeeping -------------------------------------------------------------------------------------------
def splits_of(F, e1, e2, d, k=1):
    """(picked, effective) column-split counts of a tile-kernel launch, read from the workspace size of the ABI."""
    lib = L.load()
    cfg = F._cfg("inner", e1, e2, d)
    n1, n2 = e1.shape[0], e2.shape[0]
    picked = lib.oea_sim_topk_workspace_bytes(C.byref(cfg), k) // (n1 * k * 8)
    tiles = (n2 + TILE - 1) // TILE
    per = (tiles + picked - 1) // picked
    return picked, (tiles + per - 1) // per, per


# ---- tile kernel, exact mode -------------------------------------------------------------------------------------
def check_exact(F, e1, e2, metric, k, csls_k=0, gold=None, shortk=(False, True), monkeypatch=None, wants=True):
    """All three epilogues of the tile kernel (and the short-K store kernel) on integer rows, bit for bit.  Returns the
    reference matrix."""
    n1, n2 = e1.shape[0], e2.shape[0]
    d = e1.shape[1]
    t1, t2 = dev_rows(F, e1), dev_rows(F, e2)
    s = exact_sim(e1, e2, metric)
    r = c = None
    if csls_k:
        rr, cc = exact_means(s, csls_k), exact_means(s.T, csls_k)
        r, c = F.csls_offsets(t1, t2, d, metric, csls_k)
        assert np.array_equal(host(r), rr) and np.array_equal(host(c), cc), "CSLS means"
        s = csls(s, rr, cc)
    # store epilogue: the streaming tile kernel and the resident-panel short-K kernel give the same bits
    for no_short in shortk:
        if monkeypatch is not None:
            monkeypatch.setenv("OEA_SIM_NO_SHORTK", "1" if no_short else "0")
        got = host(F.sim_matrix(t1, t2, d, metric, r, c))
        assert np.array_equal(got, s), "store epilogue (no_shortk=%s): %d entries differ" % (no_short, int((got != s).sum()))
    # top-k epilogue + merge, each output alone and all three together
    wv, wi = topk_ref(s, k)
    # the mean of k integers is exact: inner and L1 without CSLS (CSLS values and L2 values are not integers)
    wm = wv.astype(np.float64).sum(1).astype(F32) / F32(k) if metric != "euclidean" and not csls_k else None
    res = F.topk(t1, t2, d, metric, k, r, c)
    assert np.array_equal(host(res["idx"]), wi), "top-k indices: %d rows differ" % int((host(res["idx"]) != wi).any(1).sum())
    assert np.array_equal(host(res["val"]), wv), "top-k values"
    if wm is not None:
        assert np.array_equal(host(res["mean"]), wm), "top-k means"
    if wants:
        for want in ("val", "idx", "mean"):
            one = F.topk(t1, t2, d, metric, k, r, c, want=(want,))
            assert set(k_ for k_, v in one.items() if v is not None) == {want}
            assert np.array_equal(host(one[want]), host(res[want])), "top-k %s requested alone" % want
    # rank epilogue
    gold = np.arange(n1) % n2 if gold is None else np.asarray(gold)
    w1, wr = rank_ref(s, gold)
    top1, rk = F.rank(t1, t2, d, metric, torch.as_tensor(gold, dtype=torch.int32, device=t1.device), r, c)
    assert np.array_equal(host(top1), w1), "top-1: %d rows differ" % int((host(top1) != w1).sum())
    assert np.array_equal(host(rk), wr), "rank: %d rows differ" % int((host(rk) != wr).sum())
    return s


def check_eval_both_strategies(F, e1, e2, metric, csls_k, gold):
    """eval_alignment streaming and materialised: identical top-1 and rank, equal to the exact reference."""
    s = exact_sim(e1, e2, metric)
    s = csls(s, exact_means(s, csls_k), exact_means(s.T, csls_k))
    w1, wr = rank_ref(s, gold)
    for mat in (False, True):
        top1, rk, *_ = F.eval_alignment(e1, e2, [1, 5], metric, False, csls_k, gold=gold, materialize=mat)
        assert np.array_equal(host(top1), w1), "top-1, materialize=%s" % mat
        assert np.array_equal(host(rk), wr), "rank, materialize=%s" % mat


def tie_rows(rng, n2, d, n_dup, spread):
    """n2 integer rows in which `n_dup` copies of one row sit at columns spread over the whole range (other tiles, other
    splits), the first copy at column 0 and the last at column n2 − 1."""
    e2 = ints(rng, n2, d)
    cols = np.unique(np.concatenate([[0, n2 - 1], rng.choice(n2, n_dup - 2, replace=False)]))[:n_dup] if spread else \
        np.arange(n_dup)
    e2[cols] = e2[cols[0]]
    return e2, cols


# ---- bound mode --------------------------------------------------------------------------------------------------
def real_rows(rng, n, d, kind, base=None):
    if kind == "random":
        return rng.standard_normal((n, d)).astype(F32)
    if kind == "near":          # near-duplicates of `base`: values 1e-4 apart, many near-ties
        return (base[rng.integers(0, len(base), n)] + 1e-4 * rng.standard_normal((n, d))).astype(F32)
    x = rng.standard_normal((n, d))
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(F32)


def check_bound(F, e1, e2, metric, k, csls_k=0, normalize=False, gold=None):
    """Values within the fp32 bound of float64, indices by the interval rules (top-k, rank, both CSLS strategies)."""
    n1, n2 = e1.shape[0], e2.shape[0]
    d = e1.shape[1]
    cosine = metric == "cosine" or normalize
    t1, t2, _ = F._prep_pair(e1, e2, metric, normalize)
    a = torch.as_tensor(e1, dtype=torch.float64, device=t1.device)
    b = torch.as_tensor(e2, dtype=torch.float64, device=t1.device)
    if cosine:
        a, b = a / a.norm(dim=1, keepdim=True), b / b.norm(dim=1, keepdim=True)
    s64, dl = bound_matrix(a, b, metric, d, cosine)
    r = c = None
    if csls_k:
        r64, dr = bound_means(s64, dl, csls_k)
        c64, dc = bound_means(s64.T, dl.T, csls_k)
        r, c = F.csls_offsets(t1, t2, d, metric, csls_k)
        check_values_bound(host(r), r64, dr, "row means")
        check_values_bound(host(c), c64, dc, "column means")
        s64, dl = bound_csls(s64, dl, r64, dr, c64, dc)
    check_values_bound(host(F.sim_matrix(t1, t2, d, metric, r, c)), s64, dl, "stored matrix")
    res = F.topk(t1, t2, d, metric, k, r, c)
    check_topk_interval(host(res["val"]), host(res["idx"]), s64, dl, k, "top-k")
    gold = np.arange(n1) % n2 if gold is None else np.asarray(gold)
    top1, rk = F.rank(t1, t2, d, metric, torch.as_tensor(gold, dtype=torch.int32, device=t1.device), r, c)
    check_rank_interval(host(top1), host(rk), s64, dl, gold, "rank")
    if csls_k:
        for mat in (False, True):
            top1, rk, *_ = F.eval_alignment(e1, e2, [1], metric, normalize, csls_k, gold=gold, materialize=mat)
            check_rank_interval(host(top1), host(rk), s64, dl, gold, "eval_alignment materialize=%s" % mat)


# ---- stored-matrix kernels (raw ABI) -----------------------------------------------------------------------------
def check_matrix_rank(dev, n_rows, n_cols, ld, col_shift, csls_on, seed):
    """oea_matrix_rank on an integer matrix with leading dimension `ld` and the column offsets starting `col_shift`
    floats into their buffer (col_shift % 4 != 0 → unaligned: the scalar path).  Gold at every position mod 4, inside
    tie classes, at column 0 and at the last column."""
    lib = L.load()
    rng = np.random.default_rng(seed)
    s = rng.integers(-4, 5, (n_rows, n_cols)).astype(F32)
    store = np.zeros((n_rows, ld), dtype=F32)
    store[:, :n_cols] = s
    gold = rng.integers(0, n_cols, n_rows)
    gold[:8] = [0, n_cols - 1, 1 % n_cols, 2 % n_cols, 3 % n_cols, 4 % n_cols, 5 % n_cols, 6 % n_cols]
    rv = (rng.integers(-40, 41, n_rows) / 4).astype(F32)
    cv = (rng.integers(-40, 41, n_cols) / 4).astype(F32)
    want = csls(s, rv, cv) if csls_on else s
    w1, wr = rank_ref(want, gold)
    t = torch.as_tensor(store, device=dev)
    cbuf = torch.zeros(n_cols + col_shift, dtype=torch.float32, device=dev)
    cbuf[col_shift:] = torch.as_tensor(cv)
    cpt = cbuf[col_shift:]
    rt = torch.as_tensor(rv, device=dev)
    g = torch.as_tensor(gold, dtype=torch.int32, device=dev)
    top1 = torch.empty(n_rows, dtype=torch.int32, device=dev)
    rk = torch.empty(n_rows, dtype=torch.int32, device=dev)
    L.check(lib.oea_matrix_rank(_ptr(t), ld, n_rows, n_cols, _ptr(rt) if csls_on else None, _ptr(cpt) if csls_on else None,
                                _ptr(g), _ptr(top1), _ptr(rk), None), "oea_matrix_rank")
    _sync(dev)
    assert np.array_equal(host(top1), w1), "top-1: %d rows differ" % int((host(top1) != w1).sum())
    assert np.array_equal(host(rk), wr), "rank: %d rows differ" % int((host(rk) != wr).sum())
    assert set((gold % 4).tolist()) == {0, 1, 2, 3}


def check_matrix_means(dev, n_rows, n_cols, k, seed, lo=-50, hi=50):
    """oea_matrix_topk_mean by row and by column on an integer matrix: exact sums, bit-identical means.  Returns the
    number of rows per split of the column form."""
    lib = L.load()
    rng = np.random.default_rng(seed)
    s = rng.integers(lo, hi + 1, (n_rows, n_cols)).astype(F32)
    ld = (n_cols + 3) // 4 * 4
    store = np.zeros((n_rows, ld), dtype=F32)
    store[:, :n_cols] = s
    t = torch.as_tensor(store, device=dev)
    out = torch.empty(max(n_rows, n_cols), dtype=torch.float32, device=dev)
    if k <= n_cols:
        L.check(lib.oea_matrix_topk_mean(_ptr(t), ld, n_rows, n_cols, k, 0, _ptr(out), None, 0, None), "row means")
        _sync(dev)
        assert np.array_equal(host(out[:n_rows]), exact_means(s, k)), "row means"
    nb = lib.oea_matrix_topk_mean_workspace_bytes(n_rows, n_cols, k, 1)
    ws = torch.empty(max(16, nb), dtype=torch.uint8, device=dev)
    L.check(lib.oea_matrix_topk_mean(_ptr(t), ld, n_rows, n_cols, k, 1, _ptr(out), _ptr(ws), nb, None), "column means")
    _sync(dev)
    assert np.array_equal(host(out[:n_cols]), exact_means(s.T, k)), "column means"
    kcap = 4 if k <= 4 else 8 if k <= 8 else 10 if k <= 10 else 16 if k <= 16 else 32
    n_splits = nb // (kcap * ld * 4)
    return (n_rows + n_splits - 1) // n_splits


# ---- selection (raw ABI) -----------------------------------------------------------------------------------------
def select_ref(s, k):
    """The first k columns by (value descending, index ascending), listed in ascending column order."""
    return np.sort(order_desc(s)[:, :k], axis=1).astype(np.int32)


def check_select(dev, s, k, col_ids=None, ld_extra=0):
    """oea_rows_select_topk: exactly the reference set, in ascending column order; then oea_rows_gather_sort of it:
    the first k columns by (value descending, index ascending).  ld_extra % 4 != 0 takes the scalar loads."""
    lib = L.load()
    n_rows, n_cols = s.shape
    ld = (n_cols + 3) // 4 * 4 + ld_extra
    store = np.zeros((n_rows, ld), dtype=F32)
    store[:, :n_cols] = s
    t = torch.as_tensor(store, device=dev)
    out = torch.full((n_rows, k), -7, dtype=torch.int32, device=dev)
    ids = None if col_ids is None else torch.as_tensor(col_ids, dtype=torch.int32, device=dev)
    L.check(lib.oea_rows_select_topk(_ptr(t), ld, n_rows, n_cols, k, _ptr(ids), _ptr(out), None), "oea_rows_select_topk")
    _sync(dev)
    want = select_ref(s, k)
    if col_ids is not None:
        want = np.asarray(col_ids, dtype=np.int32)[want]
    got = host(out)
    assert np.array_equal(got, want), "selected set: %d rows differ" % int((got != want).any(1).sum())
    if col_ids is None and k <= 128:
        val = torch.empty(n_rows, k, dtype=torch.float32, device=dev)
        L.check(lib.oea_rows_gather_sort(_ptr(t), ld, n_rows, k, _ptr(out), _ptr(val), None), "oea_rows_gather_sort")
        _sync(dev)
        wv, wi = topk_ref(s, k)
        assert np.array_equal(host(out), wi), "gather-sorted lists"
        assert np.array_equal(host(val), wv), "gather-sorted values"


def selection_matrix(rng, n_rows, n_cols, k):
    """Rows whose tie classes straddle the k-th value: small integers (lots of ties), a constant row, a row of zeros with
    a block of maxima at the start and the end, negative values and ±FLT_MAX."""
    s = rng.integers(-3, 4, (n_rows, n_cols)).astype(F32)
    fmax = np.finfo(np.float32).max
    if n_rows > 0:
        s[0] = 0.0                                              # every column ties
    if n_rows > 1:
        s[1] = 0.0
        h = max(1, k // 2)
        s[1, :h] = 5.0
        s[1, n_cols - h:] = 5.0                                 # the k-th value is in a tie class at both ends
    if n_rows > 2:
        s[2] = -(rng.integers(1, 4, n_cols).astype(F32))        # all negative
    if n_rows > 3:
        s[3, ::3] = fmax
        s[3, 1::3] = -fmax
    if n_rows > 4:
        s[4] = -fmax
        s[4, n_cols // 2:] = fmax
    return s


# ---- normalisation (raw ABI) -------------------------------------------------------------------------------------
def normalize_rows_device(dev, x, in_pitch, out_pitch):
    lib = L.load()
    n, dim = x.shape
    src = np.full((n, in_pitch), 7.0, dtype=F32)               # columns past dim must not be read
    src[:, :dim] = x
    t = torch.as_tensor(src, device=dev)
    out = torch.full((n, out_pitch), 9.0, dtype=torch.float32, device=dev)
    L.check(lib.oea_rows_normalize(_ptr(t), in_pitch, n, dim, _ptr(out), out_pitch, None), "oea_rows_normalize")
    _sync(dev)
    o = host(out)
    assert not o[:, dim:].any(), "padding up to out_pitch must be zero"
    return o[:, :dim]


def normalize_inputs(rng, dim):
    """Random rows and the degenerate ones: zero, 1e-23 (the squared norm underflows), 1e-7 (norm below 10·eps: kept as
    it is), 1e-5 (normalised); each at least 2x away from the 10·eps boundary."""
    x = rng.standard_normal((9, dim)).astype(F32)
    x[0] = 0
    x[1] = 0
    x[1, 0] = 1e-23
    x[2] = 1e-23
    x[3] = 0
    x[3, -1] = 1e-7
    x[4] = 1e-7 / np.sqrt(dim)
    x[5] = 0
    x[5, 0] = -1e-5
    x[6] = 1e-5
    return x


def _col_means(a, b, k, block=4096):
    """float64 column top-k means of a @ b.T and their bound, over every row, in row blocks."""
    top = dmax = None
    for r0 in range(0, a.shape[0], block):
        s, dl = bound_matrix(a[r0:r0 + block], b, "inner", a.shape[1])
        top = torch.topk(s if top is None else torch.cat([top, s]), k, dim=0).values
        m = dl.max(0).values
        dmax = m if dmax is None else torch.maximum(dmax, m)
    c = top.mean(0)
    return c, dmax + gamma(k - 1) * (top.abs().mean(0) + dmax) + U * c.abs()


def check_waves(F, n, d, csls_k, materialize, seed, n_sample=700):
    """eval_alignment of n × n inner-product rows (near-duplicates plus 64 exact duplicates, a permuted gold): the
    first and last row blocks, the duplicates and `n_sample` random rows are checked by the interval rule against
    float64 computed on the engine's device.  Returns (row blocks, effective column splits) of the launch."""
    rng = np.random.default_rng(seed)
    e2 = rng.standard_normal((n, d)).astype(F32)
    e1 = (e2 + 0.8 * rng.standard_normal((n, d))).astype(F32)
    e1[n // 2:n // 2 + 64] = e2[:64]                            # exact duplicates: ties at the top
    gold = rng.permutation(n).astype(np.int32)
    t1, t2 = dev_rows(F, e1), dev_rows(F, e2)
    _, eff, _ = splits_of(F, t1, t2, d)
    top1, rk, *_ = F.eval_alignment(e1, e2, [1], "inner", False, csls_k, gold=gold, materialize=materialize)
    top1, rk = host(top1), host(rk)
    sample = np.unique(np.concatenate([np.arange(min(n, TILE)), np.arange(max(0, n - TILE), n),
                                       np.arange(n // 2, min(n, n // 2 + 64)), rng.choice(n, min(n, n_sample), replace=False)]))
    a = torch.as_tensor(e1, dtype=torch.float64, device=t1.device)
    b = torch.as_tensor(e2, dtype=torch.float64, device=t1.device)
    if csls_k:
        c64, dc = _col_means(a, b, csls_k)
    for lo in range(0, len(sample), 256):
        idx = sample[lo:lo + 256]
        s, dl = bound_matrix(a[torch.as_tensor(idx, device=a.device)], b, "inner", d)
        if csls_k:
            r64, dr = bound_means(s, dl, csls_k)
            s, dl = bound_csls(s, dl, r64, dr, c64, dc)
        check_rank_interval(top1[idx], rk[idx], s, dl, gold[idx], "rows from %d" % idx[0])
    return (n + TILE - 1) // TILE, eff


def _sync(dev):
    if str(dev).startswith("cuda"):
        torch.cuda.synchronize()
