"""The sampled-NCE head, ProjE's batch norms and the device samplers of openea_b200/csrc/oea_proje.cu at their edges,
called through the raw C-ABI (oea_nce_score_fed, oea_proje_score_fed, oea_logu_sample_unique, oea_pairs_draw) against
float64 references.  tests/test_emu_nce_edges.py runs these cases on the warp emulator, tests/test_zz_nce_edges_gpu.py
on the GPU.

Edge-dominated data.  The class-table rows of the sampled set are zero except at the *edge slots* 0, S − 1 and every
16·j − 1 and 16·j below S: every split boundary head_grids can produce is a multiple of kTk = 16, so these slots sit on
both sides of every split boundary on any SM count, and of every 128-column tile edge.  Input rows are zero except at
the same positions of the batch, and labels come from the edge classes and a few classes outside the sampled set.  Every
gradient element is then a short sum of known terms, and is checked against its own bound c·γ_k·Σ|terms| (k from the
kernel's summation structure: the longest chain inside one split plus the number of splits) plus the propagated error of
the logits, G, the expected counts and __expf — never against a tolerance scaled by the largest element of the array.

Every call runs in a workspace of exactly oea_*_workspace_bytes bytes inside a larger buffer of 0xFF bytes (NaN as
fp32): a read of a workspace element the step did not write shows up as NaN, and the bytes past the end must still be
0xFF afterwards.  Each case also proves it can fail: the reference recomputed with one edge class, one edge row or one
row's true-class term left out must differ from the full one by more than 10× the allowed error at some element.
"""
import ctypes as C
import math

import numpy as np
import torch

from openea_b200 import engine as eng
from openea_b200 import lib as L
from oracle.triple_ext import l2n
from tests import proje_oracle as po

F32 = np.float32
U = 2.0 ** -24                                   # unit round-off of fp32
FLT_MIN = float(np.finfo(np.float32).tiny)       # what an underflowing exponential can lose
NORM_EPS = 1e-12
KTK, KTILE = 16, 128
CANARY = 256
BOUND_C = 2.0                                    # slack on every first-order bound
RAW = {"in": False, "w": False}
NORMED = {"in": True, "w": True}


def gamma(k):
    if not torch.is_tensor(k):
        k = np.asarray(k, dtype=np.float64)
    return k * U / (1 - k * U)


def cdiv(a, b):
    return -(-a // b)


def expf_ulps(x):
    """CUDA's __expf: at most 2 + floor(1.173·|x|) ulp (CUDA C Programming Guide, intrinsic functions); glibc's expf on
    the emulator is within 1 ulp, so the device's figure bounds both."""
    return 2 + torch.floor(1.173 * x.abs())


def edge_positions(m):
    """0, m − 1 and every 16·j − 1 and 16·j below m."""
    e = {0, m - 1}
    for j in range(KTK, m, KTK):
        e.update((j - 1, j))
    return np.array(sorted(e), dtype=np.int64)


def head_splits(n, S, sms):
    """(split of the sampled set for dX, split of the batch for dW) as head_grids computes them: about two CTAs per SM,
    each split a multiple of kTk.  sms None: the emulator's fixed 2·kTk."""
    if sms is None:
        return 2 * KTK, 2 * KTK
    mt_b, mt_s, want = cdiv(n, KTILE), cdiv(S, KTILE), 2 * sms
    split_of = lambda length, parts: cdiv(cdiv(length, parts), KTK) * KTK
    return split_of(S, cdiv(want, mt_b)), split_of(n, cdiv(want, mt_s))


def split_kind(length, split):
    """'one' (the whole reduction is one split), 'ragged' (several splits, the last one shorter) or 'even'."""
    if length <= split:
        return "one"
    return "ragged" if length % split else "even"


def loss_depth(n, S, sms):
    """Longest fp32 chain of loss terms one thread sums: the logits kernel's 64 outputs per tile over the tiles one CTA
    takes, and the rows a warp of the true-class kernel takes, each plus the warp and block reductions."""
    tiles = cdiv(n, KTILE) * cdiv(cdiv(S, 4) * 4, KTILE)
    lg = tiles if sms else 2
    rows = min(max(cdiv(n, 8), 1), 8 * sms) if sms else 2
    return 64 * cdiv(tiles, lg) + 8, cdiv(n, 8 * rows) + 8


def _split_depth(nonzero, split):
    """Longest chain in a split-then-atomic reduction over `nonzero` terms: the most non-zero terms inside one split
    plus the number of splits (adding an exact zero rounds nothing)."""
    nz = np.asarray(nonzero, dtype=np.int64)
    windows = [int(nz[s:s + split].sum()) for s in range(0, len(nz), split)]
    return max(windows) + len(windows)


# ---- device buffers ------------------------------------------------------------------------------------------------
class DevTable:
    """An oea_table over torch tensors on `dev` (the emulator's device pointers are host pointers)."""

    def __init__(self, values, norm, dev):
        values = np.asarray(values, dtype=F32)
        self.rows, self.d = values.shape
        self.pitch = (self.d + 3) // 4 * 4
        w = np.zeros((self.rows, self.pitch), dtype=F32)
        w[:, :self.d] = values
        self.weight = torch.from_numpy(w).to(dev)
        self.grad = torch.zeros_like(self.weight)
        self.s1, self.s2 = torch.zeros_like(self.weight), torch.zeros_like(self.weight)
        self.touched = torch.zeros(self.rows, dtype=torch.int32, device=dev)
        self.struct = L.Table(self.weight.data_ptr(), self.grad.data_ptr(), self.s1.data_ptr(), self.s2.data_ptr(),
                              self.touched.data_ptr(), self.rows, self.d, self.pitch, int(norm))

    def got(self):
        return self.grad[:, :self.d].double().cpu().numpy()


def _ints(a, dev):
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.int32), device=dev)


def _sync(dev):
    if dev.type == "cuda":
        torch.cuda.synchronize(dev)


def poisoned_workspace(need, dev):
    """`need` bytes of 0xFF followed by CANARY more; the call is given exactly `need`."""
    buf = torch.full((need + CANARY,), 0xFF, dtype=torch.uint8, device=dev)
    assert buf.data_ptr() % 16 == 0
    return buf


def check_canary(buf, need):
    assert bool((buf[need:] == 0xFF).all()), "bytes past the workspace were written"


def run_nce(dev, tables, inputs, labels, sampled, num_tries, scale):
    lib = L.load()
    n, S = len(inputs), len(sampled)
    need = lib.oea_nce_workspace_bytes(n, S, tables["in"].d, tables["w"].rows)
    ws = poisoned_workspace(need, dev)
    ii, ll, smp, nt = _ints(inputs, dev), _ints(labels, dev), _ints(sampled, dev), _ints([num_tries], dev)
    out = torch.zeros(1, dtype=torch.float64, device=dev)
    m = L.Nce(*[C.pointer(tables[k].struct) for k in ("in", "w", "b")])
    rc = lib.oea_nce_score_fed(C.byref(m), eng._ptr(ii), eng._ptr(ll), n, eng._ptr(smp), eng._ptr(nt), S, scale,
                               eng._ptr(ws), need, eng._ptr(out), eng._stream_ptr())
    _sync(dev)
    assert rc == 0, rc
    check_canary(ws, need)
    return float(out.cpu()[0])


def run_proje(dev, tables, pos, sampled, num_tries):
    lib = L.load()
    n, S = pos.shape[1], len(sampled)
    need = lib.oea_proje_workspace_bytes(n, S, tables["ent"].d, tables["w"].rows)
    ws = poisoned_workspace(need, dev)
    p = [_ints(pos[i], dev) for i in range(3)]
    smp, nt = _ints(sampled, dev), _ints([num_tries], dev)
    out = torch.zeros(1, dtype=torch.float64, device=dev)
    m = L.Proje(*[C.pointer(tables[k].struct) for k in PROJE_NAMES])
    rc = lib.oea_proje_score_fed(C.byref(m), eng._ptr(p[0]), eng._ptr(p[1]), eng._ptr(p[2]), n, eng._ptr(smp),
                                 eng._ptr(nt), S, eng._ptr(ws), need, eng._ptr(out), eng._stream_ptr())
    _sync(dev)
    assert rc == 0, rc
    check_canary(ws, need)
    return float(out.cpu()[0])


# ---- the general sampled-NCE step: cases -----------------------------------------------------------------------------
# (name, d, S, n, extra).  Every width, S % 4 != 0 and S % 16 != 0, S = every class, n = 1 and the row-tile edges; the
# split extremes (n or S past (2·SM − 1)·128) are added by the GPU file from the device's SM count.
NCE_GPU_CASES = [
    ("d1-S1-n1", 1, 1, 1, {}),
    ("d3-S2-n2", 3, 2, 2, {"scale": 1.0}),
    ("d4-S3-n127", 4, 3, 127, {"scale": 0.37}),
    ("d5-S5-n128-every-class", 5, 5, 128, {"C": 5}),
    ("d15-S15-n129", 15, 15, 129, {"scale": 1.0}),
    ("d16-S16-n257", 16, 16, 257, {}),
    ("d17-S17-n5000", 17, 17, 5000, {"scale": 0.37}),
    ("d33-S127-n129", 33, 127, 129, {}),
    ("d64-S128-n257", 64, 128, 257, {"scale": 1.0}),
    ("d100-S129-n5000", 100, 129, 5000, {}),
    ("d127-S129-n128-every-class", 127, 129, 128, {"C": 129, "scale": 0.37}),
    ("d128-S4095-n129", 128, 4095, 129, {}),
    ("d128-S4097-n5000-every-class", 128, 4097, 5000, {"C": 4097}),
    ("d100-S4097-n257", 100, 4097, 257, {"scale": 1.0}),
    ("same-label-sampled", 17, 129, 257, {"kind": "same_label"}),
    ("same-input", 16, 129, 257, {"kind": "same_input"}),
    ("all-labels-sampled", 33, 127, 257, {"kind": "hits"}),
    ("input-is-own-label", 17, 17, 129, {"kind": "self_label"}),
    ("saturated-logits", 4, 17, 129, {"kind": "saturate", "raw_only": True}),
    ("expected-count-shortcut", 16, 129, 129, {"kind": "shortcut"}),
    ("E200000-last-class", 100, 4097, 257, {"kind": "last_class", "C": 200000}),
]

# the same kinds of case at the emulator's sizes (its splits are 32 long)
NCE_EMU_CASES = [
    ("d1-S1-n1", 1, 1, 1, {}),
    ("d3-S2-n2", 3, 2, 2, {"scale": 1.0}),
    ("d4-S3-n33", 4, 3, 33, {"scale": 0.37}),
    ("d5-S5-n17-every-class", 5, 5, 17, {"C": 5}),
    ("d15-S15-n65", 15, 15, 65, {"scale": 1.0}),
    ("d16-S16-n33", 16, 16, 33, {}),
    ("d17-S17-n31", 17, 17, 31, {}),
    ("d33-S33-n17", 33, 33, 17, {"scale": 0.37}),
    ("d64-S37-n34", 64, 37, 34, {}),
    ("d100-S65-n9", 100, 65, 9, {}),
    ("d127-S70-n7-every-class", 127, 70, 7, {"C": 70}),
    ("d128-S129-n3", 128, 129, 3, {"scale": 1.0}),
    ("d8-S130-n130", 8, 130, 130, {}),
    ("same-label-sampled", 17, 37, 40, {"kind": "same_label"}),
    ("same-input", 16, 37, 40, {"kind": "same_input"}),
    ("all-labels-sampled", 12, 35, 40, {"kind": "hits"}),
    ("input-is-own-label", 17, 17, 33, {"kind": "self_label"}),
    ("saturated-logits", 4, 17, 33, {"kind": "saturate", "raw_only": True}),
    ("expected-count-shortcut", 16, 33, 20, {"kind": "shortcut"}),
    ("E200000-last-class", 20, 35, 17, {"kind": "last_class", "C": 200000}),
]


def nce_case(d, S, n, extra, seed):
    """→ (tabs, inputs, labels, sampled, num_tries, scale) of edge-dominated raw values."""
    rng = np.random.default_rng(seed)
    kind = extra.get("kind")
    A = n + 8
    Cn = extra.get("C") or S + 40
    if kind == "self_label":
        Cn = max(Cn, A)
    amp = 10.0 if kind == "saturate" else 1.0
    sampled = rng.choice(Cn, S, replace=False).astype(np.int64)
    if kind == "last_class":
        hit = np.flatnonzero(sampled == Cn - 1)
        sampled[hit if len(hit) else [S - 1]] = sampled[S - 1]
        sampled[S - 1] = Cn - 1
    es, er = edge_positions(S), edge_positions(n)
    outside = np.setdiff1d(rng.choice(Cn, min(Cn, 64), replace=False), sampled)[:8]
    pool = np.concatenate([sampled[es], outside])
    labels = rng.choice(pool, n)
    inputs = rng.permutation(A)[:n]
    if kind == "same_label":
        labels[:] = sampled[S - 1]
    elif kind == "same_input":
        inputs[:] = inputs[0]
    elif kind == "hits":
        labels = rng.choice(sampled[es], n)
    elif kind == "self_label":
        labels[er] = inputs[er]

    def values(rows):
        """|v| in [0.5, 1]·amp on about 4·d / rows columns of each row (at least 2): every column is live in a few
        rows, and every gradient element stays a short sum however many edge rows there are."""
        k = min(d, max(2, cdiv(4 * d, max(rows, 1))))
        cols = rng.random((rows, d)).argsort(1)[:, :k]
        v = np.zeros((rows, d))
        np.put_along_axis(v, cols, rng.uniform(0.5, 1.0, (rows, k)) * rng.choice([-1.0, 1.0], (rows, k)) * amp, 1)
        return v

    x = np.zeros((A, d))
    x[inputs[er]] = values(len(er))
    w = np.zeros((Cn, d))
    live = np.union1d(sampled[es], labels)
    w[live] = values(len(live))
    b = rng.uniform(-1.0, 1.0, (Cn, 1))
    if kind == "shortcut":
        tries = S
    elif kind == "last_class":
        tries = 1000 * S
    else:
        tries = S + 1 + int(rng.integers(0, 2 * S + 8))
    scale = extra.get("scale", 1.0 / n)
    tabs = {"in": x.astype(F32), "w": w.astype(F32), "b": b.astype(F32)}
    return tabs, inputs, labels, sampled, tries, scale


# ---- the general sampled-NCE step: float64 reference and bounds ------------------------------------------------------
def _t(a, dev):
    return torch.as_tensor(np.asarray(a, dtype=np.float64), device=dev)


def _long(a, dev):
    return torch.as_tensor(np.asarray(a, dtype=np.int64), device=dev)


def _softplus(x):
    return torch.clamp(x, min=0) + torch.log1p(torch.exp(-x.abs()))


def _normed(M, on):
    ss = (M * M).sum(1)
    inv = torch.rsqrt(torch.clamp(ss, min=NORM_EPS)) if on else torch.ones_like(ss)
    return M * inv[:, None], inv, ((ss >= NORM_EPS) & on).double()


def _jac(g, xh, inv, proj):
    """The gradient w.r.t. a raw row from the gradient w.r.t. its l2-normalised lookup (rows of g)."""
    return (g - xh * ((xh * g).sum(1) * proj)[:, None]) * inv[:, None]


def _jac_abs(a, axh, inv, proj):
    return (a + axh * ((axh * a).sum(1) * proj)[:, None]) * inv[:, None]


def nce_reference(tabs, norms, inputs, labels, sampled, num_tries, scale, dev, sms=None, drop=None):
    """loss_scale · Σ_b nce_loss in closed form, float64 on `dev`, with the expected counts in fp32 as TF computes them
    (the maths of tests/attr2vec_oracle.py, checked against it in tests/test_emu_nce_edges.py).  drop: None or
    ("class", slot) / ("row", b) / ("true", b), the term left out.  Returns {"loss", "in", "w", "b", "err"}: the
    gradients as float64 arrays in the tables' shapes and, in "err", each output's first-order fp32 error bound (before
    BOUND_C): the rounding of its own sum, c·γ_k·Σ|terms|, plus the propagated error of the logits (γ_{pitch+3} of their
    terms, 16u of the fp32 log expected count), of G and g = σ(t) − 1 (σ' times the logit error, 8u of the value, and
    FLT_MIN where the exponential underflows), and of the normalisation's Jacobian."""
    Xt, xinv, xproj = _normed(_t(tabs["in"], dev), norms["in"])
    Wt, winv, wproj = _normed(_t(tabs["w"], dev), norms["w"])
    bias = _t(tabs["b"], dev).reshape(-1)
    A_rows, d = Xt.shape
    Cn, n, S = Wt.shape[0], len(inputs), len(sampled)
    P = (d + 3) // 4 * 4
    inp, lab, smp = _long(inputs, dev), _long(labels, dev), _long(sampled, dev)
    lq = lambda ids: torch.log(_t(po.expected_count(np.asarray(ids), Cn, S, num_tries), dev))
    lqs, lqt = lq(sampled), lq(labels)
    X, Ws, Wl = Xt[inp], Wt[smp], Wt[lab]
    ls = X @ Ws.T + bias[smp] - lqs
    lt = (X * Wl).sum(1) + bias[lab] - lqt
    ms, mt = torch.ones_like(ls), torch.ones_like(lt)
    if drop is not None:
        what, j = drop
        if what == "class":
            ms[:, j] = 0
        elif what == "row":
            ms[j] = 0
            mt[j] = 0
        else:
            mt[j] = 0
    sig_s, sig_nt = torch.sigmoid(ls), torch.sigmoid(-lt)
    G = scale * sig_s * ms
    gt = -scale * sig_nt * mt
    sp_s, sp_t = _softplus(ls), _softplus(-lt)
    loss = scale * ((sp_s * ms).sum() + (sp_t * mt).sum())
    dX = G @ Ws + gt[:, None] * Wl
    dWs, dWt = G.T @ X, gt[:, None] * X
    zeros = lambda rows, cols: torch.zeros(rows, cols, dtype=torch.float64, device=dev)
    g_in = zeros(A_rows, d).index_add_(0, inp, _jac(dX, X, xinv[inp], xproj[inp]))
    g_w = zeros(Cn, d).index_add_(0, smp, _jac(dWs, Ws, winv[smp], wproj[smp]))
    g_w.index_add_(0, lab, _jac(dWt, Wl, winv[lab], wproj[lab]))
    g_b = zeros(Cn, 1).index_add_(0, smp, G.sum(0)[:, None]).index_add_(0, lab, gt[:, None])
    out = {"loss": float(loss), "in": g_in.cpu().numpy(), "w": g_w.cpu().numpy(), "b": g_b.cpu().numpy()}

    # bounds
    extra = 2 * P + 16 if (norms["in"] or norms["w"]) else 0          # relative error of the normalised operands
    a = abs(scale)
    dlq = lambda v: 16 * U * (1 + v.abs())
    k_dot = float(gamma(P + 3 + extra))
    aX, aWs, aWl = X.abs(), Ws.abs(), Wl.abs()
    dls = k_dot * (aX @ aWs.T + bias[smp].abs() + lqs.abs()) + dlq(lqs)
    dlt = k_dot * ((aX * aWl).sum(1) + bias[lab].abs() + lqt.abs()) + dlq(lqt)
    dG = a * (sig_s * (1 - sig_s) * dls + 8 * U * sig_s + FLT_MIN) * ms
    dgt = a * (sig_nt * (1 - sig_nt) * dlt + 8 * U * sig_nt + FLT_MIN) * mt
    aG, agt = G.abs(), gt.abs()
    split_s, split_b = head_splits(n, S, sms)
    k_x = _split_depth((aWs.sum(1) > 0).cpu().numpy(), split_s) + 3 + extra
    k_w = _split_depth((aX.sum(1) > 0).cpu().numpy(), split_b) + 3 + extra
    A_dX = aG @ aWs + agt[:, None] * aWl
    E_dX = dG @ aWs + dgt[:, None] * aWl + float(gamma(k_x)) * A_dX
    A_dWs = aG.T @ aX
    E_dWs = dG.T @ aX + float(gamma(k_w)) * A_dWs
    A_dWt = agt[:, None] * aX
    E_dWt = dgt[:, None] * aX + U * A_dWt

    def pushed(Agrad, Egrad, xh, inv, proj, on):
        if not on:                                   # through_norm with the normalisation off is exact
            return Agrad, Egrad
        Ar = _jac_abs(Agrad, xh.abs(), inv, proj)
        return Ar, _jac_abs(Egrad, xh.abs(), inv, proj) + float(gamma(P + 8 + extra)) * Ar

    def count(ids, rows):
        return torch.bincount(ids, minlength=rows).double()

    Ai, Ei = pushed(A_dX, E_dX, X, xinv[inp], xproj[inp], norms["in"])
    A_in, E_in = zeros(A_rows, d).index_add_(0, inp, Ai), zeros(A_rows, d).index_add_(0, inp, Ei)
    E_in += gamma(count(inp, A_rows))[:, None] * A_in
    As, Es = pushed(A_dWs, E_dWs, Ws, winv[smp], wproj[smp], norms["w"])
    At, Et = pushed(A_dWt, E_dWt, Wl, winv[lab], wproj[lab], norms["w"])
    A_w = zeros(Cn, d).index_add_(0, smp, As).index_add_(0, lab, At)
    E_w = zeros(Cn, d).index_add_(0, smp, Es).index_add_(0, lab, Et)
    E_w += gamma(count(smp, Cn) + count(lab, Cn))[:, None] * A_w
    A_b = zeros(Cn, 1).index_add_(0, smp, aG.sum(0)[:, None]).index_add_(0, lab, agt[:, None])
    E_b = zeros(Cn, 1).index_add_(0, smp, dG.sum(0)[:, None]).index_add_(0, lab, dgt[:, None])
    E_b += gamma(n + count(lab, Cn) + 2)[:, None] * A_b
    m_s, m_t = loss_depth(n, S, sms)
    e_sp = lambda sig, dl, sp, l: sig * dl + 4 * U * sp + 2 * U * expf_ulps(l) * torch.exp(-l.abs()) + FLT_MIN
    E_loss = a * ((e_sp(sig_s, dls, sp_s, ls) * ms).sum() + (e_sp(sig_nt, dlt, sp_t, lt) * mt).sum()
                  + float(gamma(m_s)) * (sp_s * ms).sum() + float(gamma(m_t)) * (sp_t * mt).sum()) + 2 * U * abs(loss)
    out["err"] = {"in": E_in.cpu().numpy(), "w": E_w.cpu().numpy(), "b": E_b.cpu().numpy(), "loss": float(E_loss)}
    return out


def _worst(err, bound):
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err > 0, err / bound, 0.0)
    return r


def check_within(name, got, want, bound):
    err = np.abs(got - want)
    ok = err <= bound
    if not ok.all():
        r = _worst(err, bound)
        at = np.unravel_index(np.argmax(r), r.shape)
        raise AssertionError("%s: %d elements outside the bound, worst err/bound %.3g at %s (got %r, want %r)" % (
            name, int((~ok).sum()), float(r[at]), at, got[at], want[at]))


def check_touched(tab, ids, what):
    want = np.zeros(tab.rows, dtype=bool)
    want[np.asarray(ids, dtype=np.int64)] = True
    got = tab.touched.cpu().numpy() != 0
    assert np.array_equal(got, want), "%s: touched on %s, referenced %s" % (
        what, np.flatnonzero(got & ~want)[:8], np.flatnonzero(want & ~got)[:8])


def check_padding(tab, what):
    assert not bool(tab.grad[:, tab.d:].any()), what + ": padding columns of grad were written"


def self_check(full, dropped, keys, allowed, what):
    """One term left out of the reference must move some element of `keys` by more than 10× the allowed error."""
    worst = 0.0
    for k in keys:
        diff = np.abs(np.asarray(full[k], dtype=np.float64) - np.asarray(dropped[k], dtype=np.float64))
        worst = max(worst, float(np.max(_worst(diff, allowed[k]), initial=0.0)))
    assert worst > 10, "%s: the check cannot see it (largest change / allowed error %.3g)" % (what, worst)


def case_nce(dev, d, S, n, extra, norms, sms=None, seed=0):
    """One oea_nce_score_fed call on edge-dominated data against the float64 reference, element by element."""
    tabs, inputs, labels, sampled, tries, scale = nce_case(d, S, n, extra, seed)
    tables = {k: DevTable(v, norms.get(k, False), dev) for k, v in tabs.items()}
    got_loss = run_nce(dev, tables, inputs, labels, sampled, tries, scale)
    ref = nce_reference(tabs, norms, inputs, labels, sampled, tries, scale, dev, sms)
    allowed = {k: BOUND_C * ref["err"][k] for k in ("in", "w", "b")}
    if extra.get("kind") == "saturate":
        assert np.abs(nce_logits(tabs, inputs, sampled, labels)).max() > 90, "the case does not saturate"
    for k, tab in tables.items():
        got = tab.got()
        assert np.isfinite(got).all(), k + ": non-finite gradient (a poisoned workspace element was read?)"
        check_within(k, got, ref[k], allowed[k])
        check_padding(tab, k)
    assert math.isfinite(got_loss)
    assert abs(got_loss - ref["loss"]) <= BOUND_C * ref["err"]["loss"], (got_loss, ref["loss"], ref["err"]["loss"])
    check_touched(tables["in"], inputs, "in")
    check_touched(tables["w"], np.union1d(labels, sampled), "w")
    check_touched(tables["b"], np.union1d(labels, sampled), "b")
    args = (tabs, norms, inputs, labels, sampled, tries, scale, dev, sms)
    er = edge_positions(n)
    keys = ("in", "w", "b")
    self_check(ref, nce_reference(*args, drop=("class", S - 1)), keys, allowed, "edge class S − 1 left out")
    self_check(ref, nce_reference(*args, drop=("row", int(er[-1]))), keys, allowed, "edge row n − 1 left out")
    self_check(ref, nce_reference(*args, drop=("true", 0)), keys, allowed, "row 0's true class left out")
    return ref


def nce_logits(tabs, inputs, sampled, labels):
    X = tabs["in"].astype(np.float64)[inputs]
    W = tabs["w"].astype(np.float64)
    return np.concatenate([(X @ W[sampled].T).ravel(), (X * W[labels]).sum(1)])


def split_extreme_cases(sms):
    """n past (2·SM − 1)·128 rows: the whole sampled set is one dX split; S past it with n = 129: the whole batch is
    one dW split."""
    edge = (2 * sms - 1) * KTILE + 1
    return [("rows-past-2SM-tiles", 16, 17, edge, {}), ("classes-past-2SM-tiles", 64, edge, 129, {"C": edge + 40})]


# ---- ProjE -----------------------------------------------------------------------------------------------------------
PROJE_NAMES = ("ent", "rel", "w", "b", "params")
PROJE_NORMS = {"ent": True, "rel": True}
PROJE_RTOL = 2e-4

# (name, d, n, S, extra); S = "every" samples every class.  n past (2·SM − 1)·128 is added by the GPU file.
PROJE_GPU_CASES = [
    ("d1-n1-S1", 1, 1, 1, {}),
    ("d4-n2-S17", 4, 2, 17, {}),
    ("d17-n129-S129", 17, 129, 129, {}),
    ("d64-n5000-S17", 64, 5000, 17, {}),
    ("d127-n129-S-every", 127, 129, "every", {}),
    ("d128-n5000-S129", 128, 5000, 129, {}),
    ("d128-n1-S-every", 128, 1, "every", {}),
    ("zero-mlp-w-column", 17, 129, 17, {"kind": "zero_w_col"}),
    ("same-head-and-relation", 16, 257, 17, {"kind": "same_hr"}),
]
PROJE_EMU_CASES = [
    ("d1-n1-S1", 1, 1, 1, {}),
    ("d4-n2-S17", 4, 2, 17, {}),
    ("d17-n33-S33", 17, 33, 33, {}),
    ("d64-n40-S17", 64, 40, 17, {}),
    ("d127-n9-S-every", 127, 9, "every", {}),
    ("d128-n3-S35", 128, 3, 35, {}),
    ("zero-mlp-w-column", 17, 33, 17, {"kind": "zero_w_col"}),
    ("same-head-and-relation", 16, 40, 17, {"kind": "same_hr"}),
]


def proje_case(d, n, S, extra, seed):
    rng = np.random.default_rng(seed)
    kind = extra.get("kind")
    E = 48 if S == "every" else S + 40
    S = E if S == "every" else S
    n_rel = 7
    sampled = rng.choice(E, S, replace=False).astype(np.int64)
    es = edge_positions(S)
    outside = np.setdiff1d(np.arange(E), sampled)[:8]
    tails = rng.choice(np.concatenate([sampled[es], outside]), n)
    heads, rels = rng.integers(0, E - 1, n), rng.integers(0, n_rel, n)
    heads[-1] = E - 1                   # the last positive's head is its own: leaving it out empties that ent row
    if kind == "same_hr":
        heads[:], rels[:] = heads[0], rels[0]
    w = np.zeros((E, d))
    live = np.union1d(sampled[es], tails)
    w[live] = rng.uniform(0.5, 1.0, (len(live), d)) * rng.choice([-1.0, 1.0], (len(live), d)) / math.sqrt(d)
    lim = math.sqrt(3.0 / d)
    params = np.stack([rng.uniform(-lim, lim, d), rng.uniform(-lim, lim, d), rng.standard_normal(d) * 0.1,
                       rng.standard_normal(d) * 0.1])
    if kind == "zero_w_col":
        params[0, d // 2] = 0.0
    tabs = {"ent": rng.standard_normal((E, d)) / math.sqrt(d), "rel": rng.standard_normal((n_rel, d)) / math.sqrt(d),
            "w": w, "b": rng.uniform(-1.0, 1.0, (E, 1)), "params": params}
    tries = S + 2 + int(rng.integers(0, 2 * S + 8))   # never S or S − 1: leaving a class out keeps every q(c)
    pos = np.stack([heads, rels, tails]).astype(np.int64)
    # exact zeros and cancellations hold for the gradient of the lookups; the normalisation's Jacobian mixes columns
    norms = {"ent": False, "rel": False} if kind in ("zero_w_col", "same_hr") else PROJE_NORMS
    return {k: v.astype(F32) for k, v in tabs.items()}, pos, sampled, tries, kind, norms


def _proje_dz_abs(tabs, norms, pos, sampled, tries, dev):
    """Σ_b of the magnitudes of the terms of dz (the output batch norm's input gradient) per column, in float64: what
    the gradients of mlp_bias and the input beta, zero in exact arithmetic, may round to."""
    t = {k: _t(v, dev) for k, v in tabs.items()}
    h, r, tl = (_long(x, dev) for x in pos)
    E, P_ = t["w"].shape[0], t["params"]
    nrm = lambda k: l2n(t[k]) if norms[k] else t[k]
    xh, xr = nrm("ent")[h], nrm("rel")[r]
    bn = lambda x: ((x - x.mean(0)) / torch.sqrt(x.var(0, unbiased=False) + po.BN_EPS))
    z = (bn(xh) + P_[2]) * P_[0] + (bn(xr) + P_[2]) * P_[0] + P_[1]
    mz, rz = z.mean(0), 1 / torch.sqrt(z.var(0, unbiased=False) + po.BN_EPS)
    zh = (z - mz) * rz
    X = zh + P_[3]
    s = _long(sampled, dev)
    lq = lambda ids: torch.log(_t(po.expected_count(np.asarray(ids), E, len(sampled), tries), dev))
    b = t["b"].reshape(-1)
    G = torch.sigmoid(X @ t["w"][s].T + b[s] - lq(sampled))
    gt = -torch.sigmoid(-((X * t["w"][tl]).sum(1) + b[tl] - lq(pos[2])))
    dX = G @ t["w"][s] + gt[:, None] * t["w"][tl]
    m1, m2 = dX.mean(0), (dX * zh).mean(0)
    return (rz * (dX.abs() + m1.abs() + (z.abs() + mz.abs()) * rz * m2.abs())).sum(0).cpu().numpy()


def _row_allowed(want):
    """PROJE_RTOL of the largest element of each table row: the batch norms mix the whole batch into every element."""
    return PROJE_RTOL * np.abs(want).max(axis=1, keepdims=True) * np.ones_like(want)


def case_proje(dev, d, n, S, extra, sms=None, seed=0):
    tabs, pos, sampled, tries, kind, norms = proje_case(d, n, S, extra, seed)
    tables = {k: DevTable(v, norms.get(k, False), dev) for k, v in tabs.items()}
    got_loss = run_proje(dev, tables, pos, sampled, tries)
    want_loss, want = po.fwd_bwd(tabs, norms, pos, sampled, tries, device=dev)
    want = {k: v.reshape(tables[k].rows, -1) for k, v in want.items()}
    n = pos.shape[1]
    allowed = {k: _row_allowed(v) for k, v in want.items()}
    # mlp_bias and the input beta: the output batch norm's gradient sums to zero over the batch
    P = (d + 3) // 4 * 4
    dz_abs = _proje_dz_abs(tabs, norms, pos, sampled, tries, dev)
    canc = 16 * gamma(cdiv(n, 256) + P + 24) * dz_abs
    prm = tabs["params"].astype(np.float64)
    allowed["params"][1] = canc
    allowed["params"][2] = canc * 2 * np.abs(prm[0])
    got = {k: t.got() for k, t in tables.items()}
    if kind == "same_hr":
        for k, idx in (("ent", pos[0, 0]), ("rel", pos[1, 0])):
            allowed[k][idx] = shared_row_bound(tabs, norms, pos, sampled, tries, dev, k)
        # mlp_w's gradient Σ_b dz·(x̂_h + x̂_r + 2β) is a cancellation too: Σ_b dz = 0, and x̂ = (x − mean)·rstd is
        # fp32's rounding of the mean times rstd = 1/√ε where float64 has 0
        x_abs = np.abs(tabs["ent"][pos[0, 0]].astype(np.float64)) + np.abs(tabs["rel"][pos[1, 0]].astype(np.float64))
        allowed["params"][0] = canc * (2 * np.abs(prm[2]) + 2 + x_abs / math.sqrt(po.BN_EPS))
    for k in PROJE_NAMES:
        assert np.isfinite(got[k]).all(), k
        check_within(k, got[k], want[k], allowed[k])
        check_padding(tables[k], k)
    if n == 1:                 # every term of the batch norms' backward cancels exactly
        assert not got["ent"].any() and not got["rel"].any(), "n = 1: ent / rel gradients must be exactly 0"
    if kind == "zero_w_col":
        c = d // 2
        assert not got["ent"][:, c].any() and not got["rel"][:, c].any(), "zero mlp_w column: gradients must be 0"
    assert abs(got_loss - want_loss) <= 2e-5 * abs(want_loss), (got_loss, want_loss)
    check_touched(tables["ent"], pos[0], "ent")
    check_touched(tables["rel"], pos[1], "rel")
    check_touched(tables["w"], np.union1d(pos[2], sampled), "w")
    check_touched(tables["b"], np.union1d(pos[2], sampled), "b")
    check_touched(tables["params"], np.arange(4), "params")
    # self-checks: one edge class, one positive, one true-class term
    S_ = len(sampled)
    keys = ("ent", "rel", "w", "b") if n > 1 else ("w", "b")
    if S_ > 1:
        _, drop = po.fwd_bwd(tabs, norms, pos, np.delete(sampled, S_ - 1), tries, device=dev)
        self_check(want, {k: v.reshape(want[k].shape) for k, v in drop.items()}, keys, allowed,
                   "edge class S − 1 left out")
    if n > 1:
        _, drop = po.fwd_bwd(tabs, norms, pos[:, :-1], sampled, tries, device=dev)
        self_check(want, {k: v.reshape(want[k].shape) for k, v in drop.items()}, keys, allowed,
                   "the last positive left out")
    _, drop = po.fwd_bwd(tabs, norms, pos, sampled, tries, device=dev, drop_true=0)
    self_check(want, {k: v.reshape(want[k].shape) for k, v in drop.items()}, keys, allowed,
               "positive 0's true class left out")


def shared_row_bound(tabs, norms, pos, sampled, tries, dev, which):
    """Every positive has the same head and relation: the one shared row's gradient is Σ_b part_b, zero in exact
    arithmetic.  The parts are the gradients of n copies of the row (one per positive, identical values, so the
    forward is unchanged); the sum may round to γ_k·Σ_b|part_b|, k the longest summation chain."""
    n = pos.shape[1]
    col = 0 if which == "ent" else 1
    copies = dict(tabs)
    copies[which] = np.repeat(tabs[which][pos[col, :1]], n, axis=0)
    cpos = pos.copy()
    cpos[col] = np.arange(n)
    _, parts = po.fwd_bwd(copies, norms, cpos, sampled, tries, device=dev)
    d = tabs[which].shape[1]
    return 16 * gamma(n + 2 * ((d + 3) // 4 * 4) + 24) * np.abs(parts[which]).sum(0)


# ---- the sampler -----------------------------------------------------------------------------------------------------
KROUND = 4096


def run_sampler(dev, n_classes, S, seed, ws=None):
    """oea_logu_sample_unique into a sampled[] pre-filled past S with a sentinel that must survive."""
    lib = L.load()
    need = 4 * n_classes
    ws = torch.empty(need + CANARY, dtype=torch.uint8, device=dev) if ws is None else ws
    sampled = torch.full((S + 8,), -7, dtype=torch.int32, device=dev)
    tries = torch.full((1,), -1, dtype=torch.int32, device=dev)
    rc = lib.oea_logu_sample_unique(n_classes, S, seed, eng._ptr(sampled), eng._ptr(tries), eng._ptr(ws), ws.numel(),
                                    eng._stream_ptr())
    _sync(dev)
    assert rc == 0, rc
    got = sampled.cpu().numpy()
    assert (got[S:] == -7).all(), "sampled[] written past S"
    return got[:S], int(tries.cpu()[0]), ws


def check_sampler(dev, n_classes, S, seed, ws=None):
    got, tries, ws = run_sampler(dev, n_classes, S, seed, ws)
    want, want_tries = po.sample_unique(seed, n_classes, S)
    assert np.array_equal(got, want), (n_classes, S, seed)
    assert tries == want_tries, (tries, want_tries)
    return ws, tries


def round_edge_sizes(n_classes, seed):
    """S whose S-th distinct class is the last draw of the first round of kRound draws, and S whose S-th distinct class
    is the first draw of the second round, from the host draw stream (None where that draw repeats a class)."""
    seen, out = set(), {}
    for j in range(KROUND + 1):
        c = po.draw_classes(seed, j, n_classes)
        fresh = c not in seen
        seen.add(c)
        if j in (KROUND - 1, KROUND):
            out[j] = len(seen) if fresh else None
    return out[KROUND - 1], out[KROUND]


# ---- the pair draw ---------------------------------------------------------------------------------------------------
M64, M32 = (1 << 64) - 1, (1 << 32) - 1


def mix64(z):
    z = (z + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def pairs_key(seed, epoch, step):
    return mix64((seed & M64) ^ mix64(((epoch & M32) << 32) | (step & M32)))


def _mix32(x):
    x = x ^ (x >> np.uint64(16))
    x = (x * np.uint64(0x7FEB352D)) & np.uint64(M32)
    x = x ^ (x >> np.uint64(15))
    x = (x * np.uint64(0x846CA68B)) & np.uint64(M32)
    return x ^ (x >> np.uint64(16))


def feistel_perm(i, n, key):
    """The device's keyed permutation of [0, n): a 4-round balanced Feistel network on 2·⌈bits/2⌉ bits with cycle
    walking, for an array of indices."""
    i = np.asarray(i, dtype=np.uint64)
    if n <= 1:
        return np.zeros_like(i)
    bits = (n - 1).bit_length()
    hb = max((bits + 1) >> 1, 1)
    hmask = np.uint64((1 << hb) - 1)
    x, todo = i.copy(), np.ones(i.shape, dtype=bool)
    while todo.any():
        l, r = x[todo] >> np.uint64(hb), x[todo] & hmask
        for rnd in range(4):
            f = _mix32(r ^ np.uint64((key >> (16 * rnd)) & M32) ^ np.uint64((0x9E3779B9 * (rnd + 1)) & M32)) & hmask
            l, r = r, l ^ f
        x[todo] = (l << np.uint64(hb)) | r
        todo &= x >= n
    return x


def check_pairs_permutation(dev, n, seed, epoch, step):
    """batch == n: `first` is a permutation of all rows, and equal to the host restatement for the same key."""
    lib = L.load()
    pairs = torch.stack([torch.arange(n, dtype=torch.int32), torch.arange(n, dtype=torch.int32) ^ 0x55555555], 1)
    pairs = pairs.contiguous().to(dev)
    first = torch.full((n,), -1, dtype=torch.int32, device=dev)
    second = torch.full((n,), -1, dtype=torch.int32, device=dev)
    rc = lib.oea_pairs_draw(eng._ptr(pairs), n, n, seed, epoch, step, eng._ptr(first), eng._ptr(second),
                            eng._stream_ptr())
    _sync(dev)
    assert rc == 0, rc
    a, b = first.cpu().numpy().astype(np.int64), second.cpu().numpy().astype(np.int64)
    assert np.array_equal(np.sort(a), np.arange(n)), "first is not a permutation of the rows"
    assert np.array_equal(b, a ^ 0x55555555), "second is not the same row's second column"
    want = feistel_perm(np.arange(n), n, pairs_key(seed, epoch, step))
    assert np.array_equal(a, want.astype(np.int64)), "the draw differs from feistel_perm(i, n, pairs_key(…))"
