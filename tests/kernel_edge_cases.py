"""Edge cases of the path-(i) kernels, shared by tests/test_emu_kernel_edges.py (the CPU warp emulator) and
tests/test_zz_kernel_edges_gpu.py (the H100): every row width the VEC dispatch of oea_rowmath.cuh distinguishes,
batches longer than one resident wave, and degenerate rows, each compared with a float64 statement of the same
operation.  Every `check_*` function takes the engine module (the product's host layer, possibly bound to the emulator
library), the device its tables live on and the device the float64 reference runs on."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import triple_ext as ox
from tests import semantic_ext_oracle as so
from tests.helpers import make_tables, torch_triple_loss

# every pitch-bucket edge of OEA_DISPATCH_VEC (VEC = 1 | 2 | 3 | 4 at pitch <= 128 | 256 | 384 | 512) and dim < pitch
DIMS = (1, 3, 4, 127, 128, 129, 253, 256, 257, 383, 384, 385, 509, 512)
EXT_DIMS = tuple(d for d in DIMS if d <= 256)          # oea_model_score_fed: two float4 per lane at most
LOSSES = (("margin-based", 1), ("limited", 3), ("logistic", 2), ("positive", 0), ("logsigmoid", 0))

ZERO, TINY, SMALL, HOT = 0, 1, 2, 3     # entity rows: all zero, Σx² = 1e-14, Σx² = 1e-10, the hot entity
ZERO_REL = 0                            # an all-zero relation row
EDGE_ENT = (ZERO, TINY, SMALL)


def loss_kw(loss):
    return dict(margin=1.1 if loss == "margin-based" else 0.3, neg_margin=2.2, balance=0.2)


def edge_tables(rng, n_ent, n_rel, d, scale=1.0):
    """make_tables with the degenerate rows: Σx² two decades either side of l2_normalize's 1e-12, so fp32 and fp64 take
    the same branch of max(Σx², eps), and all-zero rows (normalised: x̂ = 0, Jacobian rsqrt(1e-12)·I)."""
    ent, rel = make_tables(rng, n_ent, n_rel, d, scale)
    for row, ss in ((TINY, 1e-14), (SMALL, 1e-10)):
        v = rng.standard_normal(d)
        ent[row] = (v * np.sqrt(ss / (v @ v))).astype(np.float32)
    ent[ZERO] = 0.0
    rel[ZERO_REL] = 0.0
    return ent, rel


def edge_batch(rng, n_ent, n_rel, n_pos, k, hot=0.0, zero_u=True):
    """A fed batch in the reference's layout (the k negatives of positive p at p·k … p·k+k−1) whose first positives are
    a zero head, a zero relation, a self-loop of the sub-eps row, a row just above eps against the zero row and an
    exactly zero u = ĥ + 0 − ĥ; every 7th positive's first negative is a copy of it, every 11th's a triple that shares
    no two rows with it; `hot` of the heads are the one entity HOT."""
    h, r, t = rng.integers(0, n_ent, n_pos), rng.integers(0, n_rel, n_pos), rng.integers(0, n_ent, n_pos)
    if hot:
        h[rng.random(n_pos) < hot] = HOT
    special = [(ZERO, 1 % n_rel, 4 % n_ent), (5 % n_ent, ZERO_REL, 6 % n_ent), (TINY, 1 % n_rel, TINY),
               (SMALL, 2 % n_rel, ZERO)] + ([(7 % n_ent, ZERO_REL, 7 % n_ent)] if zero_u else [])
    for i, s in enumerate(special[:n_pos]):
        h[i], r[i], t[i] = s
    pos = np.stack([h, r, t]).astype(np.int32)
    if k == 0:
        return pos, None
    neg = np.repeat(pos, k, axis=1)
    side = rng.random(n_pos * k) < 0.5
    repl = rng.integers(0, n_ent, n_pos * k)
    neg[0, side] = repl[side]
    neg[2, ~side] = repl[~side]
    gen = np.arange(3, n_pos, 11) * k
    neg[:, gen] = np.stack([rng.integers(0, n_ent, gen.size), rng.integers(0, n_rel, gen.size), rng.integers(0, n_ent, gen.size)])
    # copies only of positives without a degenerate row: a copy's exact ±1e6-scaled cancellation on such a row leaves an
    # fp32 residue of eps32 × the partial sums (~0.1), not a gradient error
    same = np.arange(0, n_pos, 7)
    same = same[~np.isin(pos[0, same], EDGE_ENT) & ~np.isin(pos[2, same], EDGE_ENT) & (pos[1, same] != ZERO_REL)]
    neg[:, same * k] = pos[:, same]
    return pos, neg.astype(np.int32)


def dev_t(x, dev):
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x)).to(dev)


EPS32 = float(np.finfo(np.float32).eps)


def occurrences(index_arrays, rows):
    """How often each of `rows` appears in the given index arrays (the terms summed into that row's gradient)."""
    ids = np.concatenate([np.asarray(a).ravel() for a in index_arrays if a is not None] + [np.zeros(0, dtype=np.int64)])
    return {r: int((ids == r).sum()) for r in rows}


def one_dim_floor(raw, counts_all):
    """Per-row atol floor for normalised rows of ONE coordinate: x̂ = ±1 has a zero Jacobian, so the exact gradient is 0
    and the kernel's is the fp32 residue (ĝ − x̂<x̂, ĝ>)·inv of each of the n terms, at most 8·eps32·6·inv·n."""
    raw = np.asarray(raw, dtype=np.float64)
    inv = 1.0 / np.sqrt(np.maximum((raw * raw).sum(1), 1e-12))
    return 8 * EPS32 * 6 * inv * np.maximum(1, counts_all)


def assert_grads(got, want, l1, edge_rows=(), what="", counts=None, floor=None):
    """The suite's tolerances: rtol 1e-4 with atol 2e-5·max|g| (L1: a bounded fraction of sign flips).  Rows at or below
    eps carry gradients scaled by up to rsqrt(1e-12) = 1e6, which would set the atol of the whole table: they are
    compared row by row.  Such a row's gradient is 1e6·Σ_j ĝ_j over the n terms that reach it, each |ĝ_j| <= 6 (|g| <= 1
    for every loss here, |d s / d û| <= 2·|u| <= 6 for unit rows), accumulated in fp32: its error is bounded by
    about 8·eps32·1e6·6·n, which the per-row atol adds to 2e-5 of the row's own scale (terms that cancel — a self-loop,
    h − t of the same row — leave exactly that fp32 residue, not a wrong gradient).  L1 rows may flip the sign of a
    coordinate where u is 0 in one precision and not in the other (d = 1 normalised rows are ±1: ties are common)."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert np.isfinite(got).all(), what
    rest = np.ones(want.shape[0], dtype=bool)
    rest[list(edge_rows)] = False
    bad = 0
    for i in edge_rows:
        n = 1 if counts is None else max(1, counts.get(i, 1))
        atol = 2e-5 * np.abs(want[i]).max() + 8 * EPS32 * 1e6 * 6 * n
        off = np.abs(got[i] - want[i]) > atol + 1e-4 * np.abs(want[i])
        bad += int(off.sum())
        if not l1:
            assert not off.any(), "%s row %d: %s against %s (atol %g)" % (what, i, got[i][off][:4], want[i][off][:4], atol)
    if l1:
        assert bad <= max(1, 5e-3 * len(edge_rows) * want.shape[1]), "%s: %d sign flips in the degenerate rows" % (what, bad)
    g, w = got[rest], want[rest]
    if l1:
        assert (np.abs(g - w) > 1e-4 * max(1.0, np.abs(w).max())).mean() < 5e-3, what
    else:
        atol = 2e-5 * max(1e-6, np.abs(w).max())
        if floor is not None:
            atol = np.maximum(atol, np.asarray(floor)[rest])[:, None]
        assert (np.abs(g - w) <= atol + 1e-4 * np.abs(w)).all(), "%s: %s against %s" % (what, g.ravel()[:6], w.ravel()[:6])


def _tables(eng, dev, ent, rel, norm, opt="Adagrad"):
    return eng.EmbeddingTable(ent, norm, opt, device=dev), eng.EmbeddingTable(rel, norm, opt, device=dev)


def _check_trainer(t, d, want_loss, want_ge, want_gr, l1, norm, what, pos, neg, ent_cols=(0, 2)):
    assert t.read_loss() == pytest.approx(want_loss, rel=1e-4), what
    b = [pos] + ([] if neg is None else [neg])
    for tab, want, cols, edge in ((t.ent, want_ge, ent_cols, EDGE_ENT), (t.rel, want_gr, tuple(c for c in (0, 1, 2) if c not in ent_cols), (ZERO_REL,))):
        idx = [x[c] for x in b for c in cols]
        floor = None
        if d == 1 and norm:
            ids = np.concatenate([np.asarray(a).ravel() for a in idx] + [np.zeros(0, dtype=np.int64)])
            floor = one_dim_floor(tab.raw().cpu().numpy(), np.bincount(ids, minlength=tab.rows))
        assert_grads(tab.grad[:, :d].cpu().numpy(), want, l1, edge if norm else (), what, occurrences(idx, edge), floor)
    assert not t.ent.grad[:, d:].any() and not t.rel.grad[:, d:].any(), "padding columns must stay zero"


# ---- TripleTrainer.score_fed -------------------------------------------------------------------------------------
def check_fed(eng, dev, d, loss_norm, loss, k, n_pos=33, norm=True, scale=1.0, grouped=False, hot=0.0, n_ent=40,
              n_rel=6, seed=0, ref_dev="cpu"):
    rng = np.random.default_rng(seed)
    ent, rel = edge_tables(rng, n_ent, n_rel, d, scale)
    pos, neg = edge_batch(rng, n_ent, n_rel, n_pos, k, hot)
    kw = loss_kw(loss)
    want_loss, want_ge, want_gr, scores = torch_triple_loss(ent, rel, pos, neg, loss, loss_norm, norm, norm,
                                                            device=ref_dev, **kw)
    te, tr = _tables(eng, dev, ent, rel, norm)
    t = eng.TripleTrainer(te, tr, eng.loss_cfg(loss, loss_norm, **kw), 0.01)
    t.score_fed(dev_t(pos, dev), dev_t(neg, dev), grouped=grouped)
    _check_trainer(t, d, want_loss, want_ge, want_gr, loss_norm == "L1", norm,
                   "fed d=%d %s %s grouped=%s" % (d, loss_norm, loss, grouped), pos, neg)
    return scores


def check_zero_u_contributes_nothing(eng, dev, d, grouped=False):
    """L1 with u exactly 0 (h == t, zero relation row): TF's sign(0) = 0, so these triples put exactly nothing into
    the relation row — whose normalisation Jacobian would otherwise scale a wrong sign by 1e6."""
    rng = np.random.default_rng(d)
    ent, rel = edge_tables(rng, 12, 3, d)
    e = np.arange(12)
    pos = np.stack([e, np.full(12, ZERO_REL), e]).astype(np.int32)
    te, tr = _tables(eng, dev, ent, rel, True)
    t = eng.TripleTrainer(te, tr, eng.loss_cfg("logistic", "L1"), 0.01)
    t.score_fed(dev_t(pos, dev), None, grouped=grouped)
    assert t.read_loss() == pytest.approx(12 * np.log(2.0), rel=1e-6)      # softplus(0) per triple
    assert not te.grad.any() and not tr.grad.any()


# ---- step_fed_grouped against a dense float64 step -----------------------------------------------------------------
def dense_step(w, s1, g, opt, lr):
    if opt == "Adagrad":
        s1 += g * g
        w -= lr * g / np.sqrt(s1)
    else:
        w -= lr * g


def check_step_fed_grouped(eng, dev, d, opt, n_pos=33, k=3, loss="limited", steps=2, seed=0, ref_dev="cpu", hot=0.0,
                           n_ent=40):
    rng = np.random.default_rng(seed)
    ent, rel = edge_tables(rng, n_ent, 6, d)
    kw = loss_kw(loss)
    te, tr = _tables(eng, dev, ent, rel, True, opt)
    t = eng.TripleTrainer(te, tr, eng.loss_cfg(loss, "L2", **kw), 0.01)
    w = [ent.astype(np.float64), rel.astype(np.float64)]
    s1 = [np.full_like(w[0], 0.1), np.full_like(w[1], 0.1)]
    # SGD moves a degenerate row by lr·1e6·g: one step, so that no later step starts from rows of that size
    for _ in range(steps if opt == "Adagrad" else 1):
        pos, neg = edge_batch(rng, n_ent, 6, n_pos, k, hot)
        want, ge, gr, _ = torch_triple_loss(w[0], w[1], pos, neg, loss, "L2", True, True, device=ref_dev, **kw)
        dense_step(w[0], s1[0], ge, opt, 0.01)
        dense_step(w[1], s1[1], gr, opt, 0.01)
        t.step_fed_grouped(dev_t(pos, dev), dev_t(neg, dev))
        assert t.read_loss() == pytest.approx(want, rel=1e-4)
    for tab, ref, edge in ((te, w[0], EDGE_ENT), (tr, w[1], (ZERO_REL,))):
        got = tab.raw().cpu().numpy()
        rest = np.ones(len(ref), dtype=bool)
        rest[list(edge)] = False
        np.testing.assert_allclose(got[rest], ref[rest], rtol=1e-4, atol=1e-6)
        # a degenerate row moves by lr times its 1e6-scaled gradient, whose fp32 error assert_grads bounds (n <= 4·n_pos)
        np.testing.assert_allclose(got[~rest], ref[~rest], rtol=1e-4, atol=0.01 * 8 * EPS32 * 1e6 * 6 * 4 * n_pos)
        assert not tab.weight[:, d:].any() and not tab.grad.any() and not tab.touched.any()


# ---- the sampled scorer, replayed through the float64 reference ------------------------------------------------------
def sampled_setup(eng, dev, rng, n_tri, n, n_rel, d, norm=True, scale=1.0, edge=True):
    """Two KGs over entities [0, n) and [n, 2n) whose triples include the degenerate rows (plain random rows when not
    `edge`) and self-loops."""
    ent, rel = (edge_tables if edge else make_tables)(rng, 2 * n, n_rel, d, scale)

    def kg(lo):
        t = np.stack([rng.integers(lo, lo + n, n_tri), rng.integers(0, n_rel, n_tri), rng.integers(lo, lo + n, n_tri)], 1)
        m = rng.random(n_tri) < 0.05
        t[m, 2] = t[m, 0]                                        # self-loops
        t[: 3 * len(EDGE_ENT), 0] = lo + np.tile(EDGE_ENT, 3)    # the degenerate rows as heads
        t[: 3, 1] = ZERO_REL
        return np.unique(t.astype(np.int32), axis=0)
    t1, t2 = kg(0), kg(n)
    kg1 = eng.DeviceKG(t1, np.arange(0, n), 2 * n, device=dev)
    kg2 = eng.DeviceKG(t2, np.arange(n, 2 * n), 2 * n, device=dev)
    tset = eng.DeviceTripleSet([kg1.triples, kg2.triples], 2 * n, n_rel, device=dev)
    return ent, rel, t1, t2, kg1, kg2, tset


def decode_dbg(rows, t1, t2, k):
    """The batch a sampled kernel drew, from its debug dump (row = [triple id, head mask, k negative entities];
    ids ≥ 2³⁰ index the second KG): pos [3, m], neg [3, m·k] in the reference's layout.  Vectorised."""
    tri = rows[:, 0].astype(np.int64)
    second = tri >= (1 << 30)
    pos = np.where(second[:, None], t2[np.where(second, tri - (1 << 30), 0)], t1[np.where(second, 0, tri)]).T
    pos = np.ascontiguousarray(pos, dtype=np.int32)
    if k == 0:
        return pos, None
    neg = np.repeat(pos, k, axis=1)
    head = ((rows[:, 1:2].astype(np.int64) >> np.arange(k)) & 1).astype(bool).ravel()
    e = rows[:, 2:2 + k].ravel()
    neg[0, head] = e[head]
    neg[2, ~head] = e[~head]
    return pos, neg


def check_sampled(eng, dev, d, loss_norm, loss, k, B, norm=True, n_tri=120, n=50, seed=0, ref_dev="cpu"):
    rng = np.random.default_rng(seed)
    ent, rel, t1, t2, kg1, kg2, tset = sampled_setup(eng, dev, rng, n_tri, n, 5, d, norm)
    kw = loss_kw(loss)
    te, tr = _tables(eng, dev, ent, rel, norm)
    t = eng.TripleTrainer(te, tr, eng.loss_cfg(loss, loss_norm, **kw), 0.01)
    dbg = torch.full((B, 2 + k), -7, dtype=torch.int32, device=dev)
    n_pos = torch.zeros(1, dtype=torch.int32, device=dev)
    t.score_sampled(kg1, kg2, tset, B, k, 1, 4242, dbg=dbg, n_pos_out=n_pos)
    m = int(n_pos.item())
    rows = dbg.cpu().numpy()[:m]
    assert m > 0 and (rows[:, 0] != -7).all() and (rows[:, 2:] != -7).all()
    pos, neg = decode_dbg(rows, t1, t2, k)
    want_loss, want_ge, want_gr, _ = torch_triple_loss(ent, rel, pos, neg, loss, loss_norm, norm, norm, device=ref_dev, **kw)
    _check_trainer(t, d, want_loss, want_ge, want_gr, loss_norm == "L1", norm, "sampled d=%d %s %s k=%d" % (d, loss_norm, loss, k), pos, neg)
    return m


# ---- the weighted margin scorer and the pair loss ------------------------------------------------------------------
def _normed(x, on):
    return x * torch.rsqrt(torch.clamp((x * x).sum(1, keepdim=True), min=1e-12)) if on else x


def check_margin_weighted(eng, dev, d, loss_norm, paths, n=37, seed=0):
    rng = np.random.default_rng(seed + d)
    n_ent, n_rel = 30, 9
    ent, rel = edge_tables(rng, n_ent, n_rel, d)
    hi = n_rel if paths else n_ent
    pos, neg = (np.stack([rng.integers(0, hi, n), rng.integers(0, n_rel, n), rng.integers(0, hi, n)]).astype(np.int32)
                for _ in range(2))
    pos[:, :3] = [[ZERO, TINY, SMALL], [1, ZERO_REL, 2], [4, TINY, ZERO]]
    neg[:, 5] = pos[:, 5]
    w = (rng.random(n) * 3 + 0.5).astype(np.float32)
    E = torch.tensor(ent, dtype=torch.float64, requires_grad=True)
    R = torch.tensor(rel, dtype=torch.float64, requires_grad=True)
    A, Rn = (_normed(R, True) if paths else _normed(E, True)), _normed(R, True)

    def score(b):
        u = A[b[0].astype(np.int64)] + Rn[b[1].astype(np.int64)] - A[b[2].astype(np.int64)]
        return u.abs().sum(1) if loss_norm == "L1" else (u * u).sum(1)
    want = 0.5 * (torch.tensor(w, dtype=torch.float64) * torch.relu(0.8 + score(pos) - score(neg))).sum()
    want.backward()
    te, tr = _tables(eng, dev, ent, rel, True)
    t = eng.TripleTrainer(te, tr, eng.loss_cfg("margin-based", loss_norm, margin=0.8), 0.01)
    t.score_margin_weighted(dev_t(pos, dev), dev_t(neg, dev), dev_t(w, dev), scale=0.5, paths=paths)
    ge = np.zeros_like(ent, dtype=np.float64) if E.grad is None else E.grad.numpy()
    _check_trainer(t, d, float(want.detach()), ge, R.grad.numpy(), loss_norm == "L1", True,
                   "weighted d=%d %s paths=%s" % (d, loss_norm, paths), pos, neg, () if paths else (0, 2))


def check_pairs(eng, dev, d, n=29, seed=0):
    rng = np.random.default_rng(seed + d)
    ent, rel = edge_tables(rng, 25, 2, d)
    a, b = rng.integers(0, 25, n).astype(np.int32), rng.integers(0, 25, n).astype(np.int32)
    a[:4], b[:4] = [ZERO, TINY, SMALL, 5], [TINY, TINY, ZERO, 5]
    w = (rng.random(n) + 0.1).astype(np.float32)
    E = torch.tensor(ent, dtype=torch.float64, requires_grad=True)
    En = _normed(E, True)
    want = 0.7 * (torch.tensor(w, dtype=torch.float64) * ((En[a.astype(np.int64)] - En[b.astype(np.int64)]) ** 2).sum(1)).sum()
    want.backward()
    te, tr = _tables(eng, dev, ent, rel, True)
    t = eng.TripleTrainer(te, tr, eng.loss_cfg("margin-based", "L2", margin=1.0), 0.01)
    t.score_pairs(a, b, dev_t(w, dev), scale=0.7)
    assert t.read_loss() == pytest.approx(float(want.detach()), rel=1e-4)
    floor = one_dim_floor(ent, np.bincount(np.concatenate([a, b]), minlength=25)) if d == 1 else None
    assert_grads(te.grad[:, :d].cpu().numpy(), E.grad.numpy(), False, EDGE_ENT, "pairs d=%d" % d, occurrences([a, b], EDGE_ENT),
                 floor)
    assert not te.grad[:, d:].any()


# ---- ModelTrainer.score_fed: TransH, TransD, DistMult, SimplE, RotatE, HolE ---------------------------------------------
EXT_CASES = (("TransH", "margin-based", 1, "L2"), ("TransH", "limited", 2, "L1"), ("TransD", "margin-based", 1, "L1"),
             ("TransD", "logistic", 2, "L2"), ("DistMult", "logistic", 2, "L2"), ("SimplE", "logistic", 1, "L2"),
             ("RotatE", "logistic", 3, "L2"), ("HolE", "margin-based", 2, "L2"))
EXT_LOSSES = {"margin-based": "margin-based", "limited": "limited", "logistic": "logistic"}
GAMMA = 6.0


def ext_tables(model, rng, n_ent, n_rel, d, norm):
    slots = (ox.SLOTS if model in ox.SLOTS else so.SLOTS)[model]
    slots = slots + (None,) * (4 - len(slots))
    tabs, norms = {}, {}
    for i, s in enumerate(slots):
        if s is None:
            continue
        rows = n_rel if i in (1, 3) else n_ent
        x = (rng.standard_normal((rows, d)) * (0.6 + 0.3 * i) / np.sqrt(d)).astype(np.float32)
        if model != "RotatE" or rows == n_rel:
            x[0] = 0.0                                               # zero rows in every table, auxiliary ones included
        if rows == n_ent:
            x[TINY] *= np.float32(np.sqrt(1e-14 / float((x[TINY].astype(np.float64) ** 2).sum())))
        tabs[s], norms[s] = x, norm
    if model == "TransH":
        norms["normal"] = True
    return slots, tabs, norms


def check_ext(eng, dev, model, loss, k, loss_norm, d, norm=None, n_pos=21, seed=0):
    # below 4 coordinates the tables are unnormalised: a normalised row of one coordinate is ±1, and TransD's
    # ê + <ê, êt>·r̂p then cancels exactly, leaving an fp32 residue that l2_normalize's sub-eps branch multiplies by 1e6
    norm = d >= 4 if norm is None else norm
    rng = np.random.default_rng(seed + d + len(model))
    n_ent, n_rel = 30, 5
    slots, tabs, norms = ext_tables(model, rng, n_ent, n_rel, d, norm)
    # RotatE: no zero entity row and no exactly zero u, where the modulus is not differentiable (TF's gradient is NaN,
    # the kernel's 0 by decision, oea_triple_ext.cu)
    pos, neg = edge_batch(rng, n_ent, n_rel, n_pos, k, zero_u=model != "RotatE")
    if model == "RotatE":                                  # nor a self-loop under the zero relation's identity rotation
        for x in (pos, neg):
            x[2] = np.where(x[0] == x[2], (x[2] + 1) % n_ent, x[2])
    kw = loss_kw(loss)
    scale = 1.0 / (n_pos * (1 + k)) if model == "DistMult" else 1.0
    if model == "RotatE":
        want_loss, want_g = so.fwd_bwd(model, tabs, norms, pos, neg, gamma=GAMMA, neg_weight=1.0)
    elif model == "HolE":
        want_loss, want_g = so.fwd_bwd(model, tabs, norms, pos, neg, margin=kw["margin"])
    else:
        want_loss, want_g, _ = ox.fwd_bwd(model, tabs, norms, pos, neg, loss, loss_norm=loss_norm, scale=scale, **kw)
    tables = [None if s is None else eng.EmbeddingTable(tabs[s], norms[s], device=dev) for s in slots]
    t = eng.ModelTrainer(model, tables, eng.loss_cfg(loss, loss_norm, **kw), 0.01, mean_loss=model == "DistMult",
                         gamma=GAMMA if model == "RotatE" else None)
    t.score_fed(dev_t(pos, dev), dev_t(neg, dev))
    what = "%s d=%d %s %s" % (model, d, loss, loss_norm)
    assert t.read_loss() == pytest.approx(want_loss, rel=1e-4), what
    for s, tab in zip(slots, tables):
        if tab is None:
            continue
        edge = ((0, TINY) if tab.rows == n_ent else (0,)) if norms[s] else ()
        cols = (1,) if tab.rows == n_rel else (0, 2)
        idx = [x[c] for x in (pos, neg) for c in cols]
        floor = None
        if d == 1:          # the models' own l2_normalize calls (TransD's projection, SimplE's h∘r) have a zero Jacobian too
            ids = np.concatenate([np.asarray(a).ravel() for a in idx])
            floor = one_dim_floor(tab.raw().cpu().numpy(), np.bincount(ids, minlength=tab.rows))
        assert_grads(tab.grad[:, :d].cpu().numpy(), want_g[s], loss_norm == "L1", edge, what + " " + s,
                     occurrences(idx, edge), floor)
        assert not tab.grad[:, d:].any(), "padding columns must stay zero"


# ---- lookup, scatter_grad, the mapping loss and the optimisers ----------------------------------------------------------
def check_lookup_scatter(eng, dev, d, n=41, seed=0):
    rng = np.random.default_rng(seed + d)
    ent, _ = edge_tables(rng, 30, 2, d)
    te = eng.EmbeddingTable(ent, True, device=dev)
    ids = rng.integers(0, 30, n).astype(np.int32)
    ids[:4] = [ZERO, TINY, SMALL, TINY]
    X = torch.tensor(ent, dtype=torch.float64, requires_grad=True)
    Xn = _normed(X, True)
    got = te.lookup(ids).cpu().numpy()
    want = Xn.detach().numpy()[ids]
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-6)
    assert (te.lookup(ids, padded=True)[:, d:] == 0).all()
    w = rng.standard_normal((n, d)).astype(np.float32)
    (Xn[torch.as_tensor(ids, dtype=torch.long)] * torch.as_tensor(w, dtype=torch.float64)).sum().backward()
    te.scatter_grad(dev_t(w, dev), ids)
    floor = one_dim_floor(ent, np.bincount(ids, minlength=30)) * np.abs(w).max() / 6 if d == 1 else None
    assert_grads(te.grad[:, :d].cpu().numpy(), X.grad.numpy(), False, EDGE_ENT, "scatter d=%d" % d, occurrences([ids], EDGE_ENT),
                 floor)
    assert not te.grad[:, d:].any()
    assert set(np.flatnonzero(te.touched.cpu().numpy())) == set(ids.tolist())


def check_mapping(eng, dev, d, n=19, alpha=0.3, seed=0):
    from openea_b200 import lib as L
    rng = np.random.default_rng(seed + d)
    p = eng.pitch_for(d)
    e1, e2 = (rng.standard_normal((n, d)).astype(np.float32) for _ in range(2))
    M = (np.eye(d) + 0.1 * rng.standard_normal((d, d)) / np.sqrt(d)).astype(np.float32)
    pad = lambda x: torch.nn.functional.pad(torch.from_numpy(x), (0, p - d)).contiguous().to(dev)
    E1, E2, Mt = pad(e1), pad(e2), pad(M)
    g1, g2, gM = torch.zeros_like(E1), torch.zeros_like(E2), torch.zeros_like(Mt)
    loss = torch.zeros(1, dtype=torch.float64, device=dev)
    lib = L.load()
    ws_bytes = lib.oea_mapping_workspace_bytes(d)
    ws = torch.zeros(max(1, ws_bytes // 4), dtype=torch.float32, device=dev)
    vp = lambda t: C.c_void_p(t.data_ptr())
    L.check(lib.oea_mapping_fwd_bwd(vp(E1), vp(E2), n, d, p, vp(Mt), p, alpha, vp(loss), vp(g1), vp(g2), vp(gM), vp(ws),
                                    ws_bytes, eng._stream_ptr()), "oea_mapping_fwd_bwd")
    a, b, m = (torch.tensor(x, dtype=torch.float64, requires_grad=True) for x in (e1, e2, M))
    res = b - a @ m
    want = alpha * ((res * res).sum() + ((m @ m.T - torch.eye(d, dtype=torch.float64)) ** 2).sum())
    want.backward()
    assert float(loss.item()) == pytest.approx(float(want.detach()), rel=1e-4)
    for got, ref, what in ((g1, a.grad, "g_e1"), (g2, b.grad, "g_e2"), (gM, m.grad, "g_M")):
        assert_grads(got[:, :d].cpu().numpy(), ref.numpy(), False, (), "mapping d=%d %s" % (d, what))
        assert not got[:, d:].any(), what


def check_apply(eng, dev, d, opt, steps=3, lr=0.05, seed=0):
    """EmbeddingTable.apply (oea_rowopt_apply) against the dense float64 TF-1 rules, gradients on a subset of rows:
    padding columns stay zero, and for the row-sparse rules (Adagrad, SGD) untouched rows keep their exact bits."""
    rng = np.random.default_rng(seed + d)
    rows = 37
    x, _ = edge_tables(rng, rows, 2, d)
    tab = eng.EmbeddingTable(x, True, opt, device=dev)
    st = ox.DenseState({"x": x}, opt)
    hit = np.zeros(rows, dtype=bool)
    for _ in range(steps):
        ids = rng.choice(rows, 11, replace=False)
        hit[ids] = True
        g = np.zeros((rows, d), dtype=np.float32)
        g[ids] = rng.standard_normal((11, d)).astype(np.float32)
        tab.grad[:, :d] = torch.from_numpy(g).to(dev)
        tab.touched[torch.as_tensor(ids, dtype=torch.long, device=dev)] = 1
        tab.apply(lr)
        st.apply({"x": g.astype(np.float64)}, lr)
    got = tab.raw().cpu().numpy()
    np.testing.assert_allclose(got, st.w["x"], rtol=1e-4, atol=1e-6)
    assert not tab.weight[:, d:].any() and not tab.grad.any() and not tab.touched.any()
    if opt in ("Adagrad", "SGD"):
        assert np.array_equal(got[~hit], x[~hit])
