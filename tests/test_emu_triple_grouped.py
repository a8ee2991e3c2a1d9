"""CPU: the grouped fed scorer (openea_b200/csrc/oea_triple_grouped.cu: one warp per positive and its negatives,
shared rows loaded once, their gradients summed in registers) on the warp emulator against the C oracle — batches in the
reference's layout, batches whose negatives share nothing with their positive (general path), mixtures, exact copies."""
import ctypes as C

import numpy as np
import pytest

from openea_b200 import lib as L
from oracle import triple as orc
from tests.emu import build_emu
from tests.helpers import make_batch, make_tables
from tests.test_emu_triple_ext import HostTable

LOSSES = {"margin-based": L.LOSS_MARGIN, "limited": L.LOSS_LIMITED, "logistic": L.LOSS_LOGISTIC,
          "positive": L.LOSS_POSITIVE, "logsigmoid": L.LOSS_LOGSIGMOID}


@pytest.fixture(scope="module")
def emu():
    return build_emu.load()


def _run(emu, ent, rel, pos, neg, loss, loss_norm, **kw):
    cfg = L.LossCfg(L.SCORE_L1 if loss_norm == "L1" else L.SCORE_L2SQ, LOSSES[loss], kw.get("margin", 0.0),
                    kw.get("neg_margin", 0.0), kw.get("balance", 1.0))
    out = np.zeros(1, dtype=np.float64)
    i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)
    p = [i32(pos[i]) for i in range(3)]
    n = [i32(neg[i]) for i in range(3)] if neg is not None else [None] * 3
    vp = lambda a: C.c_void_p(0 if a is None else a.ctypes.data)
    rc = emu.oea_triple_score_fed_grouped(C.byref(ent.struct), C.byref(rel.struct), vp(p[0]), vp(p[1]), vp(p[2]),
                                          pos.shape[1], vp(n[0]), vp(n[1]), vp(n[2]), 0 if neg is None else neg.shape[1],
                                          C.byref(cfg), vp(out), None)
    return rc, float(out[0])


@pytest.mark.parametrize("loss,k", [("limited", 3), ("logistic", 2), ("positive", 0), ("logsigmoid", 0), ("margin-based", 1)])
@pytest.mark.parametrize("loss_norm", ["L2", "L1"])
@pytest.mark.parametrize("layout", ["reference", "unrelated", "mixed"])
@pytest.mark.parametrize("d,norm", [(12, True), (75, False), (200, True)])
def test_grouped_scorer_matches_oracle(emu, loss, k, loss_norm, layout, d, norm):
    if k == 0 and layout != "reference":
        pytest.skip("no negatives")
    rng = np.random.default_rng(3 * d + k + len(layout))
    n_ent, n_rel, n_pos = 40, 5, 17
    ent, rel = make_tables(rng, n_ent, n_rel, d)
    pos, neg = make_batch(rng, n_ent, n_rel, n_pos, k)                   # negatives corrupt ONE end of their positive
    if k and layout != "reference":
        rnd = np.stack([rng.integers(0, n_ent, n_pos * k), rng.integers(0, n_rel, n_pos * k), rng.integers(0, n_ent, n_pos * k)])
        pick = np.ones(n_pos * k, dtype=bool) if layout == "unrelated" else rng.random(n_pos * k) < 0.4
        neg = np.where(pick[None, :], rnd, neg).astype(np.int32)
        neg[:, 0] = pos[:, 0]                                            # an exact copy of its positive
    kw = dict(margin=1.1 if loss == "margin-based" else 0.3, neg_margin=2.2, balance=0.2)
    want_loss, want_ge, want_gr, _ = orc.fwd_bwd(ent, rel, pos, neg, loss, loss_norm, norm, norm, **kw)
    te, tr = HostTable(ent, norm), HostTable(rel, norm)
    rc, got_loss = _run(emu, te, tr, pos, neg, loss, loss_norm, **kw)
    assert rc == 0
    assert got_loss == pytest.approx(want_loss, rel=1e-4)
    for tab, want in ((te, want_ge), (tr, want_gr)):
        got = tab.grad[:, :d]
        if loss_norm == "L1":
            bad = np.abs(got - want) > 1e-4 * max(1.0, np.abs(want).max())
            assert bad.mean() < 5e-3
        else:
            np.testing.assert_allclose(got, want, rtol=1e-4, atol=2e-5 * max(1e-6, np.abs(want).max()))
        assert not tab.grad[:, d:].any()
        assert (np.abs(want).sum(1)[tab.touched == 0] == 0).all()


def test_grouped_scorer_argument_checks(emu):
    rng = np.random.default_rng(0)
    ent, rel = make_tables(rng, 20, 3, 16)
    te, tr = HostTable(ent, True), HostTable(rel, True)
    pos, neg = make_batch(rng, 20, 3, 6, 2)
    assert _run(emu, te, tr, pos, neg[:, :11], "limited", "L2")[0] == 5          # n_neg not a multiple of n_pos
    assert _run(emu, te, tr, pos, neg, "margin-based", "L2", margin=1.0)[0] == 5   # margin pairs: k must be 1
    assert _run(emu, te, tr, pos, neg, "positive", "L2")[0] == 5                 # positive-only loss with negatives
