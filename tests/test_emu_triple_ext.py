"""CPU: the CUDA source of the score-function family (openea_b200/csrc/oea_triple_ext.cu) executed on the warp
emulator of tests/emu (32 lanes as threads, collectives as rendezvous) against oracle/triple_ext.py — the same
checks tests/test_zz_triple_ext_gpu.py makes on the GPU, at sizes a CPU finishes in seconds.  This covers the
kernels' transcription (lane striding, shuffles, chain rule, argument checks, dispatch); it is not a product path."""
import ctypes as C

import numpy as np
import pytest

from openea_b200 import lib as L
from oracle import triple_ext as ox
from tests.emu import build_emu
from tests.helpers import make_batch

LOSSES = {"margin-based": L.LOSS_MARGIN, "limited": L.LOSS_LIMITED, "logistic": L.LOSS_LOGISTIC,
          "positive": L.LOSS_POSITIVE}
KINDS = {"TransE": L.MODEL_TRANSE, "TransH": L.MODEL_TRANSH, "TransD": L.MODEL_TRANSD, "DistMult": L.MODEL_DISTMULT,
         "SimplE": L.MODEL_SIMPLE}


@pytest.fixture(scope="module")
def emu():
    return build_emu.load()


class HostTable:
    """An oea_table over NumPy buffers (the emulator's "device" memory)."""

    def __init__(self, values, norm):
        rows, d = values.shape
        self.d, self.pitch = d, (d + 3) // 4 * 4
        self.weight = np.zeros((rows, self.pitch), dtype=np.float32)
        self.weight[:, :d] = values
        self.grad = np.zeros_like(self.weight)
        self.touched = np.zeros(rows, dtype=np.int32)
        self.struct = L.Table(self.weight.ctypes.data, self.grad.ctypes.data, 0, 0, self.touched.ctypes.data,
                              rows, d, self.pitch, int(norm))


def _case(model, seed, n_ent, n_rel, d, norm):
    rng = np.random.default_rng(seed)
    slots = ox.SLOTS[model] + (None,) * (4 - len(ox.SLOTS[model]))
    tabs, norms = {}, {}
    for i, s in enumerate(slots):
        if s is None:
            continue
        rows = n_rel if i in (1, 3) else n_ent
        tabs[s] = (rng.standard_normal((rows, d)) * (0.6 + 0.3 * i) / np.sqrt(d)).astype(np.float32)
        norms[s] = norm
    if model == "TransH":
        norms["normal"] = True
    return rng, slots, tabs, norms


def _run(emu, model, slots, tables, pos, neg, loss, loss_norm, scale, **kw):
    ptr = lambda s: C.pointer(tables[s].struct) if s is not None else None
    m = L.Model(KINDS[model], *[ptr(s) for s in slots])
    cfg = L.LossCfg(L.SCORE_L1 if loss_norm == "L1" else L.SCORE_L2SQ, LOSSES[loss], kw.get("margin", 0.0),
                    kw.get("neg_margin", 0.0), kw.get("balance", 1.0))
    out = np.zeros(1, dtype=np.float64)
    i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)
    p = [i32(pos[i]) for i in range(3)]
    n = [i32(neg[i]) for i in range(3)] if neg is not None else [None] * 3
    vp = lambda a: C.c_void_p(0 if a is None else a.ctypes.data)
    rc = emu.oea_model_score_fed(C.byref(m), vp(p[0]), vp(p[1]), vp(p[2]), pos.shape[1], vp(n[0]), vp(n[1]), vp(n[2]),
                                 0 if neg is None else neg.shape[1], C.byref(cfg), scale, vp(out), None)
    return rc, float(out[0])


CASES = [("TransE", "limited", 2, "L2"), ("TransE", "margin-based", 1, "L1"),
         ("TransH", "margin-based", 1, "L2"), ("TransH", "limited", 2, "L1"),
         ("TransD", "margin-based", 1, "L2"), ("TransD", "limited", 2, "L2"), ("TransD", "logistic", 1, "L1"),
         ("TransD", "positive", 0, "L2"),
         ("DistMult", "logistic", 2, "L2"), ("SimplE", "logistic", 1, "L2"), ("SimplE", "margin-based", 1, "L2")]


@pytest.mark.parametrize("model,loss,k,loss_norm", CASES)
@pytest.mark.parametrize("d,norm", [(12, True), (75, False), (200, True)])
def test_emulated_kernels_match_oracle(emu, model, loss, k, loss_norm, d, norm):
    n_ent, n_rel, n_pos = 30, 5, 21
    rng, slots, tabs, norms = _case(model, 5 * d + k + len(model), n_ent, n_rel, d, norm)
    pos, neg = make_batch(rng, n_ent, n_rel, n_pos, k)
    kw = dict(margin=1.1 if loss == "margin-based" else 0.3, neg_margin=2.2, balance=0.2)
    scale = 1.0 / (n_pos * (1 + k)) if model == "DistMult" else 1.0
    want_loss, want_g, _ = ox.fwd_bwd(model, tabs, norms, pos, neg, loss, loss_norm=loss_norm, scale=scale, **kw)
    tables = {s: HostTable(tabs[s], norms[s]) for s in slots if s is not None}
    rc, got_loss = _run(emu, model, slots, tables, pos, neg, loss, loss_norm, scale, **kw)
    assert rc == 0
    assert got_loss == pytest.approx(want_loss, rel=1e-4)
    for s, tab in tables.items():
        got, want = tab.grad[:, :d], want_g[s]
        if loss_norm == "L1":
            bad = np.abs(got - want) > 1e-4 * max(1.0, np.abs(want).max())
            assert bad.mean() < 5e-3, s
        else:
            np.testing.assert_allclose(got, want, rtol=1e-4, atol=2e-5 * max(1e-6, np.abs(want).max()), err_msg=s)
        assert not tab.grad[:, d:].any(), "padding columns must stay zero"
        assert (np.abs(want).sum(1)[tab.touched == 0] == 0).all(), "untouched rows must have zero oracle gradient"


def test_emulated_entry_point_argument_checks(emu):
    rng, slots, tabs, norms = _case("TransD", 1, 20, 4, 16, True)
    tables = {s: HostTable(tabs[s], norms[s]) for s in slots if s is not None}
    pos, neg = make_batch(rng, 20, 4, 6, 2)
    rc, _ = _run(emu, "TransD", slots, tables, pos, neg, "margin-based", "L2", 1.0, margin=1.0)
    assert rc == 5                                        # OEA_ERR_SHAPE: margin pairs positive i with negative i
    rc, _ = _run(emu, "TransH", (slots[0], slots[1], None, None), tables, pos, neg, "limited", "L2", 1.0)
    assert rc == 1                                        # OEA_ERR_NULL: TransH without its normal vectors
    wide = {s: HostTable(np.zeros((t.weight.shape[0], 300), dtype=np.float32), True) for s, t in tables.items()}
    rc, _ = _run(emu, "TransD", slots, wide, pos, neg, "limited", "L2", 1.0)
    assert rc == 2                                        # OEA_ERR_DIM: pitch > 256


def test_emulated_adadelta_update_matches_tf_rule(emu):
    """oea_rowopt_adadelta (openea_b200/csrc/oea_optim_ext.cu) on the emulator: three dense steps equal TF1's ApplyAdadelta
    (rho 0.95, epsilon 1e-8) on every row — rows without gradient decay their accumulators too — and leave grad /
    touched zeroed."""
    rng = np.random.default_rng(2)
    rows, d = 37, 10                                            # pitch 12
    tab = HostTable(rng.standard_normal((rows, d)).astype(np.float32), False)
    acc, acc_upd = np.zeros_like(tab.weight), np.zeros_like(tab.weight)
    tab.struct = L.Table(tab.weight.ctypes.data, tab.grad.ctypes.data, acc.ctypes.data, acc_upd.ctypes.data,
                         tab.touched.ctypes.data, rows, d, tab.pitch, 0)
    st = ox.DenseState({"t": tab.weight[:, :d]}, "Adadelta")
    cfg = L.OptCfg(L.OPT_ADADELTA, 0.7, 0.95, 0.0, 1e-8, 1)
    for step in range(3):
        g = np.zeros((rows, d), dtype=np.float32)
        hot = rng.choice(rows, 9, replace=False)
        g[hot] = rng.standard_normal((9, d)).astype(np.float32)
        tab.grad[:, :d] = g
        tab.touched[hot] = 1
        assert emu.oea_rowopt_adadelta(C.byref(tab.struct), C.byref(cfg), None) == 0
        st.apply({"t": g.astype(np.float64)}, 0.7)
        np.testing.assert_allclose(tab.weight[:, :d], st.w["t"], rtol=2e-5, atol=1e-7)
        np.testing.assert_allclose(acc[:, :d], st.s1["t"], rtol=2e-5, atol=1e-12)
        np.testing.assert_allclose(acc_upd[:, :d], st.s2["t"], rtol=1e-4, atol=1e-12)
        assert not tab.grad.any() and not tab.touched.any() and not tab.weight[:, d:].any()
    bad = L.OptCfg(L.OPT_ADAM, 0.7, 0.95, 0.0, 1e-8, 1)
    assert emu.oea_rowopt_adadelta(C.byref(tab.struct), C.byref(bad), None) == 4      # OEA_ERR_KIND


def test_emulator_collectives_behave_like_cuda():
    """cuda_host_emu.h itself: butterfly reductions, broadcasts, ballots, match_any, collectives on lane SUBSETS while
    the other lanes run ahead, 64-bit payloads, shift shuffles, cross-warp exchanges between real barriers, shared and
    global atomics, __syncwarp ordering, 2-D grids."""
    so = build_emu.build_selftest()
    if so is None:
        pytest.skip("no CUDA headers for the emulator build")
    lib = C.CDLL(so)
    lib.emu_selftest.restype = C.c_int
    for _ in range(3):                       # thread interleavings differ from run to run
        assert lib.emu_selftest() == 0


@pytest.mark.parametrize("model", ["TransH", "TransD", "DistMult", "SimplE"])
def test_emulated_scorer_properties_additivity_permutation_scale(emu, model):
    """Properties that need no oracle (the ones the GPU tests use at full size): scoring a batch in two halves adds up to
    scoring it at once; permuting the batch changes nothing; loss_scale scales loss and gradients linearly."""
    rng, slots, tabs, norms = _case(model, 77, 30, 5, 20, True)
    pos, neg = make_batch(rng, 30, 5, 16, 2)
    loss = "logistic" if model in ("DistMult", "SimplE") else "limited"
    kw = dict(margin=0.3, neg_margin=2.2, balance=0.2)

    def run(p, n, scale=1.0, into=None):
        tables = into or {s: HostTable(tabs[s], norms[s]) for s in slots if s is not None}
        rc, val = _run(emu, model, slots, tables, p, n, loss, "L2", scale, **kw)
        assert rc == 0
        return val, tables
    whole, t_whole = run(pos, neg)
    first, t_split = run(pos[:, :8], neg[:, :16])
    second, _ = run(pos[:, 8:], neg[:, 16:], into=t_split)                       # gradients accumulate in the tables
    assert first + second == pytest.approx(whole, rel=1e-5)
    perm_p, perm_n = rng.permutation(16), rng.permutation(32)
    shuffled, t_perm = run(pos[:, perm_p], neg[:, perm_n])
    assert shuffled == pytest.approx(whole, rel=1e-5)
    doubled, t_double = run(pos, neg, scale=2.0)
    assert doubled == pytest.approx(2 * whole, rel=1e-5)
    for s in t_whole:
        ref = t_whole[s].grad
        tol = dict(rtol=1e-4, atol=1e-5 * max(1e-6, np.abs(ref).max()))
        np.testing.assert_allclose(t_split[s].grad, ref, **tol)
        np.testing.assert_allclose(t_perm[s].grad, ref, **tol)
        np.testing.assert_allclose(t_double[s].grad, 2 * ref, **tol)
