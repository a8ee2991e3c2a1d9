"""CPU: TransR's relation-grouped kernels (openea_b200/csrc/oea_triple_transr.cu) executed on the warp emulator of
tests/emu against the float64 oracle of tests/transr_oracle.py: every row width bucket, every loss and score, relations
split over several chunks, relations absent from the batch, negatives with another relation than their positive,
degenerate rows, the argument checks, the initialisation's scale, and a source mutation the comparison must catch."""
import ctypes as C
import math
import os
import shutil

import numpy as np
import pytest

from openea_b200 import lib as L
from tests import transr_oracle as tro
from tests.emu import build_emu
from tests.helpers import make_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK = 64                                       # kTransrChunk
LOSSES = {"margin-based": L.LOSS_MARGIN, "limited": L.LOSS_LIMITED, "logistic": L.LOSS_LOGISTIC,
          "positive": L.LOSS_POSITIVE}


@pytest.fixture(scope="module")
def emu():
    return build_emu.load()


class HostTable:
    """An oea_table over NumPy buffers (the emulator's "device" memory), with Adagrad / Adam slots."""

    def __init__(self, values, norm, pitch=None):
        rows, d = values.shape
        self.d, self.pitch = d, pitch or (d + 3) // 4 * 4
        self.weight = np.zeros((rows, self.pitch), dtype=np.float32)
        self.weight[:, :d] = values
        self.grad = np.zeros_like(self.weight)
        self.s1 = np.full_like(self.weight, 0.1)
        self.s2 = np.zeros_like(self.weight)
        self.touched = np.zeros(rows, dtype=np.int32)
        self.struct = L.Table(self.weight.ctypes.data, self.grad.ctypes.data, self.s1.ctypes.data, self.s2.ctypes.data,
                              self.touched.ctypes.data, rows, d, self.pitch, int(norm))


def _case(seed, n_ent, n_rel, d, ent_norm=True, rel_norm=True):
    rng = np.random.default_rng(seed)
    tabs = {"ent": (rng.standard_normal((n_ent, d)) * 0.6 / np.sqrt(d)).astype(np.float32),
            "rel": (rng.standard_normal((n_rel, d)) * 0.9 / np.sqrt(d)).astype(np.float32),
            "mat": (rng.standard_normal((n_rel * d, d)) / d).astype(np.float32)}
    return rng, tabs, {"ent": ent_norm, "rel": rel_norm}


def _tables(tabs, norms):
    return {"ent": HostTable(tabs["ent"], norms["ent"]), "rel": HostTable(tabs["rel"], norms["rel"]),
            "mat": HostTable(tabs["mat"], False)}


def _cfg(loss, loss_norm, margin=0.3, neg_margin=1.2, balance=0.4):
    return L.LossCfg(L.SCORE_L1 if loss_norm == "L1" else L.SCORE_L2SQ, LOSSES[loss], margin, neg_margin, balance)


def _run(lib, tables, pos, neg, cfg, scale=1.0, ws_bytes=None, kind=L.MODEL_TRANSR, n_rel=None):
    n_pos = 0 if pos is None else pos.shape[1]
    n_neg = 0 if neg is None else neg.shape[1]
    d = tables["ent"].d
    n_rel = tables["rel"].weight.shape[0] if n_rel is None else n_rel
    need = lib.oea_transr_workspace_bytes(n_pos, n_neg, d, n_rel)
    raw = np.zeros((ws_bytes if ws_bytes is not None else need) + 64, dtype=np.uint8)
    base = raw.ctypes.data + (-raw.ctypes.data) % 16
    m = L.Model(kind, C.pointer(tables["ent"].struct), C.pointer(tables["rel"].struct), None,
                C.pointer(tables["mat"].struct), 0.0, 0.0)
    out = np.zeros(1, dtype=np.float64)
    i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)
    p = [i32(pos[i]) for i in range(3)] if n_pos else [None] * 3
    q = [i32(neg[i]) for i in range(3)] if n_neg else [None] * 3
    vp = lambda a: C.c_void_p(0 if a is None else a.ctypes.data)
    rc = lib.oea_transr_score_fed(C.byref(m), vp(p[0]), vp(p[1]), vp(p[2]), n_pos, vp(q[0]), vp(q[1]), vp(q[2]), n_neg,
                                  C.byref(cfg), scale, C.c_void_p(base),
                                  ws_bytes if ws_bytes is not None else need, vp(out), None)
    return rc, float(out[0])


def _oracle(tabs, norms, pos, neg, loss, loss_norm, margin=0.3, neg_margin=1.2, balance=0.4, scale=1.0):
    kw = dict(margin=margin) if loss == "margin-based" else dict(margin=margin, neg_margin=neg_margin, balance=balance)
    if loss in ("logistic", "positive"):
        kw = {}
    return tro.fwd_bwd(tabs, norms, pos, neg, loss, loss_norm, scale=scale, **kw)


def _check(tables, want_g, d, rtol=1e-4):
    for s, tab in tables.items():
        got, want = tab.grad[:, :d], want_g[s]
        np.testing.assert_allclose(got, want, rtol=rtol, atol=2e-5 * max(1e-6, np.abs(want).max()), err_msg=s)
        assert not tab.grad[:, d:].any(), "padding columns must stay zero"
        assert (np.abs(want).sum(1)[tab.touched == 0] == 0).all(), "untouched rows must have zero oracle gradient"


def _other_relations(rng, neg, n_rel):
    """Negatives whose relation differs from their positive's (a fed batch need not corrupt only h or t)."""
    neg = neg.copy()
    flip = rng.random(neg.shape[1]) < 0.5
    neg[1, flip] = (neg[1, flip] + 1 + rng.integers(0, n_rel - 1, int(flip.sum()))) % n_rel
    return neg


@pytest.mark.parametrize("d", [12, 75, 100, 128])
@pytest.mark.parametrize("ent_norm,rel_norm", [(True, True), (False, False), (False, True)])
def test_emulated_transr_matches_oracle(emu, d, ent_norm, rel_norm):
    n_ent, n_rel, n_pos = 30, 4, 21
    rng, tabs, norms = _case(d + 7 * ent_norm + 3 * rel_norm, n_ent, n_rel, d, ent_norm, rel_norm)
    pos, neg = make_batch(rng, n_ent, n_rel, n_pos, 1)
    neg = _other_relations(rng, neg, n_rel)
    want_loss, want_g = _oracle(tabs, norms, pos, neg, "margin-based", "L2", margin=1.0)
    tables = _tables(tabs, norms)
    rc, got = _run(emu, tables, pos, neg, _cfg("margin-based", "L2", margin=1.0))
    assert rc == 0
    assert got == pytest.approx(want_loss, rel=1e-4)
    _check(tables, want_g, d)


@pytest.mark.parametrize("loss", sorted(LOSSES))
@pytest.mark.parametrize("loss_norm", ["L1", "L2"])
def test_emulated_transr_every_loss_and_score(emu, loss, loss_norm):
    n_ent, n_rel, n_pos, d = 25, 5, 17, 12
    k = {"margin-based": 1, "positive": 0}.get(loss, 3)        # the positive loss scores positives only
    rng, tabs, norms = _case(len(loss) + len(loss_norm), n_ent, n_rel, d)
    pos, neg = make_batch(rng, n_ent, n_rel, n_pos, k)
    neg = None if neg is None else _other_relations(rng, neg, n_rel)
    want_loss, want_g = _oracle(tabs, norms, pos, neg, loss, loss_norm, scale=0.5)
    tables = _tables(tabs, norms)
    rc, got = _run(emu, tables, pos, neg, _cfg(loss, loss_norm), scale=0.5)
    assert rc == 0
    assert got == pytest.approx(want_loss, rel=1e-4)
    _check(tables, want_g, d)


def test_emulated_transr_splits_a_hub_relation_into_chunks(emu):
    """One relation holds more than 2·C of the step's triples: three chunks each add a partial dM_r."""
    n_ent, n_rel, d = 60, 3, 16
    rng, tabs, norms = _case(5, n_ent, n_rel, d)
    n_pos = 2 * CHUNK + 25
    pos, neg = make_batch(rng, n_ent, n_rel, n_pos, 1)
    pos[1, :] = 1
    pos[1, :5] = 0
    neg[1, :] = 1
    neg[1, -3:] = 2
    want_loss, want_g = _oracle(tabs, norms, pos, neg, "margin-based", "L2", margin=2.0)
    tables = _tables(tabs, norms)
    rc, got = _run(emu, tables, pos, neg, _cfg("margin-based", "L2", margin=2.0))
    assert rc == 0
    assert int(((pos[1] == 1).sum() + (neg[1] == 1).sum())) > 2 * CHUNK
    assert got == pytest.approx(want_loss, rel=1e-4)
    _check(tables, want_g, d)


@pytest.mark.parametrize("opt", [L.OPT_ADAGRAD, L.OPT_SGD])
def test_emulated_transr_leaves_absent_relations_untouched(emu, opt):
    """Relations 2 and 4 are not in the batch: their matrix rows are not flagged, receive no gradient, and stay
    bit-identical through the row optimiser; the present relations' rows move."""
    n_ent, n_rel, d = 20, 6, 12
    rng, tabs, norms = _case(11, n_ent, n_rel, d)
    pos, neg = make_batch(rng, n_ent, n_rel, 15, 1)
    present = np.array([0, 1, 3, 5])
    pos[1] = present[rng.integers(0, 4, pos.shape[1])]
    neg[1] = pos[1]
    tables = _tables(tabs, norms)
    before = tables["mat"].weight.copy()
    rc, _ = _run(emu, tables, pos, neg, _cfg("margin-based", "L2", margin=3.0))
    assert rc == 0
    flagged = tables["mat"].touched.reshape(n_rel, d)
    assert not flagged[[2, 4]].any() and flagged[present].all()
    assert not tables["mat"].grad.reshape(n_rel, d, -1)[[2, 4]].any()
    cfg = L.OptCfg(opt, 0.1, 0.9, 0.999, 1e-8, 1)
    assert emu.oea_rowopt_apply(C.byref(tables["mat"].struct), C.byref(cfg), None) == 0
    after = tables["mat"].weight.reshape(n_rel, d, -1)
    assert np.array_equal(after[[2, 4]], before.reshape(n_rel, d, -1)[[2, 4]])
    assert not np.array_equal(after[present], before.reshape(n_rel, d, -1)[present])
    assert not tables["mat"].touched.any() and not tables["mat"].grad.any()


def test_emulated_transr_degenerate_rows(emu):
    """n_pos = 1; repeated entities; a zero entity row; an all-zero M_r (projections below the l2_normalize epsilon:
    TF's max() takes the gradient's scale from the epsilon, and so does the kernel)."""
    n_ent, n_rel, d = 8, 3, 12
    rng, tabs, norms = _case(21, n_ent, n_rel, d)
    tabs["ent"][3] = 0.0
    tabs["mat"][2 * d:3 * d] = 0.0
    for pos, neg in ((np.array([[1], [0], [1]]), np.array([[1], [1], [3]])),
                     (np.array([[3, 3, 1, 5], [2, 1, 0, 2], [3, 4, 1, 3]]), np.array([[3, 6, 1, 5], [2, 2, 0, 1], [7, 4, 3, 3]]))):
        want_loss, want_g = _oracle(tabs, norms, pos, neg, "margin-based", "L2", margin=5.0)
        tables = _tables(tabs, norms)
        rc, got = _run(emu, tables, pos, neg, _cfg("margin-based", "L2", margin=5.0))
        assert rc == 0 and np.isfinite(got)
        assert got == pytest.approx(want_loss, rel=1e-4)
        for s, tab in tables.items():                   # rows at or below eps: gradients scaled by up to 1e6
            assert np.isfinite(tab.grad).all()
            want = want_g[s]
            np.testing.assert_allclose(tab.grad[:, :d], want, rtol=2e-4, atol=1e-4 * max(1e-6, np.abs(want).max()), err_msg=s)


def test_emulated_transr_argument_checks(emu):
    n_ent, n_rel, d = 20, 4, 12
    rng, tabs, norms = _case(1, n_ent, n_rel, d)
    pos, neg = make_batch(rng, n_ent, n_rel, 6, 1)
    tables = _tables(tabs, norms)
    cfg = _cfg("margin-based", "L2")
    need = emu.oea_transr_workspace_bytes(6, 6, d, n_rel)
    assert _run(emu, tables, pos, neg, cfg, ws_bytes=need - 1)[0] == 7          # OEA_ERR_WORKSPACE
    wide = {"ent": HostTable(np.zeros((n_ent, 132), np.float32), True), "rel": HostTable(np.zeros((n_rel, 132), np.float32), True),
            "mat": HostTable(np.zeros((n_rel * 132, 132), np.float32), False)}
    assert _run(emu, wide, pos, neg, cfg)[0] == 2                                  # OEA_ERR_DIM: pitch 132 > 128
    short = dict(tables, mat=HostTable(tabs["mat"][:-d], False))
    assert _run(emu, short, pos, neg, cfg)[0] == 5                                 # OEA_ERR_SHAPE: rows != R·d
    assert _run(emu, tables, pos, neg[:, :5], cfg)[0] == 5                         # margin pairs need n_neg == n_pos
    assert _run(emu, tables, pos, neg, cfg, kind=L.MODEL_TRANSD)[0] == 4          # only the TransR kind
    assert _run(emu, tables, None, None, cfg)[0] == 0                              # an empty batch is a no-op
    m = L.Model(L.MODEL_TRANSR, C.pointer(tables["ent"].struct), C.pointer(tables["rel"].struct), None,
                C.pointer(tables["mat"].struct), 0.0, 0.0)
    out = np.zeros(1)
    p = np.ascontiguousarray(pos, dtype=np.int32)
    vp = lambda a: C.c_void_p(a.ctypes.data)
    assert emu.oea_model_score_fed(C.byref(m), vp(p[0]), vp(p[1]), vp(p[2]), 6, vp(p[0]), vp(p[1]), vp(p[2]), 6,
                                   C.byref(cfg), 1.0, C.c_void_p(out.ctypes.data), None) == 4   # needs a workspace
    assert not any(t.grad.any() for t in tables.values())


@pytest.mark.parametrize("init", ["normal", "xavier"])
def test_transr_matrix_is_drawn_with_the_reference_shape(init):
    """rel_matrix = init_embeddings([R, d²], …): 'normal' is a truncated normal with σ = 1/√(d²) = 1/d (not 1/√d),
    'xavier' has fan R + d²; the values are then stored as R·d rows of width d."""
    from openea_b200.modules.base import initializers
    n_rel, d = 40, 30
    initializers.set_seed(3)
    v = initializers.init_values([n_rel, d * d], init).reshape(n_rel * d, d)
    assert tuple(v.shape) == (n_rel * d, d)
    # torch's truncation at ±2σ leaves a standard deviation of 0.8796·σ
    sigma = 1.0 / d if init == "normal" else math.sqrt(1.3 * 2.0 / (n_rel + d * d))
    assert float(v.std()) == pytest.approx(0.8796 * sigma, rel=0.02)
    assert float(v.abs().max()) <= 2 * sigma + 1e-7
    assert float(v.std()) < 0.8796 / math.sqrt(d) / 2                  # far from the [R·d, d] draw's σ = 1/√d


MUTATION = ("tile_gemm(acc, Gs, ld, 1, Ms, ld, 1, d, ty, tx);          // dX[j][k] = Σ_i G[j][i]·M[i][k]",
            "tile_gemm(acc, Gs, ld, 1, Ms, 1, ld, d, ty, tx);          // dX[j][k] = Σ_i G[j][i]·M[i][k]")


def test_emulated_transr_transposed_backward_mutation_is_caught(tmp_path):
    """The comparison with the oracle has teeth: the kernel source with M_r instead of M_rᵀ in dĥ / dt̂, built for the
    emulator, must disagree with the oracle on the entity gradient, while the matrix gradient still agrees."""
    if build_emu.cuda_include() is None:
        pytest.skip("no CUDA headers for the emulator build")
    csrc = tmp_path / "openea_b200" / "csrc"
    shutil.copytree(os.path.join(ROOT, "openea_b200", "csrc"), csrc)
    shutil.copytree(os.path.join(ROOT, "include"), tmp_path / "include")
    src = (csrc / "oea_triple_transr.cu").read_text()
    assert src.count(MUTATION[0]) == 1, "the mutated statement is not in the kernel source any more"
    (csrc / "oea_triple_transr.cu").write_text(src.replace(MUTATION[0], MUTATION[1]))
    main = tmp_path / "mutant.cpp"
    main.write_text('#include "cuda_host_emu.h"\n#include "openea_b200/csrc/oea_triple_transr.cu"\n')
    mutant = build_emu.load(build_emu.compile(str(main), str(tmp_path / "libmutant.so")),
                            ["oea_transr_score_fed", "oea_transr_workspace_bytes"])
    d = 12
    rng, tabs, norms = _case(12, 30, 4, d)
    pos, neg = make_batch(rng, 30, 4, 13, 1)
    _, want_g = _oracle(tabs, norms, pos, neg, "margin-based", "L2", margin=2.0)
    tables = _tables(tabs, norms)
    rc, _ = _run(mutant, tables, pos, neg, _cfg("margin-based", "L2", margin=2.0))
    assert rc == 0
    with pytest.raises(AssertionError):
        _check({"ent": tables["ent"]}, want_g, d)
    for s in ("mat", "rel"):
        np.testing.assert_allclose(tables[s].grad[:, :d], want_g[s], rtol=1e-4, atol=2e-5 * np.abs(want_g[s]).max())
