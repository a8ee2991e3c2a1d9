"""CPU: ConvE's step (oea_conve_score_fed in openea_b200/csrc/oea_proje.cu) on the warp emulator of tests/emu against the
float64 oracle of tests/conve_oracle.py: row widths whose factorisations are 1 × d, 2 × 5, 4 × 3, 5 × 15, 10 × 10 and
8 × 16, one to 32 filters, batches of one to 500 positives, keep_prob 1 and 0.7 with the masks restated on the host,
repeated labels and labels inside the sampled set, whole Adam steps on the eight tables, and the argument checks.

Tolerances follow from the longest contraction a gradient passes through: the dense layer's 2Fd terms, the nine taps
of each of F filters, the S sampled classes and the row width, each term in fp32 (γ(k) = k·u/(1 − k·u), u = 2⁻²⁴).
A ReLU whose pre-activation lies within fp32 rounding of 0 could take the other branch on the device, so each case
first checks that every pre-activation reaching the loss exceeds its own fp32 rounding bound, γ(k)·Σ|terms| of its sum
(tests/conve_oracle.py kink_ratios).

The factor 16 on γ: a gradient passes through four contractions in turn (the head's dX over S, the dense layer's dA over
d, the transposed convolution over 9F, the normalisation push over the row), and the bound of each is γ(k_i)·Σ|terms|;
γ(Σk_i) bounds their sum, and 16 allows for the ratio Σ|terms|/|result| of these well-conditioned inputs."""
import ctypes as C
import math

import numpy as np
import pytest

from openea_b200 import lib as L
from tests import conve_oracle as co
from tests.emu import build_emu
from tests.test_emu_proje import HostTable, _aligned

NORMS = {"ent": True, "rel": True}
ERR = {"NULL": 1, "DIM": 2, "SHAPE": 5, "RANGE": 6, "WORKSPACE": 7}
U = 2.0 ** -24
KINK = 1.0                                   # a kink ratio: |pre-activation| over its rounding bound


@pytest.fixture(scope="module")
def emu():
    return build_emu.load()


def gamma(k):
    return k * U / (1 - k * U)


def _case(seed, n_ent, n_rel, d, F):
    rng = np.random.default_rng(seed)
    _, y = co.dim_factorization(d)
    K = 2 * F * d
    tabs = {"ent": rng.standard_normal((n_ent, d)), "rel": rng.standard_normal((n_rel, d)),
            "w": rng.standard_normal((n_ent, d)) * math.sqrt(2.6 / (n_ent + d)),
            "b": rng.standard_normal((n_ent, 1)) * math.sqrt(1.3 / n_ent),
            "conv": np.concatenate([rng.uniform(-1, 1, (F, 9)) * math.sqrt(6 / (9 + 9 * F)) * 3,
                                    rng.standard_normal((F, 1)) * 0.1, rng.uniform(0.5, 1.5, (F, 1)),
                                    rng.standard_normal((F, 1)) * 0.1], 1),
            "bn_in": np.stack([rng.uniform(0.5, 1.5, y) * math.sqrt(d), rng.standard_normal(y) * 0.1]),
            "fc_w": rng.uniform(-1, 1, (K, d)) * math.sqrt(6 / (K + d)) * 2,
            "fc_out": np.stack([rng.standard_normal(d) * 0.1, rng.uniform(0.5, 1.5, d), rng.standard_normal(d) * 0.1])}
    return rng, {k: v.astype(np.float32) for k, v in tabs.items()}


def _tables(tabs):
    return {k: HostTable(v, NORMS.get(k, False)) for k, v in tabs.items()}


def _batch(rng, n_ent, n_rel, n):
    return np.stack([rng.integers(0, n_ent, n), rng.integers(0, n_rel, n), rng.integers(0, n_ent, n)]).astype(np.int32)


def _run(lib, tables, pos, sampled, num_tries, keep=1.0, seed=0, ws_bytes=None, num_sampled=None):
    n_pos = 0 if pos is None else pos.shape[1]
    S = len(sampled) if num_sampled is None else num_sampled
    d, E, F = tables["ent"].d, tables["w"].weight.shape[0], max(1, tables["conv"].weight.shape[0])
    need = lib.oea_conve_workspace_bytes(n_pos, max(1, S), d, F, E)
    raw, base = _aligned(need)
    m = L.Conve(*[C.pointer(tables[k].struct) for k in co.NAMES])
    out = np.zeros(1, dtype=np.float64)
    smp = np.ascontiguousarray(sampled, dtype=np.int32)
    nt = np.array([num_tries], dtype=np.int32)
    p = [np.ascontiguousarray(pos[i], dtype=np.int32) for i in range(3)] if n_pos else [None] * 3
    vp = lambda a: C.c_void_p(0 if a is None else a.ctypes.data)
    rc = lib.oea_conve_score_fed(C.byref(m), vp(p[0]), vp(p[1]), vp(p[2]), n_pos, vp(smp), vp(nt), S, keep, seed,
                                 C.c_void_p(base), need if ws_bytes is None else ws_bytes, vp(out), None)
    return rc, float(out[0])


def _tol(d, F, S):
    pitch = (d + 3) // 4 * 4
    return 16 * gamma(2 * F * d + 9 * F + S + pitch + 64)


def _check(tables, want_g, tol):
    for k, tab in tables.items():
        got, want = tab.grad[:, :tab.d], want_g[k].reshape(tab.grad.shape[0], -1)
        np.testing.assert_allclose(got, want, rtol=tol, atol=tol * max(1e-6, np.abs(want).max()), err_msg=k)
        assert not tab.grad[:, tab.d:].any(), "padding columns must stay zero"
        if k in ("conv", "bn_in", "fc_w", "fc_out"):
            assert tab.touched.all(), "every row of a tower table is flagged"
        else:
            assert (np.abs(want).sum(1)[tab.touched == 0] == 0).all(), "untouched rows must have zero oracle gradient"


def _compare(emu, d, F, n, keep=1.0, n_ent=60, n_rel=7, S=24, seed=0, tweak=None):
    sampled, tries = co.sample_unique(seed + 11, n_ent, S)
    for attempt in range(20):                    # the first inputs with no ReLU input within rounding of a kink
        rng, tabs = _case(seed + 101 * d + 7 * F + n + 100003 * attempt, n_ent, n_rel, d, F)
        pos = _batch(rng, n_ent, n_rel, n)
        if tweak is not None:
            pos = tweak(pos, sampled)
        dseed = 0x5EED0000 + seed + d + n + attempt
        m0, m1 = co.masks(dseed, n, d, F, keep)
        if co.kink_margin(tabs, NORMS, pos, keep, m0, m1) > KINK:
            break
    else:
        pytest.fail("no inputs clear of the ReLU kinks in 20 draws")
    want_loss, want_g = co.fwd_bwd(tabs, NORMS, pos, sampled, tries, keep, m0, m1)
    tables = _tables(tabs)
    rc, got = _run(emu, tables, pos, sampled, tries, keep, dseed)
    assert rc == 0
    tol = _tol(d, F, S)
    assert got == pytest.approx(want_loss, rel=tol)
    _check(tables, want_g, tol)


@pytest.mark.parametrize("d", [7, 10, 12, 75, 100, 128])
def test_emulated_step_matches_oracle_at_every_width(emu, d):
    _compare(emu, d, 3, 5)


@pytest.mark.parametrize("F", [1, 3, 32])
def test_emulated_step_matches_oracle_at_every_filter_count(emu, F):
    _compare(emu, 12, F, 6)


@pytest.mark.parametrize("n", [1, 2, 37])
def test_emulated_step_matches_oracle_at_every_batch(emu, n):
    _compare(emu, 10, 2, n)


def test_emulated_step_matches_oracle_at_a_batch_of_500(emu):
    """Four row tiles of the dense layer's GEMMs and several splits of each reduction."""
    _compare(emu, 7, 1, 500, S=40)


@pytest.mark.parametrize("d,F,n", [(10, 3, 9), (75, 2, 4), (100, 3, 2)])
def test_emulated_step_with_dropout(emu, d, F, n):
    _compare(emu, d, F, n, keep=0.7)


def test_keep_prob_one_is_the_identity(emu):
    """keep_prob = 1: the result does not depend on the dropout seed (the gradients up to the order of the emulator's
    atomic additions)."""
    rng, tabs = _case(5, 40, 5, 12, 2)
    pos = _batch(rng, 40, 5, 9)
    sampled, tries = co.sample_unique(3, 40, 10)
    runs = []
    for seed in (1, 2 ** 63 + 5):
        tables = _tables(tabs)
        rc, loss = _run(emu, tables, pos, sampled, tries, 1.0, seed)
        assert rc == 0
        runs.append((loss, {k: t.grad.copy() for k, t in tables.items()}))
    assert runs[0][0] == runs[1][0]
    for k, g in runs[0][1].items():
        np.testing.assert_allclose(runs[1][1][k], g, rtol=1e-5, atol=1e-6 * np.abs(g).max(), err_msg=k)


def test_dropout_masks_keep_the_expected_share():
    m0, m1 = co.masks(77, 200, 100, 4, 0.7)
    assert abs(m0.mean() - 0.7) < 0.01 and abs(m1.mean() - 0.7) < 0.005
    assert co.masks(77, 3, 10, 2, 1.0)[1].all()


def test_emulated_step_with_repeats_and_accidental_hits(emu):
    """Repeated tails, tails inside the sampled set, repeated heads."""
    def tweak(pos, sampled):
        pos = pos.copy()
        pos[2, :6] = pos[2, 0]
        pos[2, 6:12] = sampled[:6]
        pos[0, 3:9] = pos[0, 3]
        return pos
    _compare(emu, 16, 2, 29, S=20, tweak=tweak)


def test_emulated_adam_steps_match_dense_float64_steps(emu):
    n_ent, n_rel, d, F, lr, keep = 50, 5, 12, 2, 0.01, 0.7
    rng, tabs = _case(3, n_ent, n_rel, d, F)
    tables = _tables(tabs)
    st = co.DenseState(dict(tabs), "Adam")
    for step in range(3):
        pos = _batch(rng, n_ent, n_rel, 23)
        sampled, tries = co.sample_unique(50 + step, n_ent, 16)
        m0, m1 = co.masks(900 + step, 23, d, F, keep)
        assert co.kink_margin({k: v.astype(np.float32) for k, v in st.w.items()}, NORMS, pos, keep, m0, m1) > KINK
        want = co.step(st, NORMS, pos, sampled, tries, keep, m0, m1, lr)
        rc, got = _run(emu, tables, pos, sampled, tries, keep, 900 + step)
        assert rc == 0 and got == pytest.approx(want, rel=1e-4)
        for tab in tables.values():
            tab.adam_t += 1
            cfg = L.OptCfg(L.OPT_ADAM, lr, 0.9, 0.999, 1e-8, tab.adam_t)
            assert emu.oea_rowopt_apply(C.byref(tab.struct), C.byref(cfg), None) == 0
    for k, tab in tables.items():
        got, want = tab.weight[:, :tab.d], st.w[k].reshape(tab.weight.shape[0], -1)
        np.testing.assert_allclose(got, want, rtol=1e-4, atol=2e-6, err_msg=k)


def test_emulated_argument_checks(emu):
    n_ent, n_rel, d, F = 30, 4, 12, 2
    rng, tabs = _case(1, n_ent, n_rel, d, F)
    pos = _batch(rng, n_ent, n_rel, 6)
    sampled, tries = co.sample_unique(1, n_ent, 8)
    tables = _tables(tabs)
    need = emu.oea_conve_workspace_bytes(6, 8, d, F, n_ent)
    assert _run(emu, tables, pos, sampled, tries, ws_bytes=need - 1)[0] == ERR["WORKSPACE"]
    for keep in (0.0, -0.5, 1.5, float("nan")):
        assert _run(emu, tables, pos, sampled, tries, keep=keep)[0] == ERR["RANGE"]
    assert _run(emu, tables, pos, sampled, tries, num_sampled=0)[0] == ERR["RANGE"]
    assert _run(emu, tables, pos, np.arange(n_ent + 1), tries)[0] == ERR["RANGE"]
    no_filters = dict(tables, conv=HostTable(np.zeros((0, 12), np.float32), False))
    assert _run(emu, no_filters, pos, sampled, tries)[0] == ERR["DIM"]                   # F < 1
    wide = {k: HostTable(np.zeros((v.weight.shape[0], 132 if k not in ("b", "conv", "bn_in") else v.d), np.float32),
                         False) for k, v in tables.items()}
    assert _run(emu, wide, pos, sampled, tries)[0] == ERR["DIM"]                         # pitch 132 > 128
    assert _run(emu, dict(tables, rel=HostTable(tabs["rel"], True, pitch=16)), pos, sampled, tries)[0] == ERR["DIM"]
    for k, bad in (("b", tabs["b"][:-1]), ("conv", tabs["conv"][:, :11]), ("bn_in", tabs["bn_in"][:, :2]),
                   ("fc_w", tabs["fc_w"][:-1]), ("fc_out", tabs["fc_out"][:2])):
        assert _run(emu, dict(tables, **{k: HostTable(bad, False)}), pos, sampled, tries)[0] == ERR["SHAPE"], k
    for k in co.NAMES:
        t = HostTable(tabs[k], False)
        t.struct.weight = None
        assert _run(emu, dict(tables, **{k: t}), pos, sampled, tries)[0] == ERR["NULL"], k
    assert _run(emu, tables, None, sampled, tries)[0] == 0                                # an empty batch is a no-op
    assert not any(t.grad.any() for t in tables.values())
    assert emu.oea_conve_workspace_bytes(6, 8, d, 0, n_ent) == 0
