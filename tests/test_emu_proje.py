"""CPU: ProjE's kernels (openea_b200/csrc/oea_proje.cu) on the warp emulator of tests/emu (tests/emu/build_emu_proje.py):
the unique log-uniform sampler against the sequential loop over the same draw stream, the step's forward and backward
against the float64 oracle of tests/proje_oracle.py (row widths, batch sizes down to one positive, sampled sets up to
every class, repeated labels, labels inside the sampled set, TF's expected-count shortcut), whole Adam steps on the five
tables, and the argument checks."""
import ctypes as C
import math

import numpy as np
import pytest
from scipy import stats

from openea_b200 import lib as L
from tests import proje_oracle as po
from tests.emu import build_emu_proje


def _bind(lib):
    for name in ("oea_logu_sample_unique", "oea_proje_workspace_bytes", "oea_proje_score_fed", "oea_rowopt_apply"):
        res, args = L.SIGNATURES[name]
        getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    return lib


@pytest.fixture(scope="module")
def emu():
    so_path = build_emu_proje.build()
    if so_path is None:
        pytest.skip("no CUDA headers for the emulator build")
    return _bind(C.CDLL(so_path))


def _aligned(nbytes):
    raw = np.zeros(nbytes + 64, dtype=np.uint8)
    return raw, raw.ctypes.data + (-raw.ctypes.data) % 16


class HostTable:
    """An oea_table over NumPy buffers (the emulator's "device" memory) with Adam slots."""

    def __init__(self, values, norm, pitch=None):
        values = np.asarray(values, dtype=np.float32)
        rows, d = values.shape
        self.d, self.pitch = d, pitch or (d + 3) // 4 * 4
        self.weight = np.zeros((rows, self.pitch), dtype=np.float32)
        self.weight[:, :d] = values
        self.grad = np.zeros_like(self.weight)
        self.s1 = np.zeros_like(self.weight)
        self.s2 = np.zeros_like(self.weight)
        self.touched = np.zeros(rows, dtype=np.int32)
        self.adam_t = 0
        self.struct = L.Table(self.weight.ctypes.data, self.grad.ctypes.data, self.s1.ctypes.data, self.s2.ctypes.data,
                              self.touched.ctypes.data, rows, d, self.pitch, int(norm))


NAMES = ("ent", "rel", "w", "b", "params")


def _case(seed, n_ent, n_rel, d):
    rng = np.random.default_rng(seed)
    lim = math.sqrt(3.0 / d)
    tabs = {"ent": rng.standard_normal((n_ent, d)) * math.sqrt(1.3 * 2 / (n_ent + d)),
            "rel": rng.standard_normal((n_rel, d)) * math.sqrt(1.3 * 2 / (n_rel + d)),
            "w": rng.standard_normal((n_ent, d)) * math.sqrt(1.3 * 2 / (n_ent + d)),
            "b": rng.standard_normal((n_ent, 1)) * math.sqrt(1.3 / n_ent),
            "params": np.stack([rng.uniform(-lim, lim, d), rng.uniform(-lim, lim, d),
                                rng.standard_normal(d) * 0.1, rng.standard_normal(d) * 0.1])}
    return rng, {k: v.astype(np.float32) for k, v in tabs.items()}


NORMS = {"ent": True, "rel": True}


def _tables(tabs):
    return {k: HostTable(v, NORMS.get(k, False)) for k, v in tabs.items()}


def _sample(lib, n_classes, S, seed, ws_bytes=None):
    need = lib.oea_proje_workspace_bytes(1, S, 4, n_classes)
    raw, base = _aligned(need)
    sampled = np.full(S, -1, dtype=np.int32)
    tries = np.zeros(1, dtype=np.int32)
    rc = lib.oea_logu_sample_unique(n_classes, S, seed, C.c_void_p(sampled.ctypes.data), C.c_void_p(tries.ctypes.data),
                                    C.c_void_p(base), need if ws_bytes is None else ws_bytes, None)
    return rc, sampled, int(tries[0])


def _run(lib, tables, pos, sampled, num_tries, ws_bytes=None, num_sampled=None):
    n_pos = 0 if pos is None else pos.shape[1]
    S = len(sampled) if num_sampled is None else num_sampled
    d, E = tables["ent"].d, tables["w"].weight.shape[0]
    need = lib.oea_proje_workspace_bytes(n_pos, max(1, S), d, E)
    raw, base = _aligned(need)
    m = L.Proje(*[C.pointer(tables[k].struct) for k in NAMES])
    out = np.zeros(1, dtype=np.float64)
    smp = np.ascontiguousarray(sampled, dtype=np.int32)
    nt = np.array([num_tries], dtype=np.int32)
    p = [np.ascontiguousarray(pos[i], dtype=np.int32) for i in range(3)] if n_pos else [None] * 3
    vp = lambda a: C.c_void_p(0 if a is None else a.ctypes.data)
    rc = lib.oea_proje_score_fed(C.byref(m), vp(p[0]), vp(p[1]), vp(p[2]), n_pos, vp(smp), vp(nt), S, C.c_void_p(base),
                                 need if ws_bytes is None else ws_bytes, vp(out), None)
    return rc, float(out[0])


def _check(tables, want_g, rtol=2e-4):
    for k, tab in tables.items():
        got, want = tab.grad[:, :tab.d], want_g[k].reshape(tab.grad.shape[0], -1)
        np.testing.assert_allclose(got, want, rtol=rtol, atol=1e-4 * max(1e-6, np.abs(want).max()), err_msg=k)
        assert not tab.grad[:, tab.d:].any(), "padding columns must stay zero"
        assert (np.abs(want).sum(1)[tab.touched == 0] == 0).all(), "untouched rows must have zero oracle gradient"


def _batch(rng, n_ent, n_rel, n):
    return np.stack([rng.integers(0, n_ent, n), rng.integers(0, n_rel, n), rng.integers(0, n_ent, n)]).astype(np.int32)


# ---- the sampler -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_classes,sizes", [(40, (2, 12, 39, 40)), (1000, (2, 64, 999)), (30000, (2, 4096))])
def test_emulated_sampler_is_the_sequential_loop(emu, n_classes, sizes):
    for i, S in enumerate(sizes):
        seed = 1000003 * n_classes + 7 * i
        rc, got, tries = _sample(emu, n_classes, S, seed)
        assert rc == 0
        want, want_tries = po.sample_unique(seed, n_classes, S)
        assert np.array_equal(got, want) and tries == want_tries
        assert len(set(got.tolist())) == S and got.min() >= 0 and got.max() < n_classes


def test_first_draw_follows_the_log_uniform_distribution():
    """Chi-square of the first draw of 20 000 seeds (the restatement the emulated sampler equals) against P(c)."""
    n_classes, n = 50, 20000
    counts = np.bincount([po.draw_classes(s * 7919 + 3, 0, n_classes) for s in range(n)], minlength=n_classes)
    p = po.probability(np.arange(n_classes), n_classes).astype(np.float64)
    p /= p.sum()
    assert stats.chisquare(counts, n * p).pvalue > 1e-3


# ---- the step ------------------------------------------------------------------------------------------------------
def _compare(emu, d, n_pos, n_ent=60, n_rel=7, S=24, seed=0, tweak=None, shortcut=False):
    rng, tabs = _case(seed + d + n_pos, n_ent, n_rel, d)
    pos = _batch(rng, n_ent, n_rel, n_pos)
    sampled, tries = po.sample_unique(seed + 11, n_ent, S)
    if shortcut:
        tries = S
    if tweak is not None:
        pos = tweak(pos, sampled)
    want_loss, want_g = po.fwd_bwd(tabs, NORMS, pos, sampled, tries)
    tables = _tables(tabs)
    rc, got = _run(emu, tables, pos, sampled, tries)
    assert rc == 0
    assert got == pytest.approx(want_loss, rel=2e-5)
    _check(tables, want_g)


@pytest.mark.parametrize("d", [10, 75, 100, 128])
def test_emulated_step_matches_oracle_at_every_width(emu, d):
    _compare(emu, d, 37)


@pytest.mark.parametrize("n_pos", [1, 2, 37, 500])
def test_emulated_step_matches_oracle_at_every_batch(emu, n_pos):
    """n_pos = 1: every batch norm sees a variance of 0; 500: four row tiles and sixteen splits of the batch."""
    _compare(emu, 75, n_pos, S=40 if n_pos == 500 else 24)


@pytest.mark.parametrize("S", [2, 59, 60])
def test_emulated_step_matches_oracle_for_sampled_sets_up_to_every_class(emu, S):
    _compare(emu, 12, 21, S=S, seed=S)


def test_emulated_step_with_the_expected_count_shortcut(emu):
    """num_tries == S: q(c) = P(c)·S, fed explicitly."""
    _compare(emu, 20, 17, S=16, shortcut=True)


def test_emulated_step_with_repeats_and_accidental_hits(emu):
    """Repeated tails, tails inside the sampled set, repeated heads."""
    def tweak(pos, sampled):
        pos = pos.copy()
        pos[2, :6] = pos[2, 0]
        pos[2, 6:12] = sampled[:6]
        pos[0, 3:9] = pos[0, 3]
        return pos
    _compare(emu, 16, 29, S=20, tweak=tweak)


def test_emulated_adam_steps_match_dense_float64_steps(emu):
    n_ent, n_rel, d, lr = 50, 5, 20, 0.01
    rng, tabs = _case(3, n_ent, n_rel, d)
    tables = _tables(tabs)
    st = po.DenseState({k: v for k, v in tabs.items()}, "Adam")
    for step in range(3):
        pos = _batch(rng, n_ent, n_rel, 23)
        sampled, tries = po.sample_unique(50 + step, n_ent, 16)
        want = po.step(st, NORMS, pos, sampled, tries, lr)
        rc, got = _run(emu, tables, pos, sampled, tries)
        assert rc == 0 and got == pytest.approx(want, rel=2e-5)
        for tab in tables.values():
            tab.adam_t += 1
            cfg = L.OptCfg(L.OPT_ADAM, lr, 0.9, 0.999, 1e-8, tab.adam_t)
            assert emu.oea_rowopt_apply(C.byref(tab.struct), C.byref(cfg), None) == 0
    for k, tab in tables.items():
        got, want = tab.weight[:, :tab.d], st.w[k].reshape(tab.weight.shape[0], -1)
        if k == "params":
            # mlp_bias and the input beta feed the output batch norm, whose backward sums to zero over the batch: their
            # gradient is 0 up to rounding, which Adam turns into steps of up to lr either way (in TF as well)
            assert np.abs(got[1:3] - want[1:3]).max() <= 2 * 3 * lr
            got, want = got[[0, 3]], want[[0, 3]]
        np.testing.assert_allclose(got, want, rtol=1e-4, atol=2e-6, err_msg=k)


def test_emulated_argument_checks(emu):
    n_ent, n_rel, d = 30, 4, 12
    rng, tabs = _case(1, n_ent, n_rel, d)
    pos = _batch(rng, n_ent, n_rel, 6)
    sampled, tries = po.sample_unique(1, n_ent, 8)
    tables = _tables(tabs)
    need = emu.oea_proje_workspace_bytes(6, 8, d, n_ent)
    assert _run(emu, tables, pos, sampled, tries, ws_bytes=need - 1)[0] == L_ERR["WORKSPACE"]
    assert _run(emu, tables, pos, sampled, tries, num_sampled=0)[0] == L_ERR["RANGE"]
    assert _run(emu, tables, pos, np.arange(n_ent + 1), tries)[0] == L_ERR["RANGE"]
    wide = dict(tables, ent=HostTable(np.zeros((n_ent, 132), np.float32), True))
    assert _run(emu, wide, pos, sampled, tries)[0] == L_ERR["DIM"]
    wide = {k: HostTable(np.zeros((v.weight.shape[0], 132 if k != "b" else 1), np.float32), False) for k, v in tables.items()}
    assert _run(emu, wide, pos, sampled, tries)[0] == L_ERR["DIM"]                       # pitch 132 > 128
    other = dict(tables, rel=HostTable(tabs["rel"], True, pitch=16))
    assert _run(emu, other, pos, sampled, tries)[0] == L_ERR["DIM"]                      # pitches disagree
    assert _run(emu, dict(tables, b=HostTable(tabs["b"][:-1], False)), pos, sampled, tries)[0] == L_ERR["SHAPE"]
    assert _run(emu, dict(tables, b=HostTable(np.zeros((n_ent, 2)), False)), pos, sampled, tries)[0] == L_ERR["SHAPE"]
    assert _run(emu, dict(tables, params=HostTable(tabs["params"][:3], False)), pos, sampled, tries)[0] == L_ERR["SHAPE"]
    assert _run(emu, tables, None, sampled, tries)[0] == 0                                # an empty batch is a no-op
    assert not any(t.grad.any() for t in tables.values())
    assert _sample(emu, 10, 11, 0)[0] == L_ERR["RANGE"]
    assert _sample(emu, 10, 0, 0)[0] == L_ERR["RANGE"]
    assert _sample(emu, 10, 5, 0, ws_bytes=39)[0] == L_ERR["WORKSPACE"]


L_ERR = {"NULL": 1, "DIM": 2, "SHAPE": 5, "RANGE": 6, "WORKSPACE": 7}
