"""CPU: the RotatE and HolE kernels of openea_b200/csrc/oea_triple_ext.cu executed on the warp emulator of tests/emu
against the float64 oracle of tests/semantic_ext_oracle.py, at sizes a CPU finishes in seconds: forward and backward
for both kinds, a source mutation the comparison must catch, the zero-modulus case of RotatE and the argument checks of
the new kinds."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

from openea_b200 import lib as L
from tests import semantic_ext_oracle as so
from tests.emu import build_emu
from tests.helpers import make_batch
from tests.test_emu_triple_ext import HostTable

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = {"RotatE": L.MODEL_ROTATE, "HolE": L.MODEL_HOLE}
GAMMA = 12.0


def _bind(lib):
    res, args = L.SIGNATURES["oea_model_score_fed"]
    lib.oea_model_score_fed.restype, lib.oea_model_score_fed.argtypes = res, args
    return lib


@pytest.fixture(scope="module")
def emu():
    so_path = build_emu.build()
    if so_path is None:
        pytest.skip("no CUDA headers for the emulator build")
    return _bind(C.CDLL(so_path))


def _case(model, seed, n_ent, n_rel, d, norm):
    rng = np.random.default_rng(seed)
    tabs, norms = {}, {}
    for i, s in enumerate(so.SLOTS[model]):
        rows = n_rel if s == "rel" else n_ent
        tabs[s] = (rng.standard_normal((rows, d)) * (0.6 + 0.3 * i) / np.sqrt(d)).astype(np.float32)
        norms[s] = norm
    return rng, tabs, norms


def _run(emu, model, tables, pos, neg, loss_kind, scale=1.0, gamma=GAMMA, margin=0.3, slots=None):
    slots = so.SLOTS[model] if slots is None else slots
    ptrs = [C.pointer(tables[s].struct) if s is not None else None for s in slots] + [None] * (4 - len(slots))
    d = next(iter(tables.values())).d
    phase = math.pi / ((gamma + 2.0) / d) if model == "RotatE" else 0.0
    m = L.Model(KINDS[model], *ptrs, gamma if model == "RotatE" else 0.0, phase)
    cfg = L.LossCfg(L.SCORE_L2SQ, loss_kind, margin, 0.0, 1.0)
    out = np.zeros(1, dtype=np.float64)
    i32 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.int32)
    p = [i32(pos[i]) if pos is not None else None for i in range(3)]
    n = [i32(neg[i]) if neg is not None else None for i in range(3)]
    vp = lambda a: C.c_void_p(0 if a is None else a.ctypes.data)
    rc = emu.oea_model_score_fed(C.byref(m), vp(p[0]), vp(p[1]), vp(p[2]), 0 if pos is None else pos.shape[1],
                                 vp(n[0]), vp(n[1]), vp(n[2]), 0 if neg is None else neg.shape[1], C.byref(cfg), scale,
                                 vp(out), None)
    return rc, float(out[0])


def _rotate(emu, tables, pos, neg, neg_weight):
    """RotatE's loss: the positives at weight 1, the negatives at neg_weight (two calls when it differs from 1)."""
    if neg_weight == 1.0:
        return _run(emu, "RotatE", tables, pos, neg, L.LOSS_LOGISTIC)
    rc1, a = _run(emu, "RotatE", tables, pos, None, L.LOSS_LOGISTIC)
    rc2, b = _run(emu, "RotatE", tables, None, neg, L.LOSS_LOGISTIC, scale=neg_weight)
    return max(rc1, rc2), a + b


def _check_grads(tables, want_g, d):
    for s, tab in tables.items():
        got, want = tab.grad[:, :d], want_g[s]
        np.testing.assert_allclose(got, want, rtol=1e-4, atol=2e-5 * max(1e-6, np.abs(want).max()), err_msg=s)
        assert not tab.grad[:, d:].any(), "padding columns must stay zero"
        assert (np.abs(want).sum(1)[tab.touched == 0] == 0).all(), "untouched rows must have zero oracle gradient"


@pytest.mark.parametrize("d", [12, 75, 200])
@pytest.mark.parametrize("norm", [True, False])
@pytest.mark.parametrize("k,neg_weight", [(3, 1.0 / 3), (3, 1.0), (1, 1.0)])
def test_emulated_rotate_matches_oracle(emu, d, norm, k, neg_weight):
    n_ent, n_rel, n_pos = 30, 5, 13
    rng, tabs, norms = _case("RotatE", 3 * d + k + int(norm), n_ent, n_rel, d, norm)
    pos, neg = make_batch(rng, n_ent, n_rel, n_pos, k)
    want_loss, want_g = so.fwd_bwd("RotatE", tabs, norms, pos, neg, gamma=GAMMA, neg_weight=neg_weight)
    tables = {s: HostTable(tabs[s], norms[s]) for s in so.SLOTS["RotatE"]}
    rc, got = _rotate(emu, tables, pos, neg, neg_weight)
    assert rc == 0
    assert got == pytest.approx(want_loss, rel=1e-4)
    _check_grads(tables, want_g, d)


def test_emulated_rotate_alignment_loss_is_the_positive_half(emu):
    """BootEA_RotatE's alignment loss −Σ log σ(γ − d) (bootea_rotate.py:153-158) is OEA_LOSS_LOGSIGMOID on positives."""
    rng, tabs, norms = _case("RotatE", 4, 30, 5, 20, True)
    pos, _ = make_batch(rng, 30, 5, 17, 0)
    want_loss, want_g = so.fwd_bwd("RotatE", tabs, norms, pos, None, gamma=GAMMA)
    tables = {s: HostTable(tabs[s], norms[s]) for s in so.SLOTS["RotatE"]}
    rc, got = _run(emu, "RotatE", tables, pos, None, L.LOSS_LOGSIGMOID)
    assert rc == 0 and got == pytest.approx(want_loss, rel=1e-4)
    _check_grads(tables, want_g, 20)


@pytest.mark.parametrize("d", [12, 75, 200])
@pytest.mark.parametrize("norm", [True, False])
@pytest.mark.parametrize("k", [1, 3])
def test_emulated_hole_matches_oracle(emu, d, norm, k):
    n_ent, n_rel, n_pos = 30, 5, 13
    rng, tabs, norms = _case("HolE", 5 * d + k + int(norm), n_ent, n_rel, d, norm)
    pos, neg = make_batch(rng, n_ent, n_rel, n_pos, k)
    margin = 0.3
    want_loss, want_g = so.fwd_bwd("HolE", tabs, norms, pos, neg, margin=margin)
    tables = {s: HostTable(tabs[s], norms[s]) for s in so.SLOTS["HolE"]}
    rc, got = _run(emu, "HolE", tables, pos, neg, L.LOSS_MARGIN, margin=margin)
    assert rc == 0
    assert got == pytest.approx(want_loss, rel=1e-4)
    _check_grads(tables, want_g, d)


def test_direct_correlation_equals_the_fft_form():
    """The O(d²) sum the kernel evaluates is the reference's real(ifft(conj(fft(a))·fft(b))), at odd and even d."""
    import torch
    rng = np.random.default_rng(1)
    for d in (1, 7, 75, 100):
        a, b = rng.standard_normal((4, d)), rng.standard_normal((4, d))
        want = so.ccorr(torch.as_tensor(a), torch.as_tensor(b)).numpy()
        np.testing.assert_allclose(so.ccorr_direct(a, b), want, rtol=1e-10, atol=1e-10)


def test_emulated_rotate_zero_modulus_is_finite(emu):
    """h = t with r = 0: every coordinate's modulus is 0.  TF's tf.norm gradient is NaN there; the engine takes it as 0,
    so loss and gradients stay finite (and the positive's own rows receive no gradient from the modulus)."""
    d = 16
    rng, tabs, norms = _case("RotatE", 9, 10, 3, d, True)
    tabs["rel"][1] = 0.0
    pos = np.array([[2, 4], [1, 1], [2, 4]], dtype=np.int32)
    neg = np.array([[3, 5], [0, 2], [2, 4]], dtype=np.int32)
    tables = {s: HostTable(tabs[s], norms[s]) for s in so.SLOTS["RotatE"]}
    rc, got = _run(emu, "RotatE", tables, pos, neg, L.LOSS_LOGISTIC)
    assert rc == 0
    assert np.isfinite(got)
    import torch
    tv = {k: torch.tensor(v, dtype=torch.float64) for k, v in tabs.items()}
    e_neg = so.rotate_distance(tv, norms, neg, GAMMA) - GAMMA
    want = 2 * math.log1p(math.exp(-GAMMA)) + float(torch.nn.functional.softplus(-e_neg).sum())
    assert got == pytest.approx(want, rel=1e-5)
    for tab in tables.values():
        assert np.isfinite(tab.grad).all()
    assert not tables["rel"].grad[1].any(), "r = 0 sees only zero moduli: no gradient"


def test_emulated_semantic_ext_argument_checks(emu):
    rng, tabs, norms = _case("RotatE", 1, 20, 4, 16, True)
    rt = {s: HostTable(tabs[s], norms[s]) for s in so.SLOTS["RotatE"]}
    pos, neg = make_batch(rng, 20, 4, 6, 2)
    rc, _ = _run(emu, "RotatE", rt, pos, neg, L.LOSS_MARGIN)
    assert rc == 4                                        # OEA_ERR_KIND: RotatE has no margin form
    rc, _ = _run(emu, "RotatE", rt, pos, neg, L.LOSS_LOGISTIC, slots=("re_ent", "rel"))
    assert rc == 1                                        # OEA_ERR_NULL: RotatE without its imaginary table
    _, htabs, hnorms = _case("HolE", 2, 20, 4, 16, True)
    ht = {s: HostTable(htabs[s], hnorms[s]) for s in so.SLOTS["HolE"]}
    rc, _ = _run(emu, "HolE", ht, pos, neg, L.LOSS_LOGISTIC)
    assert rc == 4                                        # OEA_ERR_KIND: HolE trains with the margin loss only
    rc, _ = _run(emu, "HolE", ht, pos, neg[:, :7], L.LOSS_MARGIN)
    assert rc == 5                                        # OEA_ERR_SHAPE: n_pos must divide n_neg
    rc, _ = _run(emu, "HolE", ht, pos, None, L.LOSS_MARGIN)
    assert rc == 5                                        # OEA_ERR_SHAPE: the margin loss needs negatives
    wide = {s: HostTable(np.zeros((t.weight.shape[0], 300), dtype=np.float32), True) for s, t in ht.items()}
    rc, _ = _run(emu, "HolE", wide, pos, neg, L.LOSS_MARGIN)
    assert rc == 2                                        # OEA_ERR_DIM: pitch > 256
    bad = L.Model(7, C.pointer(ht["ent"].struct), C.pointer(ht["rel"].struct), None, None, 0.0, 0.0)
    cfg = L.LossCfg(L.SCORE_L2SQ, L.LOSS_MARGIN, 0.2, 0.0, 1.0)
    out = np.zeros(1)
    assert emu.oea_model_score_fed(C.byref(bad), None, None, None, 0, None, None, None, 0, C.byref(cfg), 1.0,
                                   C.c_void_p(out.ctypes.data), None) == 4       # unknown kind


MUTATION = ("const float dth = fmaf(da, -fmaf(hr, sn, hi * cs), db * fmaf(hr, cs, -hi * sn));",
            "const float dth = fmaf(da, fmaf(hr, sn, hi * cs), db * fmaf(hr, cs, -hi * sn));")


def test_emulated_rotate_phase_backward_mutation_is_caught(tmp_path):
    """The comparison with the oracle has teeth: the kernel source with one sign flipped in the phase backward
    (dθ's first term), built for the emulator, must disagree with the oracle on the relation gradient."""
    inc = build_emu.cuda_include()
    if inc is None:
        pytest.skip("no CUDA headers for the emulator build")
    csrc = tmp_path / "openea_b200" / "csrc"
    shutil.copytree(os.path.join(ROOT, "openea_b200", "csrc"), csrc)
    shutil.copytree(os.path.join(ROOT, "include"), tmp_path / "include")
    (tmp_path / "tests" / "emu").mkdir(parents=True)
    shutil.copy(os.path.join(ROOT, "tests", "emu", "cuda_host_emu.h"), tmp_path / "tests" / "emu")
    src = (csrc / "oea_triple_ext.cu").read_text()
    assert src.count(MUTATION[0]) == 1, "the mutated statement is not in the kernel source any more"
    (csrc / "oea_triple_ext.cu").write_text(src.replace(MUTATION[0], MUTATION[1]))
    main = tmp_path / "tests" / "emu" / "mutant.cpp"
    main.write_text('#include "cuda_host_emu.h"\n#include "../../openea_b200/csrc/oea_triple_ext.cu"\n')
    out = tmp_path / "libmutant.so"
    cmd = ["g++", "-std=c++20", "-O1", "-pthread", "-fPIC", "-shared", "-DOEA_HOST_EMU", "-Wno-attributes",
           "-Wno-unknown-pragmas", "-I", inc, "-o", str(out), str(main),
           "-L", os.path.join(os.path.dirname(inc), "lib64"), "-lcudart"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    mutant = _bind(C.CDLL(str(out)))
    d = 20
    rng, tabs, norms = _case("RotatE", 12, 30, 5, d, True)
    pos, neg = make_batch(rng, 30, 5, 13, 3)
    _, want_g = so.fwd_bwd("RotatE", tabs, norms, pos, neg, gamma=GAMMA, neg_weight=1.0)
    tables = {s: HostTable(tabs[s], norms[s]) for s in so.SLOTS["RotatE"]}
    rc, _ = _rotate(mutant, tables, pos, neg, 1.0)
    assert rc == 0
    with pytest.raises(AssertionError):
        _check_grads(tables, want_g, d)
    # and the entity gradients, which do not pass through dθ, still agree
    for s in ("re_ent", "im_ent"):
        got, want = tables[s].grad[:, :d], want_g[s]
        np.testing.assert_allclose(got, want, rtol=1e-4, atol=2e-5 * np.abs(want).max())
