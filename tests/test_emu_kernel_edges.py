"""CPU: the path-(i) kernels at the edges of what they accept — every row width of the VEC dispatch (VEC = 1 … 4 and each
pitch-bucket edge), batches longer than one resident wave, odd positive counts for the two-positives-per-warp kernels,
and degenerate rows (zero and sub-eps rows, self-loops, negatives equal to their positive, an exactly zero L1 residual,
scores near 100 for the softplus losses) — executed from the product's kernel source on the warp emulator (tests/emu)
through the product's own host layer, against float64 references.  tests/test_zz_kernel_edges_gpu.py runs the same
cases on the GPU."""
import ctypes as C

import numpy as np
import pytest

from openea_b200 import engine as eng
from openea_b200 import lib as L
from tests import kernel_edge_cases as kc
from tests.emu import build_emu


@pytest.fixture()
def cpu_engine(monkeypatch):
    lib = build_emu.load()
    build_emu.patch_engine(monkeypatch, lib)
    return eng, lib


def _wave(lib, warps_per_block):
    """Warps in one resident wave on the emulator.  Without a device, cudaGetDevice fails, so sm_count_cached() falls
    back to 132 SMs and grid_one_wave's occupancy query to 1 CTA per SM: a grid_one_wave kernel's wave is
    132 × warps-per-block warps; grid_for caps at 132 × 8 CTAs of 8 warps, as on the H100."""
    dev = C.c_int(0)
    assert lib.cudaGetDevice(C.byref(dev)) != 0, "a CUDA device is visible: the emulator's wave is not the fallback's"
    return 132 * warps_per_block


@pytest.mark.parametrize("loss_norm", ["L2", "L1"])
@pytest.mark.parametrize("d", kc.DIMS)
def test_emulated_fed_scorers_at_every_width(cpu_engine, d, loss_norm):
    """oea_triple_score_fed and oea_triple_score_fed_grouped (duo at pitch <= 128 for L2 and k <= 16, the
    warp-per-positive kernel otherwise: at L2 and pitch <= 128 with k = 17), all five losses, edge rows in every batch."""
    e, _ = cpu_engine
    for loss, k in kc.LOSSES:
        kc.check_fed(e, "cpu", d, loss_norm, loss, k, seed=d + k)
        kc.check_fed(e, "cpu", d, loss_norm, loss, k, seed=d + k, grouped=True)
    if loss_norm == "L2" and d <= 128:
        for loss in ("limited", "logistic"):
            kc.check_fed(e, "cpu", d, loss_norm, loss, 17, seed=d + 17, grouped=True)
    # unnormalised tables scaled so that the scores reach ~100: softplus / sigmoid far from 0
    scale = 6.0 if loss_norm == "L2" else 70.0 / np.sqrt(d)
    for loss, k in (("logistic", 2), ("logsigmoid", 0)):
        for grouped in (False, True):
            scores = kc.check_fed(e, "cpu", d, loss_norm, loss, k, norm=False, scale=scale, seed=d, grouped=grouped)
            assert scores.max() > 50.0


@pytest.mark.parametrize("d", [1, 128, 512])
def test_emulated_l1_zero_residual_contributes_exactly_nothing(cpu_engine, d):
    for grouped in (False, True):
        kc.check_zero_u_contributes_nothing(cpu_engine[0], "cpu", d, grouped)


@pytest.mark.parametrize("n_pos", [1, 2, 3, 33])
@pytest.mark.parametrize("d", [4, 128])
def test_emulated_duo_scorers_take_the_unpaired_last_positive(cpu_engine, d, n_pos):
    """Odd positive counts leave half a warp idle in the duo kernels: the last positive must still be scored."""
    e, _ = cpu_engine
    for loss, k in (("limited", 3), ("margin-based", 1), ("positive", 0)):
        kc.check_fed(e, "cpu", d, "L2", loss, k, n_pos=n_pos, grouped=True, seed=n_pos)
    if d <= 128:
        kc.check_sampled(e, "cpu", d, "L2", "limited", 5, n_pos, seed=n_pos)


def test_emulated_fed_scorers_past_one_wave(cpu_engine):
    """Three waves and more: the grid-stride loops' later iterations, the duo kernel's per-warp staging reused across
    them and the loss carried in fp32 across iterations; one entity in a quarter of the triples."""
    e, lib = cpu_engine
    wave = _wave(lib, 8)
    for d, loss_norm, loss, k in ((4, "L2", "limited", 2), (129, "L1", "logistic", 2)):
        n_pos = 1100
        assert n_pos * (1 + k) > 3 * wave                                         # oea_triple_score_fed: a warp per triple
        kc.check_fed(e, "cpu", d, loss_norm, loss, k, n_pos=n_pos, hot=0.25, n_ent=400, n_rel=20, seed=d)
    n_pos = 3201
    assert (n_pos + 1) // 2 > 3 * _wave(lib, 4)                                   # k_score_fed_duo: two positives per warp
    kc.check_fed(e, "cpu", 128, "L2", "limited", 2, n_pos=n_pos, grouped=True, hot=0.25, n_ent=400, n_rel=20, seed=5)
    n_pos = 3 * 132 * 64 + 5
    assert n_pos > 3 * 132 * 64                                                   # grid_for: 132 × 8 CTAs × 8 warps
    kc.check_fed(e, "cpu", 4, "L1", "margin-based", 1, n_pos=n_pos, grouped=True, hot=0.25, n_ent=2000, n_rel=20, seed=6)


def test_emulated_sampled_scorers_past_one_wave(cpu_engine):
    e, lib = cpu_engine
    m = kc.check_sampled(e, "cpu", 12, "L2", "limited", 2, 3300, n_tri=7000, n=900, seed=1)        # duo
    assert (m + 1) // 2 > 3 * _wave(lib, 4)
    m = kc.check_sampled(e, "cpu", 12, "L2", "limited", 20, 1700, n_tri=4000, n=900, seed=2)       # octet: k > 16
    assert m > 3 * _wave(lib, 4)
    m = kc.check_sampled(e, "cpu", 129, "L1", "limited", 2, 3300, n_tri=7000, n=900, seed=3)       # warp per positive
    assert m > 3 * _wave(lib, 8)


@pytest.mark.parametrize("opt", ["Adagrad", "SGD"])
@pytest.mark.parametrize("d", [3, 4, 128, 129, 256])
def test_emulated_one_launch_fed_step_equals_dense_steps(cpu_engine, d, opt):
    kc.check_step_fed_grouped(cpu_engine[0], "cpu", d, opt, seed=d)
    kc.check_step_fed_grouped(cpu_engine[0], "cpu", d, opt, loss="margin-based", k=1, seed=d + 1)


@pytest.mark.parametrize("variant,d,loss_norm,loss,k", [
    ("duo", 1, "L2", "limited", 6), ("duo", 4, "L2", "margin-based", 1), ("duo", 127, "L2", "logistic", 3),
    ("duo", 128, "L2", "limited", 16), ("oct", 3, "L2", "limited", 20), ("oct", 128, "L2", "logistic", 17),
    ("v1", 129, "L1", "limited", 3), ("v1", 256, "L2", "logistic", 2), ("v1", 257, "L1", "margin-based", 1),
    ("v1", 384, "L2", "limited", 3), ("v1", 385, "L1", "logistic", 2), ("v1", 512, "L1", "limited", 3),
    ("v1", 512, "L2", "positive", 0)])
def test_emulated_sampled_scorers_replay_through_the_reference(cpu_engine, variant, d, loss_norm, loss, k):
    """The sampled kernels' debug dump, decoded, scored by the float64 reference: same loss and gradients.  `variant`
    names the kernel the shape reaches: duo, oct or v1 (k_score_sampled, one warp per positive)."""
    kc.check_sampled(cpu_engine[0], "cpu", d, loss_norm, loss, k, 33, seed=d + k)


@pytest.mark.parametrize("d", [1, 128, 129, 257, 512])
def test_emulated_weighted_margin_and_pair_losses(cpu_engine, d):
    for loss_norm in ("L2", "L1"):
        for paths in (False, True):
            kc.check_margin_weighted(cpu_engine[0], "cpu", d, loss_norm, paths)
    kc.check_pairs(cpu_engine[0], "cpu", d)


@pytest.mark.parametrize("d", kc.EXT_DIMS)
@pytest.mark.parametrize("model,loss,k,loss_norm", kc.EXT_CASES)
def test_emulated_model_scorers_at_every_width(cpu_engine, model, loss, k, loss_norm, d):
    kc.check_ext(cpu_engine[0], "cpu", model, loss, k, loss_norm, d)


@pytest.mark.parametrize("model", ["TransH", "TransD", "DistMult", "SimplE", "RotatE", "HolE"])
def test_emulated_model_scorers_refuse_pitch_above_256(cpu_engine, model):
    e, _ = cpu_engine
    with pytest.raises(L.OeaError, match="rc=2 "):                             # OEA_ERR_DIM
        kc.check_ext(e, "cpu", model, *{"RotatE": ("logistic", 1, "L2"), "HolE": ("margin-based", 1, "L2")}.get(
            model, ("margin-based", 1, "L2")), 257)


@pytest.mark.parametrize("d", [1, 33, 512])
def test_emulated_lookup_scatter_and_mapping(cpu_engine, d):
    kc.check_lookup_scatter(cpu_engine[0], "cpu", d)
    kc.check_mapping(cpu_engine[0], "cpu", d)


@pytest.mark.parametrize("opt", ["Adagrad", "SGD", "Adam", "Adadelta"])
@pytest.mark.parametrize("d", [1, 33, 512])
def test_emulated_optimisers_at_every_width(cpu_engine, d, opt):
    kc.check_apply(cpu_engine[0], "cpu", d, opt)
