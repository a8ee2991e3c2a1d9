"""GPU: the edge cases of tests/test_emu_kernel_edges.py on the device — every row width of the VEC dispatch, degenerate
rows, odd positive counts — and batches of more than three resident waves of the H100 (multi_processor_count × 64
warps), with the float64 reference run on the GPU so that 10⁵-triple batches stay cheap.  The last test runs the
one-launch sampled step for the duo and the octet kernels in both orders in fresh processes: each kernel sizes its
cooperative grid from its own occupancy."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from openea_b200 import engine as eng
from openea_b200 import lib as L
from tests import kernel_edge_cases as kc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _wave(dev):
    """Warps in one resident wave: 64 per SM."""
    return torch.cuda.get_device_properties(dev).multi_processor_count * 64


@pytest.mark.parametrize("loss_norm", ["L2", "L1"])
@pytest.mark.parametrize("d", kc.DIMS)
def test_fed_scorers_at_every_width(cuda_device, d, loss_norm):
    for loss, k in kc.LOSSES:
        kc.check_fed(eng, cuda_device, d, loss_norm, loss, k, seed=d + k)
        kc.check_fed(eng, cuda_device, d, loss_norm, loss, k, seed=d + k, grouped=True)
    if loss_norm == "L2" and d <= 128:                  # k_score_fed_grouped: k = 17 is past the duo
        for loss in ("limited", "logistic"):
            kc.check_fed(eng, cuda_device, d, loss_norm, loss, 17, seed=d + 17, grouped=True)
    scale = 6.0 if loss_norm == "L2" else 70.0 / np.sqrt(d)
    for loss, k in (("logistic", 2), ("logsigmoid", 0)):
        for grouped in (False, True):
            scores = kc.check_fed(eng, cuda_device, d, loss_norm, loss, k, norm=False, scale=scale, seed=d, grouped=grouped)
            assert scores.max() > 50.0


@pytest.mark.parametrize("d", [1, 128, 512])
def test_l1_zero_residual_contributes_exactly_nothing(cuda_device, d):
    for grouped in (False, True):
        kc.check_zero_u_contributes_nothing(eng, cuda_device, d, grouped)


@pytest.mark.parametrize("n_pos", [1, 2, 3, 33])
@pytest.mark.parametrize("d", [4, 128])
def test_duo_scorers_take_the_unpaired_last_positive(cuda_device, d, n_pos):
    for loss, k in (("limited", 3), ("margin-based", 1), ("positive", 0)):
        kc.check_fed(eng, cuda_device, d, "L2", loss, k, n_pos=n_pos, grouped=True, seed=n_pos)
    kc.check_sampled(eng, cuda_device, d, "L2", "limited", 5, n_pos, seed=n_pos, ref_dev=cuda_device)


def test_fed_scorers_past_three_waves(cuda_device):
    wave = _wave(cuda_device)
    big = dict(hot=0.25, n_ent=20000, n_rel=40, ref_dev=cuda_device)
    for d, loss_norm, loss, k in ((100, "L2", "limited", 2), (129, "L1", "logistic", 2), (512, "L2", "logistic", 1)):
        n_pos = 3 * wave + 7
        assert n_pos * (1 + k) > 3 * wave                                          # oea_triple_score_fed: a warp per triple
        kc.check_fed(eng, cuda_device, d, loss_norm, loss, k, n_pos=n_pos, seed=d, **big)
    n_pos = 6 * wave + 1
    assert (n_pos + 1) // 2 > 3 * wave                                             # duo: two positives per warp
    kc.check_fed(eng, cuda_device, 100, "L2", "limited", 10, n_pos=n_pos, grouped=True, seed=5, **big)
    n_pos = 3 * wave + 5
    kc.check_fed(eng, cuda_device, 200, "L1", "margin-based", 1, n_pos=n_pos, grouped=True, seed=6, **big)
    kc.check_fed(eng, cuda_device, 384, "L2", "limited", 3, n_pos=n_pos, grouped=True, seed=7, **big)


@pytest.mark.parametrize("opt", ["Adagrad", "SGD"])
def test_one_launch_fed_step_past_three_waves(cuda_device, opt):
    wave = _wave(cuda_device)
    kc.check_step_fed_grouped(eng, cuda_device, 100, opt, n_pos=6 * wave + 1, k=10, seed=1, ref_dev=cuda_device, hot=0.25,
                              n_ent=20000)
    kc.check_step_fed_grouped(eng, cuda_device, 200, opt, n_pos=3 * wave + 5, k=3, seed=2, ref_dev=cuda_device, hot=0.25,
                              n_ent=20000)


def test_sampled_scorers_past_three_waves(cuda_device):
    wave = _wave(cuda_device)
    big = dict(n_tri=14 * wave, n=20000, ref_dev=cuda_device)       # step 1 starts past the first batch
    m = kc.check_sampled(eng, cuda_device, 100, "L2", "limited", 10, 6 * wave + 200, seed=1, **big)      # duo
    assert (m + 1) // 2 > 3 * wave
    m = kc.check_sampled(eng, cuda_device, 100, "L2", "limited", 20, 3 * wave + 200, seed=2, **big)      # octet: k > 16
    assert m > 3 * wave
    m = kc.check_sampled(eng, cuda_device, 300, "L1", "limited", 4, 3 * wave + 200, seed=3, **big)       # warp per positive
    assert m > 3 * wave


@pytest.mark.parametrize("opt", ["Adagrad", "SGD"])
@pytest.mark.parametrize("d", [3, 4, 128, 129, 256])
def test_one_launch_fed_step_equals_dense_steps(cuda_device, d, opt):
    kc.check_step_fed_grouped(eng, cuda_device, d, opt, seed=d)
    kc.check_step_fed_grouped(eng, cuda_device, d, opt, loss="margin-based", k=1, seed=d + 1)


@pytest.mark.parametrize("variant,d,loss_norm,loss,k", [
    ("duo", 1, "L2", "limited", 6), ("duo", 4, "L2", "margin-based", 1), ("duo", 127, "L2", "logistic", 3),
    ("duo", 128, "L2", "limited", 16), ("oct", 3, "L2", "limited", 20), ("oct", 128, "L2", "logistic", 17),
    ("v1", 129, "L1", "limited", 3), ("v1", 256, "L2", "logistic", 2), ("v1", 257, "L1", "margin-based", 1),
    ("v1", 384, "L2", "limited", 3), ("v1", 385, "L1", "logistic", 2), ("v1", 512, "L1", "limited", 3),
    ("v1", 512, "L2", "positive", 0)])
def test_sampled_scorers_replay_through_the_reference(cuda_device, variant, d, loss_norm, loss, k):
    kc.check_sampled(eng, cuda_device, d, loss_norm, loss, k, 33, seed=d + k)


@pytest.mark.parametrize("d", [1, 128, 129, 257, 512])
def test_weighted_margin_and_pair_losses(cuda_device, d):
    for loss_norm in ("L2", "L1"):
        for paths in (False, True):
            kc.check_margin_weighted(eng, cuda_device, d, loss_norm, paths)
    kc.check_pairs(eng, cuda_device, d)


@pytest.mark.parametrize("d", kc.EXT_DIMS)
@pytest.mark.parametrize("model,loss,k,loss_norm", kc.EXT_CASES)
def test_model_scorers_at_every_width(cuda_device, model, loss, k, loss_norm, d):
    kc.check_ext(eng, cuda_device, model, loss, k, loss_norm, d)


@pytest.mark.parametrize("model", ["TransH", "TransD", "DistMult", "SimplE", "RotatE", "HolE"])
def test_model_scorers_refuse_pitch_above_256(cuda_device, model):
    with pytest.raises(L.OeaError, match="rc=2 "):                             # OEA_ERR_DIM
        kc.check_ext(eng, cuda_device, model, *{"RotatE": ("logistic", 1, "L2"), "HolE": ("margin-based", 1, "L2")}.get(
            model, ("margin-based", 1, "L2")), 257)


@pytest.mark.parametrize("d", [1, 33, 512])
def test_lookup_scatter_and_mapping(cuda_device, d):
    kc.check_lookup_scatter(eng, cuda_device, d)
    kc.check_mapping(eng, cuda_device, d)


@pytest.mark.parametrize("opt", ["Adagrad", "SGD", "Adam", "Adadelta"])
@pytest.mark.parametrize("d", [1, 33, 512])
def test_optimisers_at_every_width(cuda_device, d, opt):
    kc.check_apply(eng, cuda_device, d, opt)


# The one-launch sampled step of the duo kernel (k <= 16) and of the octet kernel (k > 16), in the order given, each
# against the two-launch path (the same scorer, then the row optimiser) on the same batch.  A batch of 20 000 positives is more than three duo
# waves of pairs at 5 CTAs × 4 warps on 132 SMs (7 920 pairs).
ORDER_SCRIPT = r"""
import sys
import numpy as np, torch
from openea_b200 import engine as eng
from tests import kernel_edge_cases as kc
order, opt = sys.argv[1].split("-then-"), sys.argv[2]
rng = np.random.default_rng(0)
ent, rel, t1, t2, kg1, kg2, tset = kc.sampled_setup(eng, "cuda", rng, 40000, 20000, 40, 100, edge=False)
make = lambda: eng.TripleTrainer(*kc._tables(eng, "cuda", ent, rel, True, opt), eng.loss_cfg("limited", "L2", 0.3, 2.2, 0.2), 0.01)
for kind in order:
    k = 10 if kind == "duo" else 20
    fused, split = make(), make()
    n_pos = torch.zeros(1, dtype=torch.int32, device="cuda")
    fused.step_sampled(kg1, kg2, tset, 20000, k, 0, 99, n_pos_out=n_pos)
    split.score_sampled(kg1, kg2, tset, 20000, k, 0, 99)
    split.apply()
    torch.cuda.synchronize()
    assert int(n_pos.item()) == 20000
    assert abs(fused.read_loss() - split.read_loss()) <= 1e-5 * abs(split.read_loss()), kind
    for a, b in ((fused.ent, split.ent), (fused.rel, split.rel)):
        np.testing.assert_allclose(a.raw().cpu().numpy(), b.raw().cpu().numpy(), rtol=1e-4, atol=1e-6, err_msg=kind)
        if opt == "Adagrad":
            np.testing.assert_allclose(a.state1.cpu().numpy(), b.state1.cpu().numpy(), rtol=1e-4, atol=1e-6, err_msg=kind)
        assert not a.grad.any() and not a.touched.any()
print("ok")
"""


@pytest.mark.parametrize("opt", ["Adagrad", "SGD"])
@pytest.mark.parametrize("order", ["oct-then-duo", "duo-then-oct"])
def test_one_launch_sampled_steps_in_either_order(cuda_device, order, opt):
    """The duo and octet one-launch steps have the same parameter list but different launch bounds (5 against 6 CTAs
    of 4 warps): whichever runs first in a process must not fix the cooperative grid of the other."""
    res = subprocess.run([sys.executable, "-c", ORDER_SCRIPT, order, opt], cwd=ROOT, capture_output=True, text=True,
                         timeout=600)
    assert res.returncode == 0 and res.stdout.strip().endswith("ok"), res.stdout[-2000:] + res.stderr[-4000:]
