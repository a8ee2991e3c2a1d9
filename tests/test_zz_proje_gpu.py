"""GPU tests of ProjE (oea_logu_sample_unique, oea_proje_score_fed) through the engine: the device sampler against the
sequential loop over the same draw stream at E = 30 000 and 200 000 with S = 4 096; a batch at the 15K shape (B = 500,
S = 4 096, E = 30 000) and one at the 100K shape (B = 5 000, E = 200 000) against float64 computed on the device; whole
Adam steps on the five tables against dense float64 steps; the lifecycle on the tiny synthetic KG; and checkpoint →
resume."""
import contextlib
import io
import math
import os

import numpy as np
import pytest
import torch

from tests import proje_oracle as po
from tests.test_zz_triple_ext_gpu import tiny_kgs, _lifecycle, _losses        # noqa: F401  (fixture + helpers)

pytestmark = pytest.mark.gpu

NAMES = ("ent", "rel", "w", "b", "params")
NORMS = {"ent": True, "rel": True}


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


def _trainer(tabs, num_sampled, lr=0.01):
    from openea_b200 import engine as eng
    tables = {k: eng.EmbeddingTable(v, NORMS.get(k, False), "Adam") for k, v in tabs.items()}
    return eng.ProjETrainer(tuple(tables[k] for k in NAMES), num_sampled, lr), tables


def _batch(rng, n_ent, n_rel, n):
    return np.stack([rng.integers(0, n_ent, n), rng.integers(0, n_rel, n), rng.integers(0, n_ent, n)]).astype(np.int32)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).cuda()


def _grads(tables):
    return {k: t.grad[:, :t.dim].double().cpu().numpy() for k, t in tables.items()}


def _assert_close(got, want, what, rtol=2e-4):
    want = want.reshape(got.shape)
    np.testing.assert_allclose(got, want, rtol=rtol, atol=2e-4 * max(1e-6, np.abs(want).max()), err_msg=what)


@pytest.mark.parametrize("n_classes", [30000, 200000])
def test_device_sampler_is_the_sequential_loop(cuda_device, n_classes):
    _, tabs = _case(0, n_classes, 3, 8)
    tr, _ = _trainer(tabs, 4096)
    for seed in (1, 2 ** 40 + 17):
        tr.sample(seed)
        want, tries = po.sample_unique(seed, n_classes, 4096)
        assert np.array_equal(tr.sampled.cpu().numpy(), want)
        assert int(tr.num_tries.item()) == tries


def _fed_batch_against_float64(n_ent, n_rel, d, n_pos, S, seed):
    rng, tabs = _case(seed, n_ent, n_rel, d)
    pos = _batch(rng, n_ent, n_rel, n_pos)
    tr, tables = _trainer(tabs, S)
    tr.sample(seed + 5)
    sampled, tries = tr.sampled.cpu().numpy(), int(tr.num_tries.item())
    tr.score_fed(_dev(pos))
    got_loss = tr.read_loss()
    want_loss, want_g = po.fwd_bwd(tabs, NORMS, pos, sampled, tries, device="cuda")      # float64 on the device
    assert got_loss == pytest.approx(want_loss, rel=2e-5)
    got = _grads(tables)
    for k in NAMES:
        _assert_close(got[k], want_g[k], k)


def test_15k_shape_batch_matches_float64_on_the_device(cuda_device):
    _fed_batch_against_float64(30000, 600, 100, 500, 4096, 15)


def test_100k_shape_batch_matches_float64_on_the_device(cuda_device):
    _fed_batch_against_float64(200000, 1000, 100, 5000, 4096, 100)


def test_adam_steps_equal_dense_float64_steps(cuda_device):
    n_ent, n_rel, d, lr = 300, 9, 75, 0.01
    rng, tabs = _case(3, n_ent, n_rel, d)
    tr, tables = _trainer(tabs, 64, lr)
    st = po.DenseState(tabs, "Adam")
    for step in range(4):
        pos = _batch(rng, n_ent, n_rel, 37)
        tr.sample(100 + step)
        sampled, tries = tr.sampled.cpu().numpy(), int(tr.num_tries.item())
        _, want_g = po.fwd_bwd(st.w, NORMS, pos, sampled, tries)
        want = po.step(st, NORMS, pos, sampled, tries, lr)
        tr.score_fed(_dev(pos))
        got_g = _grads(tables)                  # every gradient at fp32 accuracy before Adam sees it
        for k in NAMES:
            _assert_close(got_g[k], want_g[k], k)
        tr.apply()
        assert tr.read_loss() == pytest.approx(want, rel=2e-5)
    for k, tab in tables.items():
        got, want = tab.raw().cpu().numpy(), st.w[k].reshape(tab.rows, -1)
        if k == "params":       # mlp_bias and the input beta: gradient 0 up to rounding, Adam steps of up to lr
            assert np.abs(got[1:3] - want[1:3]).max() <= 2 * 4 * lr
            got, want = got[[0, 3]], want[[0, 3]]
        # Adam's early steps are ±lr for any element whose gradient is tiny, whatever its size: an element whose fp32
        # gradient is within rounding of 0 may step the other way than in float64 (one in 10⁴ here, on the device's
        # atomic summation order).  Everything else agrees to fp32 accuracy.
        close = np.isclose(got, want, rtol=1e-4, atol=5e-6)
        assert close.mean() > 0.999 and np.abs(got - want).max() <= 2 * 4 * lr, k


def test_proje_lifecycle(cuda_device, tiny_kgs, tmp_path):
    """set_args / set_kgs / init / run / test / save with presets.proje on the tiny synthetic KG: the loss falls and
    stays finite, and the reference's result lines and files appear."""
    from openea_b200 import presets
    from openea_b200.models.neural import ProjE
    args = presets.proje()
    args.batch_size, args.max_epoch, args.start_valid, args.dim, args.dnn_neg_nums = 500, 30, 1000, 32, 256
    args.learning_rate = 0.01
    model, out = _lifecycle(ProjE, args, tiny_kgs, "sharing", tmp_path)
    loss = _losses(out, "avg. triple loss:")
    assert len(loss) == 30 and np.isfinite(loss).all()
    assert loss[-1] < 0.8 * loss[0], (loss[0], loss[-1])
    assert "Training ends. Total time" in out
    for f in ("ent_embeds.npy", "rel_embeds.npy", "alignment_results_12"):
        assert os.path.exists(model.out_folder + f), f


def test_proje_resume_from_checkpoint_continues_the_same_run(cuda_device, tiny_kgs, tmp_path):
    """6 epochs in one go == 3 epochs, checkpoint, a NEW model restored from the file, 3 more epochs: all five tables
    and their Adam slots.  Gradient sums are atomics, so agreement is to fp32 accumulation noise, not bit-wise."""
    from openea_b200 import presets
    from openea_b200.models.neural import ProjE
    from openea_b200.modules.base import initializers
    from openea_b200.modules.load.kgs import read_kgs_from_folder

    def make(max_epoch, out, **extra):
        args = presets.proje()
        args.training_data, args.output = tiny_kgs, str(tmp_path) + "/" + out + "/"
        args.batch_size, args.max_epoch, args.start_valid, args.dim, args.dnn_neg_nums = 500, max_epoch, 1000, 32, 128
        for k, v in extra.items():
            setattr(args, k, v)
        initializers.set_seed(77)
        m = ProjE()
        m.set_args(args)
        m.set_kgs(read_kgs_from_folder(tiny_kgs, args.dataset_division, "sharing", True))
        m.init()
        m._epoch_seed = 424242
        return m
    with contextlib.redirect_stdout(io.StringIO()):
        straight = make(6, "a")
        straight.run()
        first = make(3, "b", checkpoint_every=3)
        first.run()
        resumed = make(6, "c")
        assert {"entity_w", "entity_b", "proje_params"} <= set(resumed._checkpoint_tables())
        assert resumed.load_checkpoint(first.out_folder + "checkpoint.pt") == 4
        resumed.run()
    for name in ("ent_embeds", "rel_embeds", "entity_w", "entity_b", "proje_params"):
        a, b = getattr(straight, name), getattr(resumed, name)
        # mlp_bias and the input beta (params rows 1, 2) have a zero gradient up to rounding, which Adam amplifies and
        # which the output batch norm cancels: only the other rows are determined by the run
        rows = [0, 3] if name == "proje_params" else slice(None)
        for what, x, y in (("weight", a.raw(), b.raw()), ("m", a.state1, b.state1)):
            want = x[rows].cpu().numpy()
            np.testing.assert_allclose(y[rows].cpu().numpy(), want, rtol=2e-3, atol=2e-4 * max(1.0, np.abs(want).max()),
                                       err_msg=name + " " + what)
        assert a.adam_t == b.adam_t
    assert resumed._epoch_seed == straight._epoch_seed
