"""GPU tests of TransR (oea_transr_score_fed) through the engine, against the float64 oracle of tests/transr_oracle.py on
identical fed batches: forward and backward at d = 75, 100 and 128; whole Adagrad / Adam / SGD steps against dense
float64 steps; a 15K-shape batch (5 000 positives over ≈ 450 relations with Zipf frequencies, so that hub relations are
split into several chunks) against float64 computed on the device; the lifecycle on the tiny synthetic KG; and
checkpoint → resume.  The reference graph goldens replay through liboea.so in tests/test_transr_goldens.py."""
import contextlib
import io
import os

import numpy as np
import pytest
import torch

from tests import transr_oracle as tro
from tests.helpers import make_batch
from tests.test_zz_triple_ext_gpu import tiny_kgs, _lifecycle, _losses        # noqa: F401  (fixture + helpers)

pytestmark = pytest.mark.gpu


def _dev(hrt):
    return None if hrt is None else torch.from_numpy(np.ascontiguousarray(hrt.astype(np.int32))).cuda()


def _case(seed, n_ent, n_rel, d, norm=True):
    rng = np.random.default_rng(seed)
    tabs = {"ent": (rng.standard_normal((n_ent, d)) * 0.6 / np.sqrt(d)).astype(np.float32),
            "rel": (rng.standard_normal((n_rel, d)) * 0.9 / np.sqrt(d)).astype(np.float32),
            "mat": (rng.standard_normal((n_rel * d, d)) / d).astype(np.float32)}
    return rng, tabs, {"ent": norm, "rel": norm}


def _trainer(tabs, norms, opt, loss="margin-based", loss_norm="L2", lr=0.01, **kw):
    from openea_b200 import engine as eng
    tables = {"ent": eng.EmbeddingTable(tabs["ent"], norms["ent"], opt),
              "rel": eng.EmbeddingTable(tabs["rel"], norms["rel"], opt),
              "mat": eng.EmbeddingTable(tabs["mat"], False, opt)}
    tr = eng.ModelTrainer("TransR", (tables["ent"], tables["rel"], None, tables["mat"]),
                          eng.loss_cfg(loss, loss_norm, **kw), lr)
    return tr, tables


def _assert_rows_close(got, want, what):
    scale = max(1e-6, float(np.abs(want).max()))
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=2e-5 * scale, err_msg=what)


def _mixed_negatives(rng, neg, n_rel):
    neg = neg.copy()
    flip = rng.random(neg.shape[1]) < 0.3
    neg[1, flip] = rng.integers(0, n_rel, int(flip.sum()))
    return neg


@pytest.mark.parametrize("d", [75, 100, 128])
@pytest.mark.parametrize("loss,loss_norm,k,norm", [("margin-based", "L2", 1, True), ("limited", "L1", 3, True),
                                                   ("logistic", "L2", 2, False)])
def test_forward_backward_matches_oracle(cuda_device, d, loss, loss_norm, k, norm):
    n_ent, n_rel, n_pos = 1500, 29, 300
    rng, tabs, norms = _case(7 * d + k + len(loss), n_ent, n_rel, d, norm)
    pos, neg = make_batch(rng, n_ent, n_rel, n_pos, k)
    neg = _mixed_negatives(rng, neg, n_rel)
    kw = {"margin-based": dict(margin=1.0), "limited": dict(margin=0.2, neg_margin=1.5, balance=0.3), "logistic": {}}[loss]
    want_loss, want_g = tro.fwd_bwd(tabs, norms, pos, neg, loss, loss_norm, **kw)
    tr, tables = _trainer(tabs, norms, "Adagrad", loss, loss_norm, **kw)
    tr.score_fed(_dev(pos), _dev(neg))
    assert tr.read_loss() == pytest.approx(want_loss, rel=1e-4)
    for s, tab in tables.items():
        _assert_rows_close(tab.grad[:, :d].cpu().numpy(), want_g[s], "%s gradient" % s)
        assert not tab.grad[:, d:].any().item(), "padding columns must stay zero"
        touched = tab.touched.cpu().numpy().astype(bool)
        assert (np.abs(want_g[s]).sum(1)[~touched] == 0).all(), "untouched rows must have zero oracle gradient"


@pytest.mark.parametrize("opt", ["Adagrad", "Adam", "SGD"])
def test_training_steps_equal_dense_float64_steps(cuda_device, opt):
    """Three whole steps (scorer + row optimiser on the three tables) equal the oracle's dense TF-style float64 steps."""
    d, n_ent, n_rel, lr = 100, 1200, 23, 0.01
    rng, tabs, norms = _case(31 + len(opt), n_ent, n_rel, d)
    st = tro.DenseState(tabs, opt)
    tr, tables = _trainer(tabs, norms, opt, lr=lr, margin=1.0)
    for it in range(3):
        pos, neg = make_batch(rng, n_ent, n_rel, 300, 1)
        want = tro.step(st, norms, pos, neg, "margin-based", lr, margin=1.0)
        tr.score_fed(_dev(pos), _dev(neg))
        tr.apply()
        assert tr.read_loss() == pytest.approx(want, rel=1e-4), it
    for s, tab in tables.items():
        got, want = tab.raw().cpu().numpy(), st.w[s]
        start = tabs[s].astype(np.float64)
        if opt == "Adam":     # Adam moves a coordinate whose gradient is ≈ 0 by up to lr in either direction
            move_ok = np.isclose(got - start, want - start, rtol=5e-3, atol=1e-6 + 2e-3 * np.abs(want - start).max())
            val_ok = np.isclose(got, want, rtol=1e-4, atol=2e-5 * max(1e-6, float(np.abs(want).max())))
            assert (move_ok & val_ok).mean() > 0.999, (s, (move_ok & val_ok).mean())
            assert np.abs(got - want).max() <= 3 * lr * 1.01, s
        else:
            np.testing.assert_allclose(got - start, want - start, rtol=5e-3,
                                       atol=1e-6 + 2e-3 * np.abs(want - start).max(), err_msg=s)
            _assert_rows_close(got, want, "%s after 3 steps" % s)
        assert not tab.grad.any().item() and not tab.touched.any().item()


def test_15k_shape_batch_matches_float64_on_the_device(cuda_device):
    """5 000 positives and 5 000 negatives over 450 relations drawn with Zipf frequencies (the largest relation holds
    several chunks' worth of triples), d = 100, the shipped margin loss: loss and every gradient against float64."""
    d, n_ent, n_rel, n_pos = 100, 15000, 450, 5000
    rng, tabs, norms = _case(2024, n_ent, n_rel, d)
    p = 1.0 / np.arange(1, n_rel + 1) ** 1.1
    rel = rng.choice(n_rel, size=n_pos, p=p / p.sum())
    pos = np.stack([rng.integers(0, n_ent, n_pos), rel, rng.integers(0, n_ent, n_pos)]).astype(np.int32)
    neg = pos.copy()
    side = rng.random(n_pos) < 0.5
    neg[0, side] = rng.integers(0, n_ent, int(side.sum()))
    neg[2, ~side] = rng.integers(0, n_ent, int((~side).sum()))
    counts = np.bincount(rel, minlength=n_rel)
    assert counts.max() > 8 * 64 and (counts == 0).any()
    want_loss, want_g = tro.fwd_bwd(tabs, norms, pos, neg, "margin-based", "L2", margin=1.5, device="cuda")
    tr, tables = _trainer(tabs, norms, "Adagrad", margin=1.5)
    tr.score_fed(_dev(pos), _dev(neg))
    assert tr.read_loss() == pytest.approx(want_loss, rel=1e-4)
    for s, tab in tables.items():
        _assert_rows_close(tab.grad[:, :d].cpu().numpy(), want_g[s], "%s gradient" % s)
    flagged = tables["mat"].touched.cpu().numpy().reshape(n_rel, d)
    assert (flagged.all(1) == (counts > 0)).all() and (flagged.any(1) == flagged.all(1)).all()


def test_transr_lifecycle(cuda_device, tiny_kgs, tmp_path):
    """set_args / set_kgs / init / run / test / save with presets.transr on the tiny synthetic KG: the loss falls and
    stays finite, the reference's result lines and files appear, and Hits@1 beats chance (1/420 = 0.24 %).  The tiny KG
    gives only three steps per epoch, so it trains at lr 0.1 for 200 epochs."""
    from openea_b200 import presets
    from openea_b200.models.trans import TransR
    from tests.test_e2e_gpu import _hits1
    args = presets.transr()
    args.batch_size, args.max_epoch, args.start_valid, args.dim, args.learning_rate = 1000, 200, 1000, 32, 0.1
    model, out = _lifecycle(TransR, args, tiny_kgs, "sharing", tmp_path)
    loss = _losses(out, "avg. triple loss:")
    assert len(loss) == 200 and np.isfinite(loss).all()
    assert loss[-1] < 0.9 * loss[0], (loss[0], loss[-1])
    assert "Training ends. Total time" in out
    assert _hits1(out, "accurate results:") > 100.0 / 420
    for f in ("ent_embeds.npy", "rel_embeds.npy", "alignment_results_12"):
        assert os.path.exists(model.out_folder + f), f
    ent = np.load(model.out_folder + "ent_embeds.npy")
    assert ent.shape == (model.kgs.entities_num, 32) and np.isfinite(ent).all()


def test_transr_resume_from_checkpoint_continues_the_same_run(cuda_device, tiny_kgs, tmp_path):
    """6 epochs in one go == 3 epochs, checkpoint, a NEW model restored from the file, 3 more epochs: the three tables
    (the matrix table included) and their Adagrad accumulators.  Gradient sums are atomics, so agreement is to fp32
    accumulation noise, not bit-wise."""
    from openea_b200 import presets
    from openea_b200.models.trans import TransR
    from openea_b200.modules.base import initializers
    from openea_b200.modules.load.kgs import read_kgs_from_folder

    def make(max_epoch, out, **extra):
        args = presets.transr()
        args.training_data, args.output = tiny_kgs, str(tmp_path) + "/" + out + "/"
        args.batch_size, args.max_epoch, args.start_valid, args.dim = 1000, max_epoch, 1000, 32
        for k, v in extra.items():
            setattr(args, k, v)
        initializers.set_seed(77)
        m = TransR()
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
        assert "rel_matrix" in resumed._checkpoint_tables()
        assert resumed.load_checkpoint(first.out_folder + "checkpoint.pt") == 4
        resumed.run()
    for name in ("ent_embeds", "rel_embeds", "rel_matrix"):
        a, b = getattr(straight, name), getattr(resumed, name)
        np.testing.assert_allclose(b.raw().cpu().numpy(), a.raw().cpu().numpy(), rtol=2e-3, atol=2e-5, err_msg=name)
        np.testing.assert_allclose(b.state1.cpu().numpy(), a.state1.cpu().numpy(), rtol=2e-3, atol=2e-5, err_msg=name)
    assert resumed._epoch_seed == straight._epoch_seed
