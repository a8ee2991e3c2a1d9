"""GPU tests of RotatE and HolE (oea_model_score_fed, OEA_MODEL_ROTATE / OEA_MODEL_HOLE) through the engine, against the
float64 oracle of tests/semantic_ext_oracle.py on identical fed batches; whole training steps against dense float64
steps; the reference lifecycles of RotatE, HolE and BootEA_RotatE on the tiny synthetic KG; checkpoint → resume of
BootEA_RotatE; and size-independent properties at the 15K batch shape, where the oracle is too slow."""
import contextlib
import io

import numpy as np
import pytest
import torch

from tests import semantic_ext_oracle as so
from tests.helpers import make_batch
from tests.test_zz_triple_ext_gpu import tiny_kgs, _lifecycle, _losses        # noqa: F401  (fixture + helpers)

pytestmark = pytest.mark.gpu

GAMMA = 12.0


def _engine():
    from openea_b200 import engine
    return engine


def _dev(hrt):
    return None if hrt is None else torch.from_numpy(np.ascontiguousarray(hrt.astype(np.int32))).cuda()


def _case(model, seed, n_ent, n_rel, d, norm):
    rng = np.random.default_rng(seed)
    tabs, norms = {}, {}
    for i, s in enumerate(so.SLOTS[model]):
        rows = n_rel if s == "rel" else n_ent
        tabs[s] = (rng.standard_normal((rows, d)) * (0.6 + 0.3 * i) / np.sqrt(d)).astype(np.float32)
        norms[s] = norm
    return rng, tabs, norms


def _trainer(model, tabs, norms, opt, neg_weight=None, margin=0.3, lr=0.01):
    eng = _engine()
    tables = tuple(eng.EmbeddingTable(tabs[s], norms[s], opt) for s in so.SLOTS[model])
    if model == "RotatE":
        tr = eng.ModelTrainer("RotatE", tables, eng.loss_cfg("logistic", "L2"), lr, gamma=GAMMA, neg_weight=neg_weight)
    else:
        tr = eng.ModelTrainer("HolE", tables, eng.loss_cfg("margin-based", "L2", margin=margin), lr)
    return tr, dict(zip(so.SLOTS[model], tables))


def _assert_rows_close(got, want, what):
    scale = max(1e-6, float(np.abs(want).max()))
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=2e-5 * scale, err_msg=what)


CASES = [("RotatE", 4, 0.25), ("RotatE", 3, 1.0), ("RotatE", 1, 1.0), ("HolE", 1, None), ("HolE", 3, None)]


@pytest.mark.parametrize("model,k,neg_weight", CASES)
@pytest.mark.parametrize("norm", [True, False])
@pytest.mark.parametrize("d", [75, 100, 200])
def test_forward_backward_matches_oracle(cuda_device, model, k, neg_weight, norm, d):
    n_ent, n_rel, n_pos = 1500, 29, 300
    rng, tabs, norms = _case(model, 7 * d + k + len(model) + int(norm), n_ent, n_rel, d, norm)
    pos, neg = make_batch(rng, n_ent, n_rel, n_pos, k)
    kw = dict(gamma=GAMMA, neg_weight=neg_weight) if model == "RotatE" else dict(margin=0.3)
    want_loss, want_g = so.fwd_bwd(model, tabs, norms, pos, neg, **kw)
    tr, tables = _trainer(model, tabs, norms, "Adagrad", neg_weight=neg_weight)
    tr.score_fed(_dev(pos), _dev(neg))
    assert tr.read_loss() == pytest.approx(want_loss, rel=1e-4)
    for s, tab in tables.items():
        _assert_rows_close(tab.grad[:, :d].cpu().numpy(), want_g[s], "%s gradient of %s" % (s, model))
        assert not tab.grad[:, d:].any().item(), "padding columns must stay zero"
        touched = tab.touched.cpu().numpy().astype(bool)
        assert (np.abs(want_g[s]).sum(1)[~touched] == 0).all(), "untouched rows must have zero oracle gradient"


def _assert_adam_tables_close(got, want, start, what):
    """Adam moves every coordinate with a non-zero gradient by ≈ lr whatever the gradient's size, so a coordinate whose
    float64 gradient is ≈ 0 (cancellation) may move the other way in fp32.  All but a per-mille of the coordinates must
    agree tightly, movement included; none may be further off than the three steps could carry it (3·lr)."""
    move_ok = np.isclose(got - start, want - start, rtol=5e-3, atol=1e-6 + 2e-3 * np.abs(want - start).max())
    val_ok = np.isclose(got, want, rtol=1e-4, atol=2e-5 * max(1e-6, float(np.abs(want).max())))
    assert (move_ok & val_ok).mean() > 0.999, (what, (move_ok & val_ok).mean())
    assert np.abs(got - want).max() <= 3 * 0.01 * 1.01, what


@pytest.mark.parametrize("model,opt,k", [("RotatE", "Adam", 4), ("RotatE", "Adagrad", 4), ("HolE", "Adagrad", 1),
                                         ("HolE", "Adagrad", 3)])
def test_training_steps_equal_dense_float64_steps(cuda_device, model, opt, k):
    """Three whole steps (scorer + row optimiser on every table) equal the oracle's dense TF-style float64 steps."""
    d, n_ent, n_rel, lr = 100, 1200, 23, 0.01
    rng, tabs, norms = _case(model, 11 + k, n_ent, n_rel, d, True)
    neg_weight = 1.0 / k if model == "RotatE" else None
    kw = dict(gamma=GAMMA, neg_weight=neg_weight) if model == "RotatE" else dict(margin=0.3)
    st = so.DenseState(tabs, opt)
    tr, tables = _trainer(model, tabs, norms, opt, neg_weight=neg_weight, lr=lr)
    for it in range(3):
        pos, neg = make_batch(rng, n_ent, n_rel, 300, k)
        want = so.step(st, model, norms, pos, neg, lr, **kw)
        tr.score_fed(_dev(pos), _dev(neg))
        tr.apply()
        assert tr.read_loss() == pytest.approx(want, rel=1e-4), it
    for s, tab in tables.items():
        got, want = tab.raw().cpu().numpy(), st.w[s]
        start = tabs[s].astype(np.float64)
        if opt == "Adam":
            _assert_adam_tables_close(got, want, start, s)
        else:
            np.testing.assert_allclose(got - start, want - start, rtol=5e-3,
                                       atol=1e-6 + 2e-3 * np.abs(want - start).max(), err_msg=s)
            _assert_rows_close(got, want, "%s after 3 steps" % s)
        assert not tab.grad.any().item() and not tab.touched.any().item()


@pytest.mark.parametrize("name", ["RotatE", "HolE"])
def test_semantic_ext_lifecycle(cuda_device, tiny_kgs, tmp_path, name):
    """set_args / set_kgs / init / run / test / save on the tiny synthetic KG: the loss falls and stays finite, the result
    lines and files of the reference appear."""
    import os
    from openea_b200 import presets
    from openea_b200.models import semantic
    from tests.test_e2e_gpu import _hits1
    args = getattr(presets, name.lower())("15K")
    args.batch_size, args.max_epoch, args.start_valid, args.dim = 1000, 60, 1000, 32
    model, out = _lifecycle(getattr(semantic, name), args, tiny_kgs, "sharing", tmp_path)
    loss = _losses(out, "avg. triple loss:")
    assert len(loss) == 60 and np.isfinite(loss).all()
    assert loss[-1] < 0.9 * loss[0], (loss[0], loss[-1])
    assert "Training ends. Total time" in out
    assert 0.0 <= _hits1(out, "accurate results:") <= 100.0
    for f in ("ent_embeds.npy", "rel_embeds.npy", "alignment_results_12"):
        assert os.path.exists(model.out_folder + f), f
    ent = np.load(model.out_folder + "ent_embeds.npy")
    assert ent.shape == (model.kgs.entities_num, 32) and np.isfinite(ent).all()
    if name == "RotatE":                   # save() writes preprocessing.normalize(re + im) (rotate.py:140-141)
        np.testing.assert_allclose(np.linalg.norm(ent, axis=1), 1.0, rtol=1e-4)


def _bootea_rotate_args(tiny, tmp_path, out, max_epoch, **extra):
    from openea_b200 import presets
    args = presets.bootea_rotate("15K")
    args.training_data, args.output = tiny, str(tmp_path) + "/" + out + "/"
    args.batch_size, args.max_epoch, args.start_valid, args.sub_epoch, args.dim = 1000, max_epoch, 1000, 5, 32
    args.start_bp, args.neg_sampling, args.truncated_epsilon, args.sim_th, args.min_iter = 5, "truncated", 0.9, 0.3, 1
    for k, v in extra.items():
        setattr(args, k, v)
    return args


def test_bootea_rotate_lifecycle(cuda_device, tiny_kgs, tmp_path):
    from openea_b200.approaches import BootEA_RotatE
    args = _bootea_rotate_args(tiny_kgs, tmp_path, "x", 60)
    model, out = _lifecycle(BootEA_RotatE, args, tiny_kgs, "swapping", tmp_path)
    for line in ("avg. triple loss", "bootstrapping", "generating neighbors of", "Training ends. Total time"):
        assert line in out, line
    loss = _losses(out, "avg. triple loss:")
    assert np.isfinite(loss).all() and loss[-1] < loss[0]
    ent = np.load(model.out_folder + "ent_embeds.npy")
    assert np.isfinite(ent).all()


def test_bootea_rotate_resume_from_checkpoint_continues_the_same_run(cuda_device, tiny_kgs, tmp_path):
    """5 epochs (with bootstrapping and alignment training at their end), checkpoint, then 5 more epochs two ways: the same
    model carrying on in memory (the straight run) and a NEW model restored from the file.  The restored model holds
    exactly the checkpointed state — variables, the triple and the alignment optimisers' Adam slots and steps, the
    bootstrapped labels, the sampler seed — and its last iteration (validation ends the run before a second
    bootstrapping) reproduces the straight run.  Uniform negatives, as the shipped configuration: the ε-truncated
    candidate lists define a set, not an order, so two runs draw different negatives from them.  Gradient sums are
    atomics and Adam turns the sign of a gradient that is ≈ 0 into a full step, so the tables agree to that noise."""
    from openea_b200.approaches import BootEA_RotatE
    from openea_b200.modules.base import initializers
    from openea_b200.modules.load.kgs import read_kgs_from_folder

    def make(max_epoch, out, **extra):
        args = _bootea_rotate_args(tiny_kgs, tmp_path, out, max_epoch, start_valid=10, neg_sampling="uniform", **extra)
        initializers.set_seed(77)
        m = BootEA_RotatE()
        m.set_args(args)
        m.set_kgs(read_kgs_from_folder(tiny_kgs, args.dataset_division, "swapping", True))
        m.init()
        m._epoch_seed = 424242
        return m
    with contextlib.redirect_stdout(io.StringIO()):
        first = make(5, "b", checkpoint_every=5)
        first.run()
        resumed = make(10, "c")
        assert resumed.load_checkpoint(first.out_folder + "checkpoint.pt") == 6
        assert torch.equal(resumed._label, first._label) and (first._label >= 0).any(), "labels must have been bootstrapped"
        assert resumed._epoch_seed == first._epoch_seed
        for name in ("re_ent_embeds", "im_ent_embeds", "rel_embeds"):
            a, b = getattr(first, name), getattr(resumed, name)
            assert torch.equal(a.weight, b.weight) and torch.equal(a.state2, b.state2) and a.adam_t == b.adam_t, name
        for x, y in zip(first.alignment_trainer.live, resumed.alignment_trainer.live):
            assert x.adam_t == y.adam_t > 0 and torch.equal(x.state1, y.state1) and torch.equal(x.state2, y.state2)
        resumed.run()
        straight = first                      # the same run carried on in memory from the checkpointed epoch
        straight.args.max_epoch, straight._start_epoch = 10, 6
        straight.run()
    assert torch.equal(resumed._label, straight._label)
    assert resumed._epoch_seed == straight._epoch_seed
    for name in ("re_ent_embeds", "im_ent_embeds", "rel_embeds"):
        a = getattr(straight, name).raw().cpu().numpy()
        b = getattr(resumed, name).raw().cpu().numpy()
        ok = np.isclose(b, a, rtol=2e-3, atol=2e-4)
        assert ok.mean() > 0.999, (name, ok.mean())
        assert np.abs(b - a).max() <= 2 * 5 * float(straight.args.learning_rate), name


@pytest.mark.parametrize("model", ["RotatE", "HolE"])
def test_full_size_properties(cuda_device, model):
    """At the 15K batch shape (5000 positives, k = 10 for RotatE, 1 for HolE as shipped): finite loss, two half batches add
    up to the whole batch, and a permutation of the batch (positives with their negatives) changes nothing."""
    rng = np.random.default_rng(12)
    n_ent, n_rel, B, d = 30000, 450, 5000, 100
    k = 10 if model == "RotatE" else 1
    tabs = {s: (rng.standard_normal((n_rel if s == "rel" else n_ent, d)) / 10).astype(np.float32) for s in so.SLOTS[model]}
    norms = {s: True for s in tabs}
    pos = np.stack([rng.integers(0, n_ent, B), rng.integers(0, n_rel, B), rng.integers(0, n_ent, B)]).astype(np.int32)
    neg = np.repeat(pos, k, axis=1)
    side = rng.random(B * k) < 0.5
    neg[0, side] = rng.integers(0, n_ent, side.sum())
    neg[2, ~side] = rng.integers(0, n_ent, (~side).sum())

    def run(batches):
        tr, tables = _trainer(model, tabs, norms, "Adagrad", neg_weight=1.0 / k if model == "RotatE" else None)
        for ps, ns in batches:
            tr.score_fed(_dev(pos[:, ps]), _dev(neg[:, ns]))
        return [tr.read_loss()] + [t.grad.clone() for t in tables.values()]

    def close(a, b):
        assert a[0] == pytest.approx(b[0], rel=1e-5)
        for x, y in zip(a[1:], b[1:]):
            assert float((x - y).abs().max()) <= 2e-4 * float(y.abs().max())
    whole = run(((slice(None), slice(None)),))
    assert np.isfinite(whole[0]) and whole[0] > 0 and all(torch.isfinite(g).all() for g in whole[1:])
    half = B // 2
    close(run(((slice(0, half), slice(0, half * k)), (slice(half, B), slice(half * k, B * k)))), whole)
    perm = rng.permutation(B)
    pos_p, neg_p = pos[:, perm], neg.reshape(3, B, k)[:, perm].reshape(3, B * k)
    tr, tables = _trainer(model, tabs, norms, "Adagrad", neg_weight=1.0 / k if model == "RotatE" else None)
    tr.score_fed(_dev(pos_p), _dev(neg_p))
    close([tr.read_loss()] + [t.grad for t in tables.values()], whole)
