"""GPU parity tests of the projected / bilinear score family (oea_model_score_fed) and of the device batch producer
(oea_triple_sample_batch), through the C-ABI, against oracle/triple_ext.py on identical fed index batches.
Tolerances as in tests/test_triple_gpu.py: 1e-4 relative on the fp32 loss, 1e-4 relative (+ a floor tied to the
gradient scale) on per-row gradients and updated tables; L1 sign gradients by counting disagreeing coordinates."""
import numpy as np
import pytest
import torch

from oracle import triple_ext as ox
from tests.helpers import make_batch

pytestmark = pytest.mark.gpu

LOSS_TOL = 1e-4


def _engine():
    from openea_b200 import engine
    return engine


def _dev(hrt):
    return None if hrt is None else torch.from_numpy(np.ascontiguousarray(hrt.astype(np.int32))).cuda()


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


def _tables(slots, tabs, norms, opt="Adagrad"):
    eng = _engine()
    return tuple(None if s is None else eng.EmbeddingTable(tabs[s], norms[s], opt) for s in slots)


def _assert_rows_close(got, want, what):
    scale = max(1e-6, float(np.abs(want).max()))
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=2e-5 * scale, err_msg=what)


CASES = [("TransE", "limited", 4, "L2"), ("TransE", "margin-based", 1, "L1"),
         ("TransH", "margin-based", 1, "L2"), ("TransH", "margin-based", 1, "L1"), ("TransH", "limited", 5, "L2"),
         ("TransD", "margin-based", 1, "L2"), ("TransD", "limited", 3, "L2"), ("TransD", "logistic", 2, "L1"),
         ("TransD", "positive", 0, "L2"),
         ("DistMult", "logistic", 3, "L2"), ("SimplE", "logistic", 2, "L2")]


@pytest.mark.parametrize("model,loss,k,loss_norm", CASES)
@pytest.mark.parametrize("norm", [True, False])
@pytest.mark.parametrize("d", [12, 75, 100, 200])
def test_model_forward_backward_matches_oracle(cuda_device, model, loss, k, loss_norm, norm, d):
    eng = _engine()
    n_ent, n_rel, n_pos = 1500, 29, 400
    rng, slots, tabs, norms = _case(model, 7 * d + k + len(model), n_ent, n_rel, d, norm)
    pos, neg = make_batch(rng, n_ent, n_rel, n_pos, k)
    kw = dict(margin=1.1 if loss == "margin-based" else 0.3, neg_margin=2.2, balance=0.2)
    mean = model == "DistMult"
    scale = 1.0 / (n_pos * (1 + k)) if mean else 1.0
    want_loss, want_g, _ = ox.fwd_bwd(model, tabs, norms, pos, neg, loss, loss_norm=loss_norm, scale=scale, **kw)

    tables = _tables(slots, tabs, norms)
    tr = eng.ModelTrainer(model, tables, eng.loss_cfg(loss, loss_norm, **kw), lr=0.01, mean_loss=mean)
    tr.score_fed(_dev(pos), _dev(neg))
    assert tr.read_loss() == pytest.approx(want_loss, rel=LOSS_TOL)
    for s, tab in zip(slots, tables):
        if s is None:
            continue
        got = tab.grad[:, :d].cpu().numpy()
        want = want_g[s]
        if loss_norm == "L1" and model in ("TransE", "TransH", "TransD"):
            bad = np.abs(got - want) > 1e-4 * max(1.0, np.abs(want).max())
            assert bad.mean() < 2e-3, s
        else:
            _assert_rows_close(got, want, "%s gradient of %s" % (s, model))
        assert not tab.grad[:, d:].any().item(), "padding columns must stay zero"
        touched = tab.touched.cpu().numpy().astype(bool)
        assert (np.abs(want).sum(1)[~touched] == 0).all(), "untouched rows must have zero oracle gradient"


def test_transe_through_the_model_entry_equals_the_k1_kernel(cuda_device):
    """OEA_MODEL_TRANSE runs the same maths as oea_triple_score_fed: losses and gradients agree to fp32 rounding."""
    eng = _engine()
    rng, slots, tabs, norms = _case("TransE", 3, 2000, 31, 100, True)
    pos, neg = make_batch(rng, 2000, 31, 500, 6)
    cfg = eng.loss_cfg("limited", "L2", margin=0.2, neg_margin=2.0, balance=0.3)
    a = _tables(slots, tabs, norms)
    b = _tables(slots, tabs, norms)
    ta = eng.ModelTrainer("TransE", a, cfg, lr=0.01)
    tb = eng.TripleTrainer(b[0], b[1], cfg, lr=0.01)
    ta.score_fed(_dev(pos), _dev(neg))
    tb.score_fed(_dev(pos), _dev(neg))
    assert ta.read_loss() == pytest.approx(tb.read_loss(), rel=1e-6)
    for x, y in zip(a[:2], b[:2]):
        # two kernels, two summation orders: agreement to fp32 rounding of the row reductions
        np.testing.assert_allclose(x.grad.cpu().numpy(), y.grad.cpu().numpy(), rtol=1e-4, atol=1e-6)
        assert torch.equal(x.touched, y.touched)


@pytest.mark.parametrize("model,loss,k", [("TransH", "margin-based", 1), ("TransD", "limited", 4),
                                          ("DistMult", "logistic", 2), ("SimplE", "logistic", 2)])
@pytest.mark.parametrize("opt", ["Adagrad", "SGD"])
def test_model_training_steps_equal_dense_tf_steps(cuda_device, model, loss, k, opt):
    """Three full steps (scorer + row optimiser on every table) equal the oracle's dense TF-style steps."""
    eng = _engine()
    d, n_ent, n_rel = 100, 1200, 23
    rng, slots, tabs, norms = _case(model, 11, n_ent, n_rel, d, True)
    kw = dict(margin=1.0 if loss == "margin-based" else 0.05, neg_margin=1.8, balance=0.25)
    mean = model == "DistMult"
    st = ox.DenseState(tabs, opt)
    tables = _tables(slots, tabs, norms, opt)
    tr = eng.ModelTrainer(model, tables, eng.loss_cfg(loss, "L2", **kw), lr=0.05, mean_loss=mean)
    for it in range(3):
        pos, neg = make_batch(rng, n_ent, n_rel, 300, k)
        scale = 1.0 / (300 * (1 + k)) if mean else 1.0
        want = ox.step(st, model, norms, pos, neg, loss, 0.05, scale=scale, **kw)
        tr.score_fed(_dev(pos), _dev(neg))
        tr.apply()
        assert tr.read_loss() == pytest.approx(want, rel=LOSS_TOL), it
    for s, tab in zip(slots, tables):
        if s is not None:
            _assert_rows_close(tab.raw().cpu().numpy(), st.w[s], "%s after 3 steps" % s)
            assert not tab.grad.any().item() and not tab.touched.any().item()


def test_adadelta_steps_equal_dense_tf_steps(cuda_device):
    """tf.train.AdadeltaOptimizer through oea_rowopt_apply (dense rule: rows without gradient decay their accumulators):
    three TransE steps equal the oracle's dense steps on every row."""
    eng = _engine()
    d, n_ent, n_rel = 100, 900, 17
    rng, slots, tabs, norms = _case("TransE", 21, n_ent, n_rel, d, True)
    kw = dict(margin=0.05, neg_margin=1.8, balance=0.25)
    st = ox.DenseState(tabs, "Adadelta")
    tables = _tables(slots, tabs, norms, "Adadelta")
    tr = eng.ModelTrainer("TransE", tables, eng.loss_cfg("limited", "L2", **kw), lr=1.0)
    for it in range(3):
        pos, neg = make_batch(rng, n_ent, n_rel, 200, 4)
        want = ox.step(st, "TransE", norms, pos, neg, "limited", 1.0, **kw)
        tr.score_fed(_dev(pos), _dev(neg))
        tr.apply()
        assert tr.read_loss() == pytest.approx(want, rel=LOSS_TOL), it
    for s, tab in zip(slots, tables):
        if s is not None:
            _assert_rows_close(tab.raw().cpu().numpy(), st.w[s], "%s after 3 Adadelta steps" % s)
            np.testing.assert_allclose(tab.state1[:, :d].cpu().numpy(), st.s1[s], rtol=1e-4, atol=1e-9)
            assert not tab.grad.any().item() and not tab.touched.any().item()


def _tiny_kgs(rng, n_ent_kg=300, n_rel=11, n_tri=2000):
    """Two KGs over disjoint entity id ranges (0..n) and (n..2n), relation ids shared."""
    def kg(lo):
        t = np.stack([rng.integers(lo, lo + n_ent_kg, n_tri), rng.integers(0, n_rel, n_tri),
                      rng.integers(lo, lo + n_ent_kg, n_tri)], axis=1).astype(np.int32)
        return np.unique(t, axis=0)
    return kg(0), kg(n_ent_kg), n_ent_kg


@pytest.mark.parametrize("sampler", ["fast", "independent"])
@pytest.mark.parametrize("k", [0, 1, 7])
def test_batch_producer_properties(cuda_device, sampler, k):
    """batch.py:36-119 invariants of the device batch producer: an epoch's positives are a permutation of the triple
    lists (each KG's share per step as batch.py:39-42), every negative keeps the relation and exactly one end of its
    positive, the corrupted end comes from the positive's own KG, negatives are (almost never) known triples, the
    fast sampler's k negatives of one positive are distinct (random.sample), and the same seed reproduces the batch."""
    eng = _engine()
    rng = np.random.default_rng(17 + k)
    t1, t2, n = _tiny_kgs(rng)
    ent = eng.EmbeddingTable(rng.standard_normal((2 * n, 16)).astype(np.float32), True)
    rel = eng.EmbeddingTable(rng.standard_normal((11, 16)).astype(np.float32), True)
    kg1 = eng.DeviceKG(t1, np.arange(0, n), 2 * n)
    kg2 = eng.DeviceKG(t2, np.arange(n, 2 * n), 2 * n)
    tset = eng.DeviceTripleSet([kg1.triples, kg2.triples], 2 * n, 11)
    tr = eng.ModelTrainer("TransE", (ent, rel), eng.loss_cfg("limited", "L2", 0.1, 2.0, 0.2), 0.01, sampler=sampler)
    B = 512
    steps = int(np.ceil((len(t1) + len(t2)) / B))
    b1 = int(len(t1) / (len(t1) + len(t2)) * B)
    known = {tuple(x) for x in np.concatenate([t1, t2]).tolist()}
    seen, n_known, n_neg, dup_rows = [], 0, 0, 0
    for step in range(steps):
        pos, neg = tr.sample_batch(kg1, kg2, tset, B, k, step, epoch_seed=12345)
        p = pos.cpu().numpy().T
        want1 = max(0, min((step + 1) * b1, len(t1)) - min(step * b1, len(t1)))
        assert (p[:want1, 0] < n).all() and (p[want1:, 0] >= n).all()      # KG1's slice first, then KG2's
        seen.append(p)
        first = (pos.clone(), None if neg is None else neg.clone())   # the producer reuses one index buffer
        pos, neg = tr.sample_batch(kg1, kg2, tset, B, k, step, epoch_seed=12345)
        assert torch.equal(first[0], pos) and (neg is None or torch.equal(first[1], neg))
        other, _ = tr.sample_batch(kg1, kg2, tset, B, k, step, epoch_seed=54321)
        assert other.shape == first[0].shape and not torch.equal(other, first[0])
        pos, neg = first
        if k == 0:
            assert neg is None
            continue
        q = neg.cpu().numpy().T.reshape(len(p), k, 3)
        assert (q[:, :, 1] == p[:, None, 1]).all()
        same_h, same_t = q[:, :, 0] == p[:, None, 0], q[:, :, 2] == p[:, None, 2]
        assert (same_h | same_t).all()
        assert ((q[:, :, 0] < n) == (p[:, None, 0] < n)).all() and ((q[:, :, 2] < n) == (p[:, None, 0] < n)).all()
        n_known += sum(tuple(x) in known for x in q.reshape(-1, 3).tolist())
        n_neg += q.shape[0] * k
        if sampler == "fast" and k > 1:     # random.sample: distinct inside one try (a re-draw after a rejection may repeat)
            dup_rows += sum(len({tuple(x) for x in row.tolist()}) < k for row in q)
    allp = np.concatenate(seen)
    assert len(allp) == len(t1) + len(t2)
    assert {tuple(x) for x in allp.tolist()} == known                      # a permutation: every triple exactly once
    if k:
        assert n_known <= 1e-3 * n_neg + 2                                 # only a last try may keep a known triple
        assert dup_rows <= 0.01 * len(allp)


def test_fast_batch_producer_draws_the_same_negatives_as_the_fused_kernel(cuda_device, monkeypatch):
    """sampler 0 shares warp_sample_negatives and the positive permutation with k_score_sampled: for one seed the
    index vectors equal the fused kernel's debug dump."""
    eng = _engine()
    monkeypatch.setenv("OEA_SCORE_V1", "1")          # the warp-per-positive fused kernel
    rng = np.random.default_rng(23)
    t1, t2, n = _tiny_kgs(rng)
    ent = eng.EmbeddingTable(rng.standard_normal((2 * n, 16)).astype(np.float32), True)
    rel = eng.EmbeddingTable(rng.standard_normal((11, 16)).astype(np.float32), True)
    kg1 = eng.DeviceKG(t1, np.arange(0, n), 2 * n)
    kg2 = eng.DeviceKG(t2, np.arange(n, 2 * n), 2 * n)
    tset = eng.DeviceTripleSet([kg1.triples, kg2.triples], 2 * n, 11)
    cfg = eng.loss_cfg("limited", "L2", 0.1, 2.0, 0.2)
    B, k, step, seed = 256, 5, 2, 777
    dbg = torch.zeros(B, 2 + k, dtype=torch.int32, device="cuda")
    eng.TripleTrainer(ent, rel, cfg, 0.01).score_sampled(kg1, kg2, tset, B, k, step, seed, dbg=dbg)
    pos, neg = eng.ModelTrainer("TransE", (ent, rel), cfg, 0.01).sample_batch(kg1, kg2, tset, B, k, step, seed)
    dbg = dbg.cpu().numpy()
    p, q = pos.cpu().numpy().T, neg.cpu().numpy().T.reshape(-1, k, 3)
    for i in range(len(p)):
        tri = dbg[i, 0]
        src = t2[tri - (1 << 30)] if tri >= (1 << 30) else t1[tri]
        assert (p[i] == src).all()
        for j in range(k):
            head = (dbg[i, 1] >> j) & 1
            want = (dbg[i, 2 + j], p[i, 1], p[i, 2]) if head else (p[i, 0], p[i, 1], dbg[i, 2 + j])
            assert tuple(q[i, j]) == tuple(want)


def test_model_entry_rejects_bad_arguments(cuda_device):
    import ctypes as C
    from openea_b200 import lib as L
    eng = _engine()
    rng, slots, tabs, norms = _case("TransD", 1, 50, 5, 16, True)
    tables = _tables(slots, tabs, norms)
    tr = eng.ModelTrainer("TransD", tables, eng.loss_cfg("margin-based", "L2", margin=1.0), 0.01)
    pos, neg = make_batch(rng, 50, 5, 8, 2)                                 # margin needs n_pos == n_neg
    with pytest.raises(L.OeaError):
        tr.score_fed(_dev(pos), _dev(neg))
    bad = eng.ModelTrainer("TransH", (tables[0], tables[1], None, None), eng.loss_cfg("limited", "L2"), 0.01)
    with pytest.raises(L.OeaError):                                         # TransH without its normal vectors
        bad.score_fed(_dev(pos), _dev(neg))


# ---- the reference lifecycle of the models built on the family ------------------------------------------------------
@pytest.fixture(scope="module")
def tiny_kgs(tmp_path_factory):
    from openea_b200.synth import write_dataset
    folder = str(tmp_path_factory.mktemp("tiny_ext")) + "/"
    write_dataset(folder, "tiny")
    return folder


def _lifecycle(model_cls, args, folder, mode, tmp_path):
    from tests.test_e2e_gpu import _run
    return _run(model_cls, args, folder, mode, tmp_path)


def _losses(out, tag):
    import re
    return [float(x) for x in re.findall(re.escape(tag) + r"\s*([0-9.]+)", out)]


@pytest.mark.parametrize("name", ["TransH", "TransD", "SimplE", "DistMult"])
def test_score_family_lifecycle(cuda_device, tiny_kgs, tmp_path, name):
    """set_args / set_kgs / init / run / test / save of the four models on the tiny synthetic KG: the epoch loss must
    fall, the result lines and files of the reference must appear, and the shared-id alignment must beat chance."""
    import os
    from openea_b200 import presets
    from openea_b200.models import trans, semantic
    from tests.test_e2e_gpu import _hits1
    cls = {"TransH": trans.TransH, "TransD": trans.TransD, "SimplE": semantic.SimplE, "DistMult": semantic.DistMult}[name]
    args = getattr(presets, name.lower())("15K")
    args.batch_size, args.max_epoch, args.start_valid, args.dim = 1000, 120, 1000, 32
    model, out = _lifecycle(cls, args, tiny_kgs, "sharing", tmp_path)
    tag = "triple loss:" if name == "DistMult" else "avg. triple loss:"
    loss = _losses(out, tag)
    assert len(loss) == 120
    if name == "DistMult":
        # reduce_mean over the batch + Adagrad at lr 0.01 on unit rows (distmult.py:58-59): the loss sits at
        # steps·ln 2 and moves only in the 4th digit over 120 epochs; it must not grow
        assert abs(loss[0] - 5 * np.log(2.0)) < 0.01 and loss[-1] <= loss[0] * 1.001, (loss[0], loss[-1])
    else:
        assert loss[-1] < 0.9 * loss[0], (loss[0], loss[-1])
    assert "Training ends. Total time" in out
    h1 = _hits1(out, "accurate results:")
    assert 0.0 <= h1 <= 100.0
    for f in ("ent_embeds.npy", "rel_embeds.npy", "alignment_results_12"):
        assert os.path.exists(model.out_folder + f), f
    ent = np.load(model.out_folder + "ent_embeds.npy")
    assert ent.shape == (model.kgs.entities_num, 32) and np.isfinite(ent).all()


def test_bootea_transh_lifecycle(cuda_device, tiny_kgs, tmp_path):
    from openea_b200 import presets
    from openea_b200.approaches import BootEA_TransH
    from tests.test_e2e_gpu import _hits1
    args = presets.bootea_transh("15K")
    args.batch_size, args.max_epoch, args.start_valid, args.sub_epoch = 1000, 200, 1000, 10
    args.truncated_epsilon, args.dim, args.sim_th = 0.9, 32, 0.5
    model, out = _lifecycle(BootEA_TransH, args, tiny_kgs, "swapping", tmp_path)
    assert "avg. triple loss" in out and "generating neighbors of" in out and "Training ends. Total time" in out
    loss = _losses(out, "avg. triple loss:")
    assert loss[-1] < loss[0]
    assert _hits1(out, "accurate results:") > 4.0        # chance = 0.24 %


def test_resume_from_checkpoint_continues_the_same_run(cuda_device, tiny_kgs, tmp_path):
    """6 epochs in one go == 3 epochs, checkpoint, a NEW model restored from the file, 3 more epochs (variables and
    Adagrad accumulators; gradient sums are atomics, so agreement is to fp32 accumulation noise, not bit-wise)."""
    import contextlib
    import io
    from openea_b200 import presets
    from openea_b200.models.trans import TransE
    from openea_b200.modules.base import initializers
    from openea_b200.modules.load.kgs import read_kgs_from_folder

    def make(max_epoch, out, **extra):
        args = presets.transe("15K")
        args.training_data, args.output = tiny_kgs, str(tmp_path) + "/" + out + "/"
        args.batch_size, args.max_epoch, args.start_valid, args.dim = 1000, max_epoch, 1000, 32
        for k, v in extra.items():
            setattr(args, k, v)
        initializers.set_seed(77)
        m = TransE()
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
        assert resumed.load_checkpoint(first.out_folder + "checkpoint.pt") == 4
        resumed.run()
    for name in ("ent_embeds", "rel_embeds"):
        a, b = getattr(straight, name), getattr(resumed, name)
        np.testing.assert_allclose(b.raw().cpu().numpy(), a.raw().cpu().numpy(), rtol=2e-3, atol=2e-5, err_msg=name)
        np.testing.assert_allclose(b.state1.cpu().numpy(), a.state1.cpu().numpy(), rtol=2e-3, atol=2e-5, err_msg=name)
    assert resumed._epoch_seed == straight._epoch_seed


def test_pipelined_host_step_equals_the_synchronous_one(cuda_device):
    """oea_triple_step_fed_host_submit / _collect (depth-2 pipeline: copies and the host wait off the critical path)
    against oea_triple_step_fed_host on the same batches from the same tables: per-step losses and the final tables."""
    eng = _engine()
    rng = np.random.default_rng(8)
    d, n_ent, n_rel = 100, 4000, 37
    from tests.helpers import make_tables
    ent, rel = make_tables(rng, n_ent, n_rel, d)
    cfg = eng.loss_cfg("limited", "L2", margin=0.01, neg_margin=2.0, balance=0.2)
    batches = []
    for _ in range(7):
        pos, neg = make_batch(rng, n_ent, n_rel, 600, 10)
        batches.append((torch.from_numpy(pos).pin_memory(), torch.from_numpy(neg).pin_memory()))
    a = eng.TripleTrainer(eng.EmbeddingTable(ent, True), eng.EmbeddingTable(rel, True), cfg, 0.01)
    want = [a.step_fed_host(p, n) for p, n in batches]
    b = eng.TripleTrainer(eng.EmbeddingTable(ent, True), eng.EmbeddingTable(rel, True), cfg, 0.01)
    pipe = eng.FedHostPipeline(b, 3 * 600 * 11)
    got = []
    for i, (p, n) in enumerate(batches):
        pipe.submit(i % 2, p, n)
        if i:
            got.append(pipe.collect((i - 1) % 2))
    got.append(pipe.collect((len(batches) - 1) % 2))
    np.testing.assert_allclose(got, want, rtol=1e-4)
    torch.cuda.synchronize()
    for x, y in ((a.ent, b.ent), (a.rel, b.rel)):
        np.testing.assert_allclose(y.raw().cpu().numpy(), x.raw().cpu().numpy(), rtol=1e-4, atol=1e-6)
        assert not y.grad.any().item() and not y.touched.any().item()


@pytest.mark.parametrize("loss,k", [("limited", 10), ("logistic", 4), ("margin-based", 1), ("positive", 0)])
@pytest.mark.parametrize("d", [75, 100, 300])
def test_grouped_fed_scorer_equals_the_per_triple_scorer(cuda_device, monkeypatch, loss, k, d):
    """oea_triple_score_fed_grouped (one warp per positive and its negatives) against oea_triple_score_fed on a batch in the
    reference's layout with some unrelated negatives mixed in; then the host-index step with OEA_FED_GROUPED=1 against
    the default."""
    eng = _engine()
    from tests.helpers import make_tables
    rng = np.random.default_rng(5 * d + k)
    n_ent, n_rel, n_pos = 3000, 31, 700
    ent, rel = make_tables(rng, n_ent, n_rel, d)
    pos, neg = make_batch(rng, n_ent, n_rel, n_pos, k)
    if k:
        swap = rng.random(n_pos * k) < 0.1
        neg[:, swap] = np.stack([rng.integers(0, n_ent, swap.sum()), rng.integers(0, n_rel, swap.sum()),
                                 rng.integers(0, n_ent, swap.sum())]).astype(np.int32)
    kw = dict(margin=1.1 if loss == "margin-based" else 0.3, neg_margin=2.2, balance=0.2)
    cfg = eng.loss_cfg(loss, "L2", **kw)
    res = []
    for grouped in (False, True):
        te, tr = eng.EmbeddingTable(ent, True), eng.EmbeddingTable(rel, True)
        t = eng.TripleTrainer(te, tr, cfg, 0.01)
        t.score_fed(_dev(pos), _dev(neg), grouped=grouped)
        res.append((t.read_loss(), te.grad.cpu().numpy(), tr.grad.cpu().numpy(), te.touched.cpu().numpy()))
    assert res[1][0] == pytest.approx(res[0][0], rel=1e-5)
    for i in (1, 2):
        _assert_rows_close(res[1][i], res[0][i], "gradient, grouped vs per-triple")
    assert np.array_equal(res[1][3] != 0, res[0][3] != 0)
    losses = []
    for flag in ("0", "1"):
        monkeypatch.setenv("OEA_FED_GROUPED", flag)
        t = eng.TripleTrainer(eng.EmbeddingTable(ent, True), eng.EmbeddingTable(rel, True), cfg, 0.01)
        losses.append([t.step_fed_host(pos, neg) for _ in range(2)] + [t.ent.raw().cpu().numpy()])
    assert losses[1][0] == pytest.approx(losses[0][0], rel=1e-5) and losses[1][1] == pytest.approx(losses[0][1], rel=1e-4)
    _assert_rows_close(losses[1][2], losses[0][2], "entity table after two host-index steps")


@pytest.mark.parametrize("shape,n_ent,n_rel,B,k", [("15K", 30000, 450, 5000, 10), ("100K", 200000, 600, 20000, 10)])
def test_full_size_properties_of_the_fed_scorers(cuda_device, shape, n_ent, n_rel, B, k):
    """At BASELINE.json's batch shapes, where the oracle is too slow: size-independent properties of the fed scorers
    (per-triple, grouped, and the TransH instance of the score family) — two half batches add up to the whole batch,
    a permutation of the batch changes nothing, and grouped == per-triple."""
    eng = _engine()
    rng = np.random.default_rng(12)
    d = 100
    ent = (rng.standard_normal((n_ent, d)) / 10).astype(np.float32)
    rel = (rng.standard_normal((n_rel, d)) / 10).astype(np.float32)
    nrm = (rng.standard_normal((n_rel, d)) / 10).astype(np.float32)
    pos = np.stack([rng.integers(0, n_ent, B), rng.integers(0, n_rel, B), rng.integers(0, n_ent, B)]).astype(np.int32)
    neg = np.repeat(pos, k, axis=1)
    side = rng.random(B * k) < 0.5
    neg[0, side] = rng.integers(0, n_ent, side.sum())
    neg[2, ~side] = rng.integers(0, n_ent, (~side).sum())
    cfg = eng.loss_cfg("limited", "L2", 0.3, 2.2, 0.2)

    def triple(grouped=False, batches=((slice(None), slice(None)),)):
        te, tr = eng.EmbeddingTable(ent, True), eng.EmbeddingTable(rel, True)
        t = eng.TripleTrainer(te, tr, cfg, 0.01)
        for ps, ns in batches:
            t.score_fed(_dev(pos[:, ps]), _dev(neg[:, ns]), grouped=grouped)
        return t.read_loss(), te.grad.clone(), tr.grad.clone()

    def close(a, b):
        assert a[0] == pytest.approx(b[0], rel=1e-5)
        for x, y in zip(a[1:], b[1:]):
            scale = float(y.abs().max())
            assert float((x - y).abs().max()) <= 2e-4 * scale
    whole = triple()
    half = B // 2
    close(triple(batches=((slice(0, half), slice(0, half * k)), (slice(half, B), slice(half * k, B * k)))), whole)
    close(triple(grouped=True), whole)
    perm = rng.permutation(B)
    pos_p, neg_p = pos[:, perm], neg.reshape(3, B, k)[:, perm].reshape(3, B * k)
    te, tr = eng.EmbeddingTable(ent, True), eng.EmbeddingTable(rel, True)
    t = eng.TripleTrainer(te, tr, cfg, 0.01)
    t.score_fed(_dev(pos_p), _dev(neg_p), grouped=True)
    close((t.read_loss(), te.grad, tr.grad), whole)
    # the TransH instance of the score family at the same size: additivity
    def transh(batches):
        tabs = (eng.EmbeddingTable(ent, True), eng.EmbeddingTable(rel, True), None, eng.EmbeddingTable(nrm, True))
        m = eng.ModelTrainer("TransH", tabs, cfg, 0.01)
        for ps, ns in batches:
            m.score_fed(_dev(pos[:, ps]), _dev(neg[:, ns]))
        return m.read_loss(), tabs[0].grad.clone(), tabs[1].grad.clone(), tabs[3].grad.clone()
    close(transh(((slice(0, half), slice(0, half * k)), (slice(half, B), slice(half * k, B * k)))),
          transh(((slice(None), slice(None)),)))


@pytest.mark.parametrize("opt", ["Adagrad", "SGD"])
@pytest.mark.parametrize("loss,k,d", [("limited", 10, 100), ("margin-based", 1, 75), ("logistic", 4, 200)])
def test_one_launch_fed_step_equals_the_two_launch_path(cuda_device, monkeypatch, opt, loss, k, d):
    """oea_triple_step_fed_grouped (grouped scoring + grid barrier + row optimiser, one cooperative launch) against
    score_fed + apply from the same tables, three steps; then the host-index step with OEA_FED_FUSED=1 against the
    default."""
    eng = _engine()
    from tests.helpers import make_tables
    rng = np.random.default_rng(11 * d + k)
    n_ent, n_rel, n_pos = 3000, 31, 700
    ent, rel = make_tables(rng, n_ent, n_rel, d)
    kw = dict(margin=1.1 if loss == "margin-based" else 0.3, neg_margin=2.2, balance=0.2)
    cfg = eng.loss_cfg(loss, "L2", **kw)
    make = lambda: eng.TripleTrainer(eng.EmbeddingTable(ent, True, opt), eng.EmbeddingTable(rel, True, opt), cfg, 0.01)
    fused, split = make(), make()
    batches = [make_batch(rng, n_ent, n_rel, n_pos, k) for _ in range(3)]
    for pos, neg in batches:
        fused.step_fed_grouped(_dev(pos), _dev(neg))
        split.score_fed(_dev(pos), _dev(neg))
        split.apply()
        assert fused.read_loss() == pytest.approx(split.read_loss(), rel=1e-5)
    torch.cuda.synchronize()
    for x, y in ((fused.ent, split.ent), (fused.rel, split.rel)):
        _assert_rows_close(x.raw().cpu().numpy(), y.raw().cpu().numpy(), "table after three one-launch steps")
        assert not x.grad.any().item() and not x.touched.any().item()
    res = []
    for flag in ("0", "1"):
        monkeypatch.setenv("OEA_FED_FUSED", flag)
        t = make()
        res.append(([t.step_fed_host(p, n) for p, n in batches], t.ent.raw().cpu().numpy()))
    np.testing.assert_allclose(res[1][0], res[0][0], rtol=1e-4)
    _assert_rows_close(res[1][1], res[0][1], "entity table after host-index steps with OEA_FED_FUSED")
