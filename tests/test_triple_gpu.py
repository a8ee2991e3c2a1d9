"""GPU parity tests of path (i): the CUDA kernels (through the C-ABI) against the CPU oracle on identical
fed index batches.  Tolerance: 1e-4 relative on the fp32 loss (BASELINE.json north_star), 1e-4 relative
(plus a small absolute floor tied to the gradient scale) on per-row gradients and updated tables."""
import numpy as np
import pytest
import torch

from oracle import triple as orc
from tests.helpers import make_batch, make_tables

pytestmark = pytest.mark.gpu

LOSS_TOL = 1e-4


def _engine():
    from openea_b200 import engine
    return engine


def _tables(ent, rel, norm, opt="Adagrad"):
    eng = _engine()
    return eng.EmbeddingTable(ent, norm, opt), eng.EmbeddingTable(rel, norm, opt)


def _dev(hrt):
    return None if hrt is None else torch.from_numpy(np.ascontiguousarray(hrt)).cuda()


def _assert_rows_close(got, want, what):
    scale = max(1e-6, float(np.abs(want).max()))
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=2e-5 * scale, err_msg=what)


@pytest.mark.parametrize("loss,k", [("limited", 10), ("logistic", 4), ("positive", 0), ("logsigmoid", 0), ("margin-based", 1)])
@pytest.mark.parametrize("loss_norm", ["L1", "L2"])
@pytest.mark.parametrize("norm", [True, False])
@pytest.mark.parametrize("d", [75, 100, 300])
def test_fed_forward_backward_matches_oracle(cuda_device, loss, k, loss_norm, norm, d):
    eng = _engine()
    rng = np.random.default_rng(99 + d + 7 * k)
    n_ent, n_rel, n_pos = 2000, 37, 500
    ent, rel = make_tables(rng, n_ent, n_rel, d)
    pos, neg = make_batch(rng, n_ent, n_rel, n_pos, k)
    kw = dict(margin=1.1 if loss == "margin-based" else 0.3, neg_margin=2.2, balance=0.2)
    want_loss, want_ge, want_gr, _ = orc.fwd_bwd(ent, rel, pos, neg, loss, loss_norm, norm, norm, **kw)

    te, tr = _tables(ent, rel, norm)
    tr_ = eng.TripleTrainer(te, tr, eng.loss_cfg(loss, loss_norm, **kw), lr=0.01)
    tr_.score_fed(_dev(pos), _dev(neg))
    got_loss = tr_.read_loss()
    assert got_loss == pytest.approx(want_loss, rel=LOSS_TOL)
    got_ge = te.grad[:, :d].cpu().numpy()
    got_gr = tr.grad[:, :d].cpu().numpy()
    if loss_norm == "L1":
        # sign(u) may flip where |u| is at fp32 rounding level; bound the number of disagreeing coordinates
        bad = np.abs(got_ge - want_ge) > 1e-4 * max(1.0, np.abs(want_ge).max())
        assert bad.mean() < 1e-3
    else:
        _assert_rows_close(got_ge, want_ge, "entity gradient")
        _assert_rows_close(got_gr, want_gr, "relation gradient")
    assert not te.grad[:, d:].any().item(), "padding columns must stay zero"
    touched = te.touched.cpu().numpy().astype(bool)
    assert (np.abs(want_ge).sum(1)[~touched] == 0).all(), "untouched rows must have zero oracle gradient"


@pytest.mark.parametrize("opt", ["Adagrad", "SGD", "Adam"])
def test_optimizer_step_equals_dense_tf_step(cuda_device, opt):
    """One full step equals the oracle's DENSE TF-style step on every row, touched or not (SURVEY §7 (3))."""
    eng = _engine()
    rng = np.random.default_rng(5)
    d, n_ent, n_rel = 100, 3000, 41
    ent, rel = make_tables(rng, n_ent, n_rel, d)
    pos, neg = make_batch(rng, n_ent, n_rel, 400, 10)
    kw = dict(margin=0.01, neg_margin=2.0, balance=0.2)
    st = orc.DenseState(ent, rel, opt)
    te, tr = _tables(ent, rel, True, opt)
    trn = eng.TripleTrainer(te, tr, eng.loss_cfg("limited", "L2", **kw), lr=0.01)
    for _ in range(3):
        want = orc.step(st, pos, neg, "limited", "L2", True, True, 0.01, **kw)
        trn.score_fed(_dev(pos), _dev(neg))
        trn.apply()
        assert trn.read_loss() == pytest.approx(want, rel=LOSS_TOL)
    np.testing.assert_allclose(te.raw().cpu().numpy(), st.ent, rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(tr.raw().cpu().numpy(), st.rel, rtol=1e-4, atol=1e-6)
    if opt == "Adagrad":
        np.testing.assert_allclose(te.state1[:, :d].cpu().numpy(), st.ent_s1, rtol=1e-4, atol=1e-7)
    assert not te.grad.any().item() and not te.touched.any().item(), "apply must leave grad/touched cleared"


def test_ten_step_loss_trajectory_config2(cuda_device):
    """10 consecutive BootEA-config steps from identical state: loss trajectory within 1e-4 rel (SURVEY §7 (4))."""
    eng = _engine()
    rng = np.random.default_rng(11)
    d, n_ent, n_rel = 100, 6000, 90
    ent, rel = make_tables(rng, n_ent, n_rel, d)
    kw = dict(margin=0.01, neg_margin=2.0, balance=0.2)
    st = orc.DenseState(ent, rel, "Adagrad")
    te, tr = _tables(ent, rel, True)
    trn = eng.TripleTrainer(te, tr, eng.loss_cfg("limited", "L2", **kw), lr=0.01)
    for step in range(10):
        pos, neg = make_batch(rng, n_ent, n_rel, 1000, 10)
        want = orc.step(st, pos, neg, "limited", "L2", True, True, 0.01, **kw)
        got = trn.step_fed_host(pos, neg)   # the session.run(feed_dict) boundary, host buffers
        assert got == pytest.approx(want, rel=LOSS_TOL), "step %d" % step
    np.testing.assert_allclose(te.raw().cpu().numpy(), st.ent, rtol=2e-4, atol=2e-6)


def test_lookup_returns_normalised_rows(cuda_device):
    rng = np.random.default_rng(3)
    ent, rel = make_tables(rng, 500, 7, 75)
    te, _ = _tables(ent, rel, True)
    ids = rng.integers(0, 500, size=64).astype(np.int32)
    got = te.lookup(ids).cpu().numpy()
    np.testing.assert_allclose(got, orc.l2_normalize(ent)[ids], rtol=1e-5, atol=1e-7)
    assert te.lookup().shape == (500, 75)


def test_empty_and_ragged_batches(cuda_device):
    eng = _engine()
    rng = np.random.default_rng(2)
    ent, rel = make_tables(rng, 100, 5, 100)
    te, tr = _tables(ent, rel, True)
    trn = eng.TripleTrainer(te, tr, eng.loss_cfg("limited", "L2", margin=0.01, neg_margin=2.0, balance=0.2), lr=0.01)
    empty = torch.zeros(3, 0, dtype=torch.int32, device="cuda")
    trn.score_fed(empty, empty)
    assert trn.read_loss() == 0.0
    # ragged: negatives not a multiple of positives (limited loss sums are independent, losses.py:53-55)
    pos, _ = make_batch(rng, 100, 5, 7, 0)
    _, neg = make_batch(rng, 100, 5, 3, 5)
    want, _, _, _ = orc.fwd_bwd(ent, rel, pos, neg, "limited", "L2", True, True, margin=0.01, neg_margin=2.0, balance=0.2)
    trn.score_fed(_dev(pos), _dev(neg))
    assert trn.read_loss() == pytest.approx(want, rel=LOSS_TOL)
    # margin loss requires paired batches (args_hander.py:19-21): the ABI reports a shape error
    bad = eng.TripleTrainer(te, tr, eng.loss_cfg("margin-based", "L2", margin=1.0), lr=0.01)
    from openea_b200.lib import OeaError
    with pytest.raises(OeaError):
        bad.score_fed(_dev(pos), _dev(neg))


def _decode_dbg(dbg, kgs_triples, k):
    """Rebuild the (pos, neg) index batch the fused kernel sampled from its debug dump."""
    pos_cols, neg_cols = [], []
    for row in dbg:
        tri, mask = int(row[0]), int(row[1])
        q = 1 if tri & (1 << 30) else 0
        h, r, t = kgs_triples[q][tri & ~(1 << 30)]
        pos_cols.append((h, r, t))
        for j in range(k):
            e = int(row[2 + j])
            neg_cols.append((e, r, t) if (mask >> j) & 1 else (h, r, e))
    neg = np.array(neg_cols, dtype=np.int32).T.copy() if neg_cols else np.zeros((3, 0), dtype=np.int32)
    return np.array(pos_cols, dtype=np.int32).T.copy(), neg


@pytest.mark.parametrize("cand,loss,k,d,norm,loss_norm", [
    (None, "limited", 10, 100, True, "L2"), ("by_id", "limited", 10, 100, True, "L2"),
    ("ent2row", "limited", 10, 100, True, "L2"),
    ("ent2row", "limited", 10, 100, True, "L1"),     # the warp-per-positive kernel on the same case
    (None, "logistic", 7, 75, True, "L2"), ("by_id", "limited", 5, 128, False, "L2"),
    (None, "margin-based", 1, 100, True, "L2"), (None, "margin-based", 1, 100, True, "L1"),
    (None, "positive", 0, 75, True, "L2"), (None, "limited", 32, 64, True, "L2"),
    (None, "limited", 10, 300, True, "L2"),          # pitch > 128: the warp-per-positive kernel
])
def test_sampled_step_replays_through_oracle(cuda_device, cand, loss, k, d, norm, loss_norm):
    """The fused sampler+scorer (the octet layouts for L2 at pitch <= 128, the warp-per-positive kernel otherwise):
    (a) its sampled batch obeys batch.py's rules, (b) replaying that exact batch through the oracle reproduces loss and
    gradients.  `cand`: truncated candidate lists, indexed by entity id or through ent2row."""
    eng = _engine()
    rng = np.random.default_rng(21 + k + d)
    n_ent, n_rel, B = 4000, 30, 512
    ent, rel = make_tables(rng, n_ent, n_rel, d)
    ents1 = np.arange(0, n_ent, 2, dtype=np.int32)
    ents2 = np.arange(1, n_ent, 2, dtype=np.int32)

    def mk_triples(ents, n, rlo, rhi):
        tri = np.stack([rng.choice(ents, n), rng.integers(rlo, rhi, n), rng.choice(ents, n)], 1).astype(np.int32)
        return np.unique(tri, axis=0)
    t1, t2 = mk_triples(ents1, 3000, 0, 15), mk_triples(ents2, 2500, 15, 30)
    kg1, kg2 = eng.DeviceKG(t1, ents1, n_ent), eng.DeviceKG(t2, ents2, n_ent)
    n_cand = 40
    if cand is not None:
        for kg, ents in ((kg1, ents1), (kg2, ents2)):
            rows = torch.from_numpy(rng.choice(ents, size=(len(ents), n_cand)).astype(np.int32)).cuda()
            # distinct ids per row are not required by the sampler (it samples distinct POSITIONS);
            # both layouts of the candidate matrix are exercised: by entity id (default) and via ent2row
            kg.set_candidates(rows, ents, direct=cand == "by_id")
    tset = eng.DeviceTripleSet([kg1.triples, kg2.triples], n_ent, n_rel)
    kw = dict(margin=1.2 if loss == "margin-based" else 0.01, neg_margin=2.0, balance=0.2)
    te, tr = _tables(ent, rel, norm)
    trn = eng.TripleTrainer(te, tr, eng.loss_cfg(loss, loss_norm, **kw), lr=0.01)
    all_set = {tuple(x) for x in t1.tolist()} | {tuple(x) for x in t2.tolist()}
    seen_tri = [set(), set()]
    T1, T2 = len(t1), len(t2)
    b1 = int(T1 / (T1 + T2) * B); b2 = B - b1
    steps = int(np.ceil((T1 + T2) / B))
    for step in range(steps):
        dbg = torch.full((B, 2 + k), -1, dtype=torch.int32, device="cuda")
        npos = torch.zeros(1, dtype=torch.int32, device="cuda")
        trn.score_sampled(kg1, kg2, tset, B, k, step, epoch_seed=777, dbg=dbg, n_pos_out=npos)
        n = int(npos.item())
        n1 = max(0, min((step + 1) * b1, T1) - min(step * b1, T1)); n2 = max(0, min((step + 1) * b2, T2) - min(step * b2, T2))
        assert n == n1 + n2
        rows = dbg.cpu().numpy()[:n]
        pos, neg = _decode_dbg(rows, (t1, t2), k)
        for row in rows:
            q = 1 if int(row[0]) & (1 << 30) else 0
            seen_tri[q].add(int(row[0]) & ~(1 << 30))
        if k > 0:
            # (a) sampler rules: same-KG corruption, filtered against the known triples
            ent_kg = np.where(np.isin(neg[0], ents1) & np.isin(neg[2], ents1), 0, np.where(np.isin(neg[0], ents2) & np.isin(neg[2], ents2), 1, -1))
            assert (ent_kg >= 0).all(), "negatives must stay inside the positive's KG"
            in_set = np.mean([tuple(x) in all_set for x in neg.T.tolist()])
            assert in_set < 0.01, "true triples must be (almost always) rejected"
            blocks = neg.reshape(3, n, k)
            if k <= 20 and cand is None:
                dup = np.mean([len({tuple(c) for c in blocks[:, i, :].T.tolist()}) < k for i in range(n)])
                assert dup < 0.05, "negatives of one positive are distinct except across rare re-tries"
        else:
            neg = None
        # (b) replay through the oracle
        want, want_ge, want_gr, _ = orc.fwd_bwd(ent, rel, pos, neg, loss, loss_norm, norm, norm, **kw)
        assert trn.read_loss() == pytest.approx(want, rel=LOSS_TOL)
        got_ge = te.grad[:, :d].cpu().numpy()
        if loss_norm == "L1":       # sign(u) may flip where |u| is at fp32 rounding level, as in the fed test above
            assert (np.abs(got_ge - want_ge) > 1e-4 * max(1.0, np.abs(want_ge).max())).mean() < 1e-3
        else:
            _assert_rows_close(got_ge, want_ge, "entity gradient (sampled)")
            _assert_rows_close(tr.grad[:, :d].cpu().numpy(), want_gr, "relation gradient (sampled)")
        assert not te.grad[:, d:].any().item()
        te.grad.zero_(); tr.grad.zero_(); te.touched.zero_(); tr.touched.zero_()
    # the epoch permutation is a bijection: slices partition (a prefix of) each triple list exactly once
    assert len(seen_tri[0]) == min(T1, steps * b1) and len(seen_tri[1]) == min(T2, steps * b2)


def _sampled_world(rng, eng, n_ent=4000, n_rel=30):
    ents1 = np.arange(0, n_ent, 2, dtype=np.int32)
    ents2 = np.arange(1, n_ent, 2, dtype=np.int32)

    def mk(ents, n, rlo, rhi):
        tri = np.stack([rng.choice(ents, n), rng.integers(rlo, rhi, n), rng.choice(ents, n)], 1).astype(np.int32)
        return np.unique(tri, axis=0)
    t1, t2 = mk(ents1, 3000, 0, 15), mk(ents2, 2500, 15, 30)
    kg1, kg2 = eng.DeviceKG(t1, ents1, n_ent), eng.DeviceKG(t2, ents2, n_ent)
    return kg1, kg2, eng.DeviceTripleSet([kg1.triples, kg2.triples], n_ent, n_rel)


@pytest.mark.parametrize("opt,d,loss,k", [("Adagrad", 100, "limited", 10), ("SGD", 75, "logistic", 4),
                                          ("Adagrad", 128, "margin-based", 1), ("Adagrad", 64, "positive", 0)])
def test_single_launch_step_equals_two_launch_step(cuda_device, opt, d, loss, k):
    """oea_triple_step_sampled as ONE cooperative launch (score, grid barrier, row optimiser) leaves the tables,
    the optimiser slots, the flags and the loss exactly where the two-launch path (score_sampled: the same score
    kernel, then apply: k_rowopt_pair) leaves them — up to the order of the float atomics in the gradient rows."""
    eng = _engine()
    rng = np.random.default_rng(5 + d)
    ent, rel = make_tables(rng, 4000, 30, d)
    kg1, kg2, tset = _sampled_world(rng, eng)
    kw = dict(margin=1.2 if loss == "margin-based" else 0.01, neg_margin=2.0, balance=0.2)
    out = {}
    for mode in ("fused", "split"):
        te, tr = _tables(ent, rel, True, opt)
        trn = eng.TripleTrainer(te, tr, eng.loss_cfg(loss, "L2", **kw), lr=0.05)
        losses = []
        for step in range(6):
            if mode == "fused":
                trn.step_sampled(kg1, kg2, tset, 512, k, step, epoch_seed=99)
            else:
                trn.score_sampled(kg1, kg2, tset, 512, k, step, epoch_seed=99)
                trn.apply()
            losses.append(trn.read_loss())
        assert not te.grad.any().item() and not tr.grad.any().item(), "gradient rows are zeroed by the optimiser"
        assert not te.touched.any().item() and not tr.touched.any().item(), "row flags are cleared"
        out[mode] = (te.weight.cpu().numpy(), tr.weight.cpu().numpy(),
                     None if opt == "SGD" else te.state1.cpu().numpy(), losses)
    a, b = out["fused"], out["split"]
    assert np.abs(a[0] - ent_pad(ent, a[0].shape[1])).max() > 1e-4, "the step moved the table"
    np.testing.assert_allclose(a[0], b[0], rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(a[1], b[1], rtol=2e-5, atol=2e-6)
    if a[2] is not None:
        np.testing.assert_allclose(a[2], b[2], rtol=2e-5, atol=1e-7)
    np.testing.assert_allclose(a[3], b[3], rtol=1e-5)


def ent_pad(x, pitch):
    out = np.zeros((x.shape[0], pitch), dtype=np.float32)
    out[:, :x.shape[1]] = x
    return out


def test_single_launch_step_inside_a_cuda_graph(cuda_device):
    """The cooperative launch is capturable: an epoch graph replays to the same tables as the eager steps."""
    eng = _engine()
    rng = np.random.default_rng(77)
    ent, rel = make_tables(rng, 4000, 30, 100)
    kg1, kg2, tset = _sampled_world(rng, eng)
    res = []
    for graph in (False, True):
        te, tr = _tables(ent, rel, True)
        trn = eng.TripleTrainer(te, tr, eng.loss_cfg("limited", "L2", margin=0.01, neg_margin=2.0, balance=0.2), lr=0.05)
        if graph:
            g = trn.capture_epoch(kg1, kg2, tset, 512, 10, 5)
            g.replay(4242)           # capture itself executes nothing
        else:
            seed_dev = torch.tensor([4242], dtype=torch.int64, device="cuda")
            for step in range(5):
                trn.step_sampled(kg1, kg2, tset, 512, 10, step, epoch_seed=0, dev_seed=seed_dev)
        torch.cuda.synchronize()
        res.append((te.weight.cpu().numpy(), trn.read_loss()))
    np.testing.assert_allclose(res[0][0], res[1][0], rtol=2e-5, atol=2e-6)
    assert res[0][1] == pytest.approx(res[1][1], rel=1e-5)
