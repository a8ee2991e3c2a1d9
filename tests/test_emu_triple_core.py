"""CPU: the core of path (i) — oea_triple.cu's fed scorers, the row optimisers, the normalised lookup and its backward,
the tensor-level losses, the on-device triple set and the warp-per-positive sampled scorer — executed from the product's
kernel SOURCE on the warp emulator (tests/emu) through the product's own Python engine over CPU tensors, against the C
oracle.  These kernels are verified on the GPU by tests/test_triple_gpu.py; here the same checks guard refactors where
no GPU exists.  The octet scorer and the one-launch step (a cooperative kernel, run as one block here) are at the end."""
import ctypes as C

import numpy as np
import pytest
import torch

from openea_b200 import engine as eng
from openea_b200 import lib as L
from oracle import triple as orc
from tests.emu import build_emu
from tests.helpers import make_batch, make_tables
from tests.kernel_edge_cases import decode_dbg


@pytest.fixture()
def cpu_engine(monkeypatch):
    so = build_emu.build()
    if so is None:
        pytest.skip("no CUDA headers for the emulator build")
    lib = C.CDLL(so)
    for name, (res, args) in L.SIGNATURES.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    monkeypatch.setattr(L, "load", lambda: lib)
    monkeypatch.setattr(eng, "_stream_ptr", lambda: C.c_void_p(0))
    return eng


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


@pytest.mark.parametrize("loss,k", [("limited", 3), ("logistic", 2), ("positive", 0), ("logsigmoid", 0), ("margin-based", 1)])
@pytest.mark.parametrize("loss_norm,norm,d", [("L2", True, 12), ("L1", False, 75), ("L2", True, 200)])
def test_emulated_fed_scorers_match_the_c_oracle(cpu_engine, loss, k, loss_norm, norm, d):
    rng = np.random.default_rng(d + k)
    n_ent, n_rel, n_pos = 40, 5, 19
    ent, rel = make_tables(rng, n_ent, n_rel, d)
    pos, neg = make_batch(rng, n_ent, n_rel, n_pos, k)
    kw = dict(margin=1.1 if loss == "margin-based" else 0.3, neg_margin=2.2, balance=0.2)
    want_loss, want_ge, want_gr, _ = orc.fwd_bwd(ent, rel, pos, neg, loss, loss_norm, norm, norm, **kw)
    te, tr = cpu_engine.EmbeddingTable(ent, norm, device="cpu"), cpu_engine.EmbeddingTable(rel, norm, device="cpu")
    t = cpu_engine.TripleTrainer(te, tr, cpu_engine.loss_cfg(loss, loss_norm, **kw), 0.01)
    t.score_fed(_t(pos), None if neg is None else _t(neg))
    assert t.read_loss() == pytest.approx(want_loss, rel=1e-4)
    for tab, want in ((te, want_ge), (tr, want_gr)):
        got = tab.grad[:, :d].numpy()
        if loss_norm == "L1":
            assert (np.abs(got - want) > 1e-4 * max(1.0, np.abs(want).max())).mean() < 5e-3
        else:
            np.testing.assert_allclose(got, want, rtol=1e-4, atol=2e-5 * max(1e-6, np.abs(want).max()))


@pytest.mark.parametrize("opt", ["Adagrad", "SGD", "Adam"])
def test_emulated_training_steps_equal_dense_tf_steps(cpu_engine, opt):
    rng = np.random.default_rng(5)
    d, n_ent, n_rel = 20, 60, 7
    ent, rel = make_tables(rng, n_ent, n_rel, d)
    kw = dict(margin=0.01, neg_margin=2.0, balance=0.2)
    st = orc.DenseState(ent, rel, opt)
    te, tr = cpu_engine.EmbeddingTable(ent, True, opt, device="cpu"), cpu_engine.EmbeddingTable(rel, True, opt, device="cpu")
    t = cpu_engine.TripleTrainer(te, tr, cpu_engine.loss_cfg("limited", "L2", **kw), 0.01)
    for _ in range(3):
        pos, neg = make_batch(rng, n_ent, n_rel, 16, 3)
        want = orc.step(st, pos, neg, "limited", "L2", True, True, 0.01, **kw)
        t.score_fed(_t(pos), _t(neg))
        t.apply()                                                    # oea_rowopt_apply_pair (Adam: two dense launches)
        assert t.read_loss() == pytest.approx(want, rel=1e-4)
    np.testing.assert_allclose(te.raw().numpy(), st.ent, rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(tr.raw().numpy(), st.rel, rtol=1e-4, atol=1e-6)
    assert not te.grad.any() and not te.touched.any()


def test_emulated_lookup_scatter_and_tensor_level_losses(cpu_engine):
    rng = np.random.default_rng(2)
    ent, _ = make_tables(rng, 30, 3, 10)
    te = cpu_engine.EmbeddingTable(ent, True, device="cpu")
    ids = rng.integers(0, 30, 11).astype(np.int32)
    got = te.lookup(ids)
    np.testing.assert_allclose(got.numpy(), orc.l2_normalize(ent)[ids], rtol=1e-5, atol=1e-7)
    # backward of the lookup: gradient of Σ w·normalise(x) w.r.t. x, accumulated over repeated ids
    w = rng.standard_normal((11, 10)).astype(np.float32)
    x = torch.tensor(ent, dtype=torch.float64, requires_grad=True)
    xn = x * torch.rsqrt(torch.clamp((x * x).sum(1, keepdim=True), min=1e-12))
    (xn[torch.as_tensor(ids, dtype=torch.long)] * torch.as_tensor(w, dtype=torch.float64)).sum().backward()
    te.scatter_grad(_t(w), ids)
    np.testing.assert_allclose(te.grad[:, :10].numpy(), x.grad.numpy(), rtol=1e-4, atol=1e-6)
    assert set(np.flatnonzero(te.touched.numpy())) == set(ids.tolist())


def test_emulated_triple_set_and_sampled_scorer_replay(cpu_engine):
    """oea_tripleset_build + the sampled kernels at d = 12 (the duo for L2, the warp-per-positive kernel for L1): the
    debug dump, replayed through the fed scorer, gives the same loss and gradients (the check tests/test_triple_gpu.py
    makes on the GPU)."""
    rng = np.random.default_rng(8)
    n, n_rel, d = 50, 4, 12
    def kg(lo):
        t = np.stack([rng.integers(lo, lo + n, 120), rng.integers(0, n_rel, 120), rng.integers(lo, lo + n, 120)], 1)
        return np.unique(t.astype(np.int32), axis=0)
    t1, t2 = kg(0), kg(n)
    ent, rel = make_tables(rng, 2 * n, n_rel, d)
    kg1 = cpu_engine.DeviceKG(t1, np.arange(0, n), 2 * n, device="cpu")
    kg2 = cpu_engine.DeviceKG(t2, np.arange(n, 2 * n), 2 * n, device="cpu")
    tset = cpu_engine.DeviceTripleSet([kg1.triples, kg2.triples], 2 * n, n_rel, device="cpu")
    from tests.test_emu_sampler import build_tripleset
    want_slots, _ = build_tripleset(np.concatenate([t1, t2]), tset.ent_bits, tset.rel_bits, capacity=tset.capacity)
    assert set(tset.slots.numpy().view(np.uint64).tolist()) == set(want_slots.tolist())       # same keys (probe order may differ)
    B, k = 32, 3
    for loss_norm in ("L2", "L1"):
        cfg = cpu_engine.loss_cfg("limited", loss_norm, 0.1, 2.0, 0.2)
        make = lambda: cpu_engine.TripleTrainer(cpu_engine.EmbeddingTable(ent, True, device="cpu"),
                                                cpu_engine.EmbeddingTable(rel, True, device="cpu"), cfg, 0.01)
        a = make()
        dbg = torch.zeros(B, 2 + k, dtype=torch.int32)
        n_pos = torch.zeros(1, dtype=torch.int32)
        a.score_sampled(kg1, kg2, tset, B, k, 1, 4242, dbg=dbg, n_pos_out=n_pos)
        pos, neg = decode_dbg(dbg.numpy()[:int(n_pos)], t1, t2, k)
        b = make()
        b.score_fed(_t(pos), _t(neg))
        assert a.read_loss() == pytest.approx(b.read_loss(), rel=1e-5), loss_norm
        np.testing.assert_allclose(a.ent.grad.numpy(), b.ent.grad.numpy(), rtol=1e-4, atol=1e-6, err_msg=loss_norm)
        np.testing.assert_allclose(a.rel.grad.numpy(), b.rel.grad.numpy(), rtol=1e-4, atol=1e-6, err_msg=loss_norm)


def _normed(x, on):
    return x * torch.rsqrt(torch.clamp((x * x).sum(1, keepdim=True), min=1e-12)) if on else x


@pytest.mark.parametrize("paths,reciprocal", [(False, False), (True, True), (False, True)])
@pytest.mark.parametrize("loss_norm,norm,d", [("L2", True, 12), ("L1", False, 75), ("L2", True, 200)])
def test_emulated_weighted_margin_scorer_matches_autograd(cpu_engine, paths, reciprocal, loss_norm, norm, d):
    """oea_triple_score_margin_weighted (IPTransE's alignment and path losses, iptranse.py:170-180) against float64
    autograd of the formula as written there; `paths`: all three rows of a triple come from the relation table."""
    rng = np.random.default_rng(d + 3 * paths + reciprocal)
    n_ent, n_rel, n = 30, 9, 23
    ent, rel = make_tables(rng, n_ent, n_rel, d)
    hi = n_rel if paths else n_ent
    pos = np.stack([rng.integers(0, hi, n), rng.integers(0, n_rel, n), rng.integers(0, hi, n)]).astype(np.int32)
    neg = np.stack([rng.integers(0, hi, n), rng.integers(0, n_rel, n), rng.integers(0, hi, n)]).astype(np.int32)
    w = (rng.random(n) * 3 + 0.5).astype(np.float32)
    w[3] = 0.0 if not reciprocal else w[3]
    margin, scale = 0.8, 0.1 if paths else 1.0

    E = torch.tensor(ent, dtype=torch.float64, requires_grad=True)
    R = torch.tensor(rel, dtype=torch.float64, requires_grad=True)
    En, Rn = _normed(E, norm), _normed(R, norm)
    A = Rn if paths else En

    def score(b):
        u = A[b[0].astype(np.int64)] + Rn[b[1].astype(np.int64)] - A[b[2].astype(np.int64)]
        return u.abs().sum(1) if loss_norm == "L1" else (u * u).sum(1)
    wt = torch.tensor(w, dtype=torch.float64)
    wt = 1.0 / wt if reciprocal else wt
    want = scale * (wt * torch.relu(margin + score(pos) - score(neg))).sum()
    want.backward()

    te, tr = cpu_engine.EmbeddingTable(ent, norm, device="cpu"), cpu_engine.EmbeddingTable(rel, norm, device="cpu")
    t = cpu_engine.TripleTrainer(te, tr, cpu_engine.loss_cfg("margin-based", loss_norm, margin=margin), 0.01)
    t.score_margin_weighted(_t(pos), _t(neg), _t(w), reciprocal=reciprocal, scale=scale, paths=paths)
    assert t.read_loss() == pytest.approx(float(want.detach()), rel=1e-4)
    for tab, ref in ((te, E), (tr, R)):
        g = np.zeros_like(ent if tab is te else rel) if ref.grad is None else ref.grad.numpy()
        got = tab.grad[:, :d].numpy()
        if loss_norm == "L1":
            assert (np.abs(got - g) > 1e-4 * max(1.0, np.abs(g).max())).mean() < 5e-3
        else:
            np.testing.assert_allclose(got, g, rtol=1e-4, atol=2e-5 * max(1e-6, np.abs(g).max()))
    if paths:
        assert not te.touched.any()
    # unweighted call == the plain margin scorer
    t2 = cpu_engine.TripleTrainer(cpu_engine.EmbeddingTable(ent, norm, device="cpu"),
                                  cpu_engine.EmbeddingTable(rel, norm, device="cpu"),
                                  cpu_engine.loss_cfg("margin-based", loss_norm, margin=margin), 0.01)
    t3 = cpu_engine.TripleTrainer(cpu_engine.EmbeddingTable(ent, norm, device="cpu"),
                                  cpu_engine.EmbeddingTable(rel, norm, device="cpu"),
                                  cpu_engine.loss_cfg("margin-based", loss_norm, margin=margin), 0.01)
    if not paths:
        t2.score_margin_weighted(_t(pos), _t(neg))
        t3.score_fed(_t(pos), _t(neg))
        assert t2.read_loss() == pytest.approx(t3.read_loss(), rel=1e-6)
        np.testing.assert_allclose(t2.ent.grad.numpy(), t3.ent.grad.numpy(), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("norm,d,weighted", [(True, 12, False), (False, 75, True), (True, 300, True)])
def test_emulated_pair_distance_loss_matches_autograd(cpu_engine, norm, d, weighted):
    rng = np.random.default_rng(d)
    ent, rel = make_tables(rng, 25, 2, d)
    a = rng.integers(0, 25, 17).astype(np.int32)
    b = rng.integers(0, 25, 17).astype(np.int32)
    b[0] = a[0]                                                    # a pair of one entity with itself: no loss, no gradient
    w = (rng.random(17) + 0.1).astype(np.float32) if weighted else None
    E = torch.tensor(ent, dtype=torch.float64, requires_grad=True)
    En = _normed(E, norm)
    dist = ((En[a.astype(np.int64)] - En[b.astype(np.int64)]) ** 2).sum(1)
    want = 0.7 * ((torch.tensor(w, dtype=torch.float64) * dist).sum() if weighted else dist.sum())
    want.backward()
    te = cpu_engine.EmbeddingTable(ent, norm, device="cpu")
    t = cpu_engine.TripleTrainer(te, cpu_engine.EmbeddingTable(rel, norm, device="cpu"),
                                 cpu_engine.loss_cfg("margin-based", "L2", margin=1.0), 0.01)
    t.score_pairs(a, b, None if w is None else _t(w), scale=0.7)
    assert t.read_loss() == pytest.approx(float(want.detach()), rel=1e-4)
    np.testing.assert_allclose(te.grad[:, :d].numpy(), E.grad.numpy(), rtol=1e-4, atol=2e-5 * float(E.grad.abs().max()))
    assert set(np.flatnonzero(te.touched.numpy())) <= set(a.tolist()) | set(b.tolist())


@pytest.fixture(params=["duo", "oct"])
def octet_k(request):
    """Negatives per positive that reach each octet-layout kernel at squared L2, pitch <= 128: the duo (two positives
    per warp) takes k <= 16, the octet (one positive per warp) k = 17 … 32.  The one-launch step is launched as one
    block on the emulator, so its grid barrier is the block's."""
    return {"duo": 6, "oct": 20}[request.param]


def test_emulated_duo_and_octet_scorers_sample_the_same_batch(cpu_engine):
    """Every sampled kernel draws the same batch from the same seed (the sampler does not read the score kind): the
    debug dump of the squared-L2 kernel (the duo, or the octet at k = 20) equals that of the warp-per-positive kernel at
    L1, and each kernel's loss, gradients and row flags equal the fed scorer's on its decoded dump.  Odd and even
    numbers of positives, k = 0 / 1 (margin) / 6 / 16 / 20, sharded launches included."""
    rng = np.random.default_rng(77)
    t1, t2, kg1, kg2, tset, _ = _sampled_setup(cpu_engine, rng)
    n, n_rel, d = 50, 4, 12
    ent, rel = make_tables(rng, 2 * n, n_rel, d)
    for loss, k, B, shard in (("limited", 6, 33, None), ("limited", 16, 32, None), ("margin-based", 1, 31, None),
                              ("positive", 0, 20, None), ("limited", 5, 37, (1, 3)), ("logistic", 3, 34, (0, 2)),
                              ("limited", 20, 35, None)):
        dumps = []
        for loss_norm in ("L2", "L1"):
            cfg = cpu_engine.loss_cfg(loss, loss_norm, 0.8 if loss == "margin-based" else 0.1, 2.0, 0.2)
            make = lambda: cpu_engine.TripleTrainer(cpu_engine.EmbeddingTable(ent, True, "Adagrad", device="cpu"),
                                                    cpu_engine.EmbeddingTable(rel, True, "Adagrad", device="cpu"), cfg, 0.01)
            tr, ref = make(), make()
            dbg = torch.full((B, 2 + k), -7, dtype=torch.int32)
            tr.score_sampled(kg1, kg2, tset, B, k, 1, 991, dbg=dbg, shard=shard)
            dumps.append(dbg.numpy().copy())
            live = dumps[-1][:, 0] != -7
            assert live.sum() > 0
            pos, neg = decode_dbg(dumps[-1][live], t1, t2, k)
            ref.score_fed(_t(pos), None if neg is None else _t(neg))
            what = (loss, loss_norm, k, B, shard)
            assert tr.read_loss() == pytest.approx(ref.read_loss(), rel=1e-5), what
            np.testing.assert_allclose(tr.ent.grad.numpy(), ref.ent.grad.numpy(), rtol=1e-4, atol=1e-6, err_msg=str(what))
            np.testing.assert_allclose(tr.rel.grad.numpy(), ref.rel.grad.numpy(), rtol=1e-4, atol=1e-6, err_msg=str(what))
            assert np.array_equal(tr.ent.touched.numpy() != 0, ref.ent.touched.numpy() != 0), what
        assert np.array_equal(dumps[0], dumps[1]), (loss, k, B, shard)


def _sampled_setup(engine, rng, opt="Adagrad"):
    n, n_rel, d = 50, 4, 12
    def kg(lo):
        t = np.stack([rng.integers(lo, lo + n, 120), rng.integers(0, n_rel, 120), rng.integers(lo, lo + n, 120)], 1)
        return np.unique(t.astype(np.int32), axis=0)
    t1, t2 = kg(0), kg(n)
    ent, rel = make_tables(rng, 2 * n, n_rel, d)
    kg1 = engine.DeviceKG(t1, np.arange(0, n), 2 * n, device="cpu")
    kg2 = engine.DeviceKG(t2, np.arange(n, 2 * n), 2 * n, device="cpu")
    tset = engine.DeviceTripleSet([kg1.triples, kg2.triples], 2 * n, n_rel, device="cpu")
    make = lambda: engine.TripleTrainer(engine.EmbeddingTable(ent, True, opt, device="cpu"),
                                        engine.EmbeddingTable(rel, True, opt, device="cpu"),
                                        engine.loss_cfg("limited", "L2", 0.1, 2.0, 0.2), 0.01)
    return t1, t2, kg1, kg2, tset, make


def test_emulated_octet_scorer_replays_through_the_fed_scorer(cpu_engine, octet_k):
    """k_score_sampled_oct (four negatives per warp pass, shared rows staged in shared memory) and the duo: the debug
    dump replayed through the per-triple fed scorer gives the same loss and gradients."""
    rng = np.random.default_rng(18)
    t1, t2, kg1, kg2, tset, make = _sampled_setup(cpu_engine, rng)
    B, k = 32, octet_k
    a = make()
    dbg = torch.zeros(B, 2 + k, dtype=torch.int32)
    n_pos = torch.zeros(1, dtype=torch.int32)
    a.score_sampled(kg1, kg2, tset, B, k, 1, 4242, dbg=dbg, n_pos_out=n_pos)
    pos, neg = decode_dbg(dbg.numpy()[:int(n_pos)], t1, t2, k)
    b = make()
    b.score_fed(_t(pos), _t(neg))
    assert a.read_loss() == pytest.approx(b.read_loss(), rel=1e-5)
    np.testing.assert_allclose(a.ent.grad.numpy(), b.ent.grad.numpy(), rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(a.rel.grad.numpy(), b.rel.grad.numpy(), rtol=1e-4, atol=1e-6)
    assert np.array_equal(a.ent.touched.numpy() != 0, b.ent.touched.numpy() != 0)


@pytest.mark.parametrize("opt", ["Adagrad", "SGD"])
def test_emulated_one_launch_step_equals_score_then_optimiser(cpu_engine, octet_k, opt):
    """k_step_sampled_duo / k_step_sampled_oct (score + grid barrier + flagged-row optimiser in one cooperative launch;
    the duo is the bench's headline kernel) against the two-launch path (the same scorer, then k_rowopt_pair) with the
    same sampling seed."""
    rng = np.random.default_rng(19)
    t1, t2, kg1, kg2, tset, make = _sampled_setup(cpu_engine, rng, opt)
    fused, split = make(), make()
    for step in range(3):
        fused.step_sampled(kg1, kg2, tset, 32, octet_k, step, 777)
        split.score_sampled(kg1, kg2, tset, 32, octet_k, step, 777)
        split.apply()
    assert fused.read_loss() == pytest.approx(split.read_loss(), rel=1e-5)
    for x, y in ((fused.ent, split.ent), (fused.rel, split.rel)):
        np.testing.assert_allclose(x.raw().numpy(), y.raw().numpy(), rtol=1e-4, atol=1e-6)
        if opt == "Adagrad":
            np.testing.assert_allclose(x.state1.numpy(), y.state1.numpy(), rtol=1e-4, atol=1e-6)
        assert not x.grad.any() and not x.touched.any()
    assert not torch.equal(fused.ent.raw(), make().ent.raw())           # the steps did move the tables


@pytest.mark.parametrize("grouped", ["0", "1", "fused"])
def test_emulated_pipelined_host_step_equals_the_synchronous_one(cpu_engine, monkeypatch, grouped):
    """oea_triple_step_fed_host_submit / _collect (two slots with their own index buffers and loss scalars; the stream /
    event ordering is trivially satisfied on the emulator) against oea_triple_step_fed_host on the same batches: slot
    bookkeeping, buffer offsets, the per-step losses and the final tables — also with the grouped scorer selected."""
    monkeypatch.setenv("OEA_FED_GROUPED", "1" if grouped == "1" else "0")
    monkeypatch.setenv("OEA_FED_FUSED", "1" if grouped == "fused" else "0")
    rng = np.random.default_rng(23)
    d, n_ent, n_rel = 20, 60, 7
    ent, rel = make_tables(rng, n_ent, n_rel, d)
    cfg = cpu_engine.loss_cfg("limited", "L2", 0.01, 2.0, 0.2)
    batches = [tuple(_t(x) for x in make_batch(rng, n_ent, n_rel, 16, 3)) for _ in range(5)]
    make = lambda: cpu_engine.TripleTrainer(cpu_engine.EmbeddingTable(ent, True, device="cpu"),
                                            cpu_engine.EmbeddingTable(rel, True, device="cpu"), cfg, 0.01)
    a = make()
    a._loss_pinned = torch.zeros(1, dtype=torch.float64)
    want = [a.step_fed_host(p, n) for p, n in batches]
    b = make()
    idx = [torch.empty(3 * 16 * 4, dtype=torch.int32) for _ in range(2)]
    loss_dev = [torch.zeros(1, dtype=torch.float64) for _ in range(2)]
    loss_host = [torch.zeros(1, dtype=torch.float64) for _ in range(2)]
    vp2 = lambda x, y: (C.c_void_p * 2)(x, y)
    pipe = L.FedPipeline(0x10, 0x20, vp2(0x30, 0x31), vp2(0x40, 0x41), vp2(idx[0].data_ptr(), idx[1].data_ptr()),
                         vp2(loss_dev[0].data_ptr(), loss_dev[1].data_ptr()), vp2(loss_host[0].data_ptr(), loss_host[1].data_ptr()))
    lib = L.load()
    got = []

    def submit(slot, pos, neg):
        opt = cpu_engine.opt_cfg(b.ent, b.lr)
        L.check(lib.oea_triple_step_fed_host_submit(C.byref(b.ent.c_struct()), C.byref(b.rel.c_struct()), C.byref(pipe), slot,
                                                    C.c_void_p(pos.data_ptr()), pos.shape[1], C.c_void_p(neg.data_ptr()),
                                                    neg.shape[1], C.byref(b.loss), C.byref(opt)), "submit")

    def collect(slot):
        out = C.c_float(0.0)
        L.check(lib.oea_triple_step_fed_host_collect(C.byref(pipe), slot, C.byref(out)), "collect")
        return float(out.value)
    for i, (p, n) in enumerate(batches):
        submit(i % 2, p, n)
        if i:
            got.append(collect((i - 1) % 2))
    got.append(collect((len(batches) - 1) % 2))
    np.testing.assert_allclose(got, want, rtol=1e-5)
    for x, y in ((a.ent, b.ent), (a.rel, b.rel)):
        np.testing.assert_allclose(y.raw().numpy(), x.raw().numpy(), rtol=1e-5, atol=1e-7)
        assert not y.grad.any() and not y.touched.any()


@pytest.mark.parametrize("opt", ["Adagrad", "SGD"])
@pytest.mark.parametrize("loss,k,d", [("limited", 3, 20), ("margin-based", 1, 75), ("logistic", 2, 200), ("positive", 0, 20)])
def test_emulated_one_launch_fed_step_equals_dense_tf_steps(cpu_engine, opt, loss, k, d):
    """oea_triple_step_fed_grouped (grouped scoring + grid barrier + octet row optimiser in one cooperative launch, run as
    one block on the emulator) against the C oracle's dense TF steps, and against the two-launch path it replaces."""
    rng = np.random.default_rng(7 * d + k)
    n_ent, n_rel = 60, 7
    ent, rel = make_tables(rng, n_ent, n_rel, d)
    kw = dict(margin=1.1 if loss == "margin-based" else 0.3, neg_margin=2.2, balance=0.2)
    cfg = cpu_engine.loss_cfg(loss, "L2", **kw)
    st = orc.DenseState(ent, rel, opt)
    make = lambda: cpu_engine.TripleTrainer(cpu_engine.EmbeddingTable(ent, True, opt, device="cpu"),
                                            cpu_engine.EmbeddingTable(rel, True, opt, device="cpu"), cfg, 0.01)
    fused, split = make(), make()
    for _ in range(3):
        pos, neg = make_batch(rng, n_ent, n_rel, 16, k)
        want = orc.step(st, pos, neg, loss, "L2", True, True, 0.01, **kw)
        fused.step_fed_grouped(_t(pos), None if neg is None else _t(neg))
        split.score_fed(_t(pos), None if neg is None else _t(neg), grouped=True)
        split.apply()
        assert fused.read_loss() == pytest.approx(want, rel=1e-4)
        assert split.read_loss() == pytest.approx(want, rel=1e-4)
    for tab, ref, other in ((fused.ent, st.ent, split.ent), (fused.rel, st.rel, split.rel)):
        np.testing.assert_allclose(tab.raw().numpy(), ref, rtol=1e-4, atol=1e-6)
        np.testing.assert_allclose(tab.raw().numpy(), other.raw().numpy(), rtol=1e-5, atol=1e-7)
        assert not tab.grad.any() and not tab.touched.any()


def test_one_launch_fed_step_refuses_what_it_does_not_cover(cpu_engine):
    rng = np.random.default_rng(3)
    ent, rel = make_tables(rng, 30, 3, 12)
    pos, neg = make_batch(rng, 30, 3, 8, 2)
    t = cpu_engine.TripleTrainer(cpu_engine.EmbeddingTable(ent, True, "Adam", device="cpu"),
                                 cpu_engine.EmbeddingTable(rel, True, "Adam", device="cpu"),
                                 cpu_engine.loss_cfg("limited", "L2", 0.1, 2.0, 0.2), 0.01)
    with pytest.raises(L.OeaError):
        t.step_fed_grouped(_t(pos), _t(neg))                       # Adam: dense update, not the flagged-row optimiser
    t = cpu_engine.TripleTrainer(cpu_engine.EmbeddingTable(ent, True, device="cpu"), cpu_engine.EmbeddingTable(rel, True, device="cpu"),
                                 cpu_engine.loss_cfg("limited", "L1", 0.1, 2.0, 0.2), 0.01)
    with pytest.raises(L.OeaError):
        t.step_fed_grouped(_t(pos), _t(neg))                       # L1 score
    assert not t.ent.grad.any()                                    # nothing was launched


def test_emulated_host_steps_with_the_one_launch_kernel(cpu_engine, monkeypatch):
    """OEA_FED_FUSED=1 on the synchronous host-index step and on the pipelined one: same losses and tables as the default;
    with Adam (not covered by the kernel) the flag falls back to the two-launch path."""
    rng = np.random.default_rng(29)
    d, n_ent, n_rel = 20, 60, 7
    ent, rel = make_tables(rng, n_ent, n_rel, d)
    cfg = cpu_engine.loss_cfg("limited", "L2", 0.01, 2.0, 0.2)
    batches = [tuple(_t(x) for x in make_batch(rng, n_ent, n_rel, 16, 3)) for _ in range(4)]
    for opt in ("Adagrad", "Adam"):
        res = []
        for flag in ("0", "1"):
            monkeypatch.setenv("OEA_FED_FUSED", flag)
            t = cpu_engine.TripleTrainer(cpu_engine.EmbeddingTable(ent, True, opt, device="cpu"),
                                         cpu_engine.EmbeddingTable(rel, True, opt, device="cpu"), cfg, 0.01)
            t._loss_pinned = torch.zeros(1, dtype=torch.float64)
            res.append(([t.step_fed_host(p, n) for p, n in batches], t.ent.raw().numpy().copy(), t.rel.raw().numpy().copy()))
        np.testing.assert_allclose(res[1][0], res[0][0], rtol=1e-5)
        np.testing.assert_allclose(res[1][1], res[0][1], rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(res[1][2], res[0][2], rtol=1e-5, atol=1e-7)
