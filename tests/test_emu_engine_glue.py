"""CPU: the Python host layer of the score-function family (openea_b200.engine.ModelTrainer, DeviceKG,
DeviceTripleSet — ctypes structs, pointer lifetimes, buffer slicing, step sequencing) driven end to end over CPU
tensors, with two entry points served by the warp emulator (tests/emu) and two (row optimiser, triple-set build) by
NumPy statements of their documented contract.
Only this test wires the engine this way; the product path loads liboea.so and nothing else."""
import ctypes as C

import numpy as np
import pytest
import torch

from openea_b200 import engine as eng
from openea_b200 import lib as L
from oracle import triple_ext as ox
from tests.emu import build_emu
from tests.test_emu_sampler import build_tripleset


def _np(ptr, shape, dtype):
    n = int(np.prod(shape))
    buf = (C.c_byte * (n * np.dtype(dtype).itemsize)).from_address(ptr)
    return np.frombuffer(buf, dtype=dtype).reshape(shape)


class HybridLib:
    """oea_model_score_fed / oea_triple_sample_batch → the emulator; oea_rowopt_apply / oea_tripleset_build → NumPy."""

    def __init__(self, emu):
        for name in ("oea_model_score_fed", "oea_triple_sample_batch"):
            setattr(self, name, getattr(emu, name))

    @staticmethod
    def oea_error_string(rc):
        return ("emulated rc %d" % rc).encode()

    @staticmethod
    def oea_rowopt_apply(table_ref, cfg_ref, stream):
        """include/oea.h: Adagrad / SGD on flagged rows, leaves grad = 0 and touched = 0."""
        t, cfg = table_ref._obj, cfg_ref._obj
        w = _np(t.weight, (t.rows, t.pitch), np.float32)
        g = _np(t.grad, (t.rows, t.pitch), np.float32)
        touched = _np(t.touched, (t.rows,), np.int32)
        rows = touched != 0
        if cfg.kind == L.OPT_ADAGRAD:
            acc = _np(t.state1, (t.rows, t.pitch), np.float32)
            acc[rows] += g[rows] ** 2
            w[rows] -= cfg.lr * g[rows] / np.sqrt(acc[rows])
        else:
            assert cfg.kind == L.OPT_SGD
            w[rows] -= cfg.lr * g[rows]
        g[:] = 0
        touched[:] = 0
        return 0

    @staticmethod
    def oea_tripleset_build(triples, n, slots, capacity, ent_bits, rel_bits, stream):
        tri = _np(triples.value, (n, 3), np.int32)
        built, _ = build_tripleset(tri, ent_bits, rel_bits, capacity=capacity)
        _np(slots.value, (capacity,), np.uint64)[:] = built
        return 0


@pytest.fixture()
def cpu_engine(monkeypatch):
    build_emu.patch_engine(monkeypatch, HybridLib(build_emu.load()))
    return eng


@pytest.mark.parametrize("model,loss,k,sampler", [("TransD", "limited", 3, "fast"), ("TransH", "margin-based", 1, "fast"),
                                                  ("DistMult", "logistic", 2, "independent"),
                                                  ("SimplE", "logistic", 1, "fast")])
def test_model_trainer_steps_on_the_emulator_equal_oracle_steps(cpu_engine, model, loss, k, sampler):
    eng_ = cpu_engine
    rng = np.random.default_rng(9)
    n, n_rel, d = 40, 4, 20

    def kg(lo):
        t = np.stack([rng.integers(lo, lo + n, 150), rng.integers(0, n_rel, 150), rng.integers(lo, lo + n, 150)], 1)
        return np.unique(t.astype(np.int32), axis=0)
    t1, t2 = kg(0), kg(n)
    slots = ox.SLOTS[model] + (None,) * (4 - len(ox.SLOTS[model]))
    tabs = {s: (rng.standard_normal((n_rel if i in (1, 3) else 2 * n, d)) / np.sqrt(d)).astype(np.float32)
            for i, s in enumerate(slots) if s}
    norms = {s: True for s in tabs}
    tables = tuple(None if s is None else eng_.EmbeddingTable(tabs[s], True, "Adagrad", device="cpu") for s in slots)
    kg1 = eng_.DeviceKG(t1, np.arange(0, n), 2 * n, device="cpu")
    kg2 = eng_.DeviceKG(t2, np.arange(n, 2 * n), 2 * n, device="cpu")
    tset = eng_.DeviceTripleSet([kg1.triples, kg2.triples], 2 * n, n_rel, device="cpu")
    kw = dict(margin=1.0 if loss == "margin-based" else 0.05, neg_margin=1.5, balance=0.3)
    mean = model == "DistMult"
    tr = eng_.ModelTrainer(model, tables, eng_.loss_cfg(loss, "L2", **kw), 0.05, mean_loss=mean, sampler=sampler)
    st = ox.DenseState(tabs, "Adagrad")
    B = 64
    steps = int(np.ceil((len(t1) + len(t2)) / B))
    total = 0
    for step in range(steps):
        pos, neg = tr.sample_batch(kg1, kg2, tset, B, k, step, epoch_seed=99)
        p, q = pos.numpy().copy(), neg.numpy().copy()
        scale = 1.0 / (p.shape[1] + q.shape[1]) if mean else 1.0
        want = ox.step(st, model, norms, p, q, loss, 0.05, scale=scale, **kw)
        n_pos = tr.step_sampled(kg1, kg2, tset, B, k, step, epoch_seed=99)     # same seed → the same batch again
        assert n_pos == p.shape[1]
        assert tr.read_loss() == pytest.approx(want, rel=1e-4)
        total += n_pos
    assert total == len(t1) + len(t2)
    for s, tab in zip(slots, tables):
        if s is not None:
            np.testing.assert_allclose(tab.raw().numpy(), st.w[s], rtol=1e-4, atol=2e-5, err_msg=s)
            assert not tab.grad.any() and not tab.touched.any()


@pytest.mark.parametrize("name", ["TransH", "TransD", "SimplE", "DistMult"])
def test_model_lifecycle_init_and_run_on_the_emulator(cpu_engine, monkeypatch, tmp_path, capsys, name):
    """set_args / set_kgs / init / run of the four model classes on a 40-entity synthetic dataset: the reference's epoch
    lines appear, the loss is finite and every table of the model has moved.  (test() / save() need the similarity
    kernels, which only run on a GPU: tests/test_zz_triple_ext_gpu.py.)"""
    import re
    from openea_b200 import presets
    from openea_b200.models import trans, semantic
    from openea_b200.modules.base import initializers
    from openea_b200.modules.load.kgs import read_kgs_from_folder
    from openea_b200.synth import write_dataset
    monkeypatch.setattr(initializers, "_make", lambda values, norm, optimizer=None: cpu_engine.EmbeddingTable(
        values, bool(norm), optimizer or "Adagrad", "cpu"))
    monkeypatch.setattr(L.load(), "oea_mapping_workspace_bytes", lambda dim: 0, raising=False)   # DistMult builds a mapper
    from openea_b200.models.trans import transe
    from openea_b200.models.semantic import distmult, simple
    for mod in (transe, distmult, simple):       # load_session() refuses to run without a CUDA device (by design)
        monkeypatch.setattr(mod, "load_session", lambda: None)
    folder = write_dataset(str(tmp_path) + "/micro/", "micro")
    cls = {"TransH": trans.TransH, "TransD": trans.TransD, "SimplE": semantic.SimplE, "DistMult": semantic.DistMult}[name]
    args = getattr(presets, name.lower())("15K")
    args.training_data, args.output = folder, str(tmp_path) + "/out/"
    args.batch_size, args.max_epoch, args.start_valid, args.dim = 64, 2, 1000, 16
    kgs = read_kgs_from_folder(folder, args.dataset_division, "sharing", args.ordered)
    model = cls()
    model.set_args(args)
    model.set_kgs(kgs)
    model.init()
    before = [t.weight.clone() for t in model.triple_trainer.live]
    model.run()
    out = capsys.readouterr().out
    tag = r"triple loss: ([0-9.]+)" if name == "DistMult" else r"avg\. triple loss: ([0-9.]+)"
    losses = [float(x) for x in re.findall(tag, out)]
    assert len(losses) == 2 and all(np.isfinite(losses)) and losses[0] > 0
    assert "Training ends. Total time" in out
    for b, t in zip(before, model.triple_trainer.live):
        assert not torch.equal(b, t.weight) and torch.isfinite(t.weight).all()
