"""GPU tests of ConvE (oea_conve_score_fed) through the engine: a batch at the 15K shape (B = 500, S = 4 096,
E = 30 000, F = 32, d = 100, keep_prob 0.7) and one at the 100K shape (B = 5 000, E = 200 000) against float64 computed on
the device with the dropout masks restated on the host; 20 Adam steps on the eight tables against dense float64 steps;
one seed drawing the same sampled sets and masks; run/main_from_args.py with presets.conve("15K") on the synthetic 15K
dataset; and checkpoint → resume.  Tolerances as tests/test_emu_conve.py derives them."""
import contextlib
import io
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import conve_oracle as co
from tests.test_emu_conve import KINK, NORMS, _batch, _case, _tol
from tests.test_zz_triple_ext_gpu import tiny_kgs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _trainer(tabs, S, keep, lr=0.01):
    from openea_b200 import engine as eng
    tables = {k: eng.EmbeddingTable(v, NORMS.get(k, False), "Adam") for k, v in tabs.items()}
    return eng.ConvETrainer(tuple(tables[k] for k in co.NAMES), S, lr, keep), tables


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).cuda()


def _grads(tables):
    return {k: t.grad[:, :t.dim].double().cpu().numpy() for k, t in tables.items()}


def _batch_against_float64(n_ent, n_rel, d, F, n, S, keep, seed):
    rng, tabs = _case(seed, n_ent, n_rel, d, F)
    pos = _batch(rng, n_ent, n_rel, n)
    tr, tables = _trainer(tabs, S, keep)
    tr.sample(seed + 5)
    sampled, tries = tr.sampled.cpu().numpy(), int(tr.num_tries.item())
    m0, m1 = co.masks(seed + 9, n, d, F, keep)
    tr.score_fed(_dev(pos), dropout_seed=seed + 9)
    got_loss = tr.read_loss()
    # at these shapes about 0.1 % of the millions of ReLU inputs lie within their worst-case fp32 rounding bound of 0
    # (γ(2Fd + 13)·Σ|a·w| for a dense one) and may take the other branch on the device: they are counted and reported
    # with any mismatch, and must stay below 0.2 % of the elements; the tolerance below absorbs their flips
    near, total = co.near_kinks(tabs, NORMS, pos, keep, m0, m1, device="cuda")
    assert near <= 2e-3 * total, (near, total)
    margin = "%d of %d ReLU inputs within rounding of a kink" % (near, total)
    want_loss, want_g = co.fwd_bwd(tabs, NORMS, pos, sampled, tries, keep, m0, m1, device="cuda")
    tol = _tol(d, F, S)
    assert got_loss == pytest.approx(want_loss, rel=tol), margin
    for k, got in _grads(tables).items():
        want = want_g[k].reshape(got.shape)
        np.testing.assert_allclose(got, want, rtol=tol, atol=tol * np.abs(want).max(),
                                   err_msg="%s (%s)" % (k, margin))


def test_15k_shape_batch_matches_float64_on_the_device(cuda_device):
    _batch_against_float64(30000, 600, 100, 32, 500, 4096, 0.7, 15)


def test_100k_shape_batch_matches_float64_on_the_device(cuda_device):
    _batch_against_float64(200000, 1000, 100, 32, 5000, 4096, 0.7, 100)


def test_adam_steps_equal_dense_float64_steps(cuda_device):
    n_ent, n_rel, d, F, lr, keep = 50, 5, 12, 2, 0.01, 0.7
    rng, tabs = _case(12, n_ent, n_rel, d, F)         # every pre-activation of the 20 steps is at least 1e-4 from a kink
    tr, tables = _trainer(tabs, 16, keep, lr)
    st = co.DenseState(dict(tabs), "Adam")
    for step in range(20):
        pos = _batch(rng, n_ent, n_rel, 23)
        tr.sample(50 + step)
        sampled, tries = tr.sampled.cpu().numpy(), int(tr.num_tries.item())
        m0, m1 = co.masks(900 + step, 23, d, F, keep)
        assert co.kink_margin({k: v.astype(np.float32) for k, v in st.w.items()}, NORMS, pos, keep, m0, m1) > KINK
        want = co.step(st, NORMS, pos, sampled, tries, keep, m0, m1, lr)
        tr.score_fed(_dev(pos), dropout_seed=900 + step)
        tr.apply()
        assert tr.read_loss() == pytest.approx(want, rel=1e-4), step
    for k, tab in tables.items():
        want = st.w[k].reshape(tab.rows, -1)
        np.testing.assert_allclose(tab.raw().double().cpu().numpy(), want, rtol=1e-3, atol=1e-5, err_msg=k)


def test_one_seed_draws_the_same_steps_and_tables_agree_to_the_atomic_order_bound(cuda_device):
    from openea_b200 import engine as eng
    d, F, n_ent, n_rel = 100, 32, 3000, 50
    rng, tabs = _case(8, n_ent, n_rel, d, F)
    pos = [_batch(rng, n_ent, n_rel, 500) for _ in range(3)]
    runs = []
    for _ in range(2):
        tr, tables = _trainer(tabs, 1024, 0.7, 0.001)
        drawn = []
        for step, p in enumerate(pos):
            seed = eng.ProjETrainer.step_seed(1234, step)
            tr.sample(seed)
            drawn.append(tr.sampled.cpu().numpy().copy())
            tr.score_fed(_dev(p), dropout_seed=tr.step_seed(seed, 0))
            tr.apply()
        runs.append((drawn, {k: t.raw().double().cpu().numpy() for k, t in tables.items()}, tr.read_loss()))
    assert all(np.array_equal(a, b) for a, b in zip(runs[0][0], runs[1][0]))
    # Adam turns a gradient at the level of atomic-order noise into a step of up to lr either way: such elements may
    # differ by 2·lr per step; every other element agrees to fp32 accumulation noise
    for k, w in runs[0][1].items():
        diff = np.abs(runs[1][1][k] - w)
        loose = diff > 1e-4 * np.abs(w) + 1e-5 * np.abs(w).max()
        assert diff.max() <= 2 * 0.001 * len(pos), k
        assert loose.mean() <= 1e-4, (k, int(loose.sum()))
    assert runs[0][2] == pytest.approx(runs[1][2], rel=1e-5)


def test_conve_through_main_from_args(cuda_device, tmp_path):
    """run/main_from_args.py with a JSON written from presets.conve("15K") on the synthetic 15K dataset: it runs to the
    end, the loss falls, and the results are written."""
    from openea_b200 import presets
    from openea_b200.synth import write_dataset
    write_dataset(str(tmp_path / "data" / "SYN_15K") + "/", "15K")
    args = presets.conve("15K")
    args.training_data, args.output = str(tmp_path / "data") + "/", str(tmp_path / "out") + "/"
    args.max_epoch, args.start_valid = 10, 1000
    path = tmp_path / "conve_args.json"
    path.write_text(json.dumps(vars(args)))
    res = subprocess.run([sys.executable, os.path.join(ROOT, "run", "main_from_args.py"), str(path), "SYN_15K",
                          args.dataset_division], capture_output=True, text=True, timeout=1200,
                         cwd=os.path.join(ROOT, "run"))
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-3000:]
    losses = [float(x) for x in re.findall(r"avg\. triple loss: ([0-9.]+)", res.stdout)]
    assert len(losses) == 10 and np.isfinite(losses).all()
    assert np.mean(losses[-3:]) < 0.95 * np.mean(losses[:3]), losses
    folder = re.search(r"results output folder: (\S+)", res.stdout).group(1)
    assert os.path.exists(folder + "ent_embeds.npy") and os.path.exists(folder + "alignment_results_12")


def test_conve_resume_from_checkpoint_continues_the_same_run(cuda_device, tiny_kgs, tmp_path):
    """6 epochs in one go == 3 epochs, checkpoint, a NEW model restored from the file, 3 more epochs: all eight tables
    and their Adam slots, to fp32 accumulation noise (gradient sums are atomics)."""
    from openea_b200 import presets
    from openea_b200.models.neural import ConvE
    from openea_b200.modules.base import initializers
    from openea_b200.modules.load.kgs import read_kgs_from_folder
    names = ("ent_embeds", "rel_embeds", "entity_w", "entity_b", "conv", "bn_in", "fc_w", "fc_out")

    def make(max_epoch, out, **extra):
        args = presets.conve()
        args.training_data, args.output = tiny_kgs, str(tmp_path) + "/" + out + "/"
        args.batch_size, args.max_epoch, args.start_valid, args.dim, args.dnn_neg_nums = 500, max_epoch, 1000, 32, 128
        args.filter_num = 4
        for k, v in extra.items():
            setattr(args, k, v)
        initializers.set_seed(77)
        m = ConvE()
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
        assert set(names) <= set(resumed._checkpoint_tables())
        assert resumed.load_checkpoint(first.out_folder + "checkpoint.pt") == 4
        resumed.run()
    for name in names:
        a, b = getattr(straight, name), getattr(resumed, name)
        for what, x, y in (("weight", a.raw(), b.raw()), ("m", a.state1, b.state1)):
            want = x.cpu().numpy()
            np.testing.assert_allclose(y.cpu().numpy(), want, rtol=2e-3, atol=2e-4 * max(1.0, np.abs(want).max()),
                                       err_msg=name + " " + what)
        assert a.adam_t == b.adam_t
    assert resumed._epoch_seed == straight._epoch_seed
