"""GPU: the general sampled-NCE step (oea_nce_score_fed) against float64 on the device at the synthetic 15K shape and
at a large vocabulary, Adagrad steps against dense float64 TF Adagrad fed the same pairs and sampled sets, the
repeatability of a seeded run, and Attr2Vec through run/main_from_args.py with presets.attr2vec("15K")."""
import json
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import attr2vec_oracle as ao

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("in", "w", "b")
BOTH = {"in": True, "w": True}


def _case(seed, A, d):
    rng = np.random.default_rng(seed)
    sd = math.sqrt(1.3 * 2 / (A + d))
    tabs = {"in": rng.standard_normal((A, d)) * sd, "w": rng.standard_normal((A, d)) * sd,
            "b": rng.standard_normal((A, 1)) * 0.1}
    return rng, {k: v.astype(np.float32) for k, v in tabs.items()}


def _trainer(tabs, S, lr=0.01, norms=BOTH):
    from openea_b200 import engine as eng
    tables = {k: eng.EmbeddingTable(v, norms.get(k, False), "Adagrad") for k, v in tabs.items()}
    return eng.NceTrainer(tuple(tables[k] for k in NAMES), S, lr), tables


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).cuda()


def _assert_close(got, want, what, rtol=2e-4):
    want = want.reshape(got.shape)
    np.testing.assert_allclose(got, want, rtol=rtol, atol=2e-4 * max(1e-6, np.abs(want).max()), err_msg=what)


def _batch_against_float64(A, d, n, S, seed, norms=BOTH):
    rng, tabs = _case(seed, A, d)
    inputs, labels = rng.integers(0, A, n), rng.integers(0, A, n)
    labels[:50] = inputs[:50]                              # an input that is its own label
    tr, tables = _trainer(tabs, S, norms=norms)
    tr.sample(seed + 5)
    sampled, tries = tr.sampled.cpu().numpy(), int(tr.num_tries.item())
    labels[50:100] = sampled[:50]                          # accidental hits
    tr.score_fed(_dev(inputs), _dev(labels))
    got_loss = tr.read_loss()
    want_loss, want_g = ao.fwd_bwd(tabs, norms, inputs, labels, sampled, tries, 1.0 / n, device="cuda")
    assert got_loss == pytest.approx(want_loss, rel=2e-5)
    for k in NAMES:
        _assert_close(tables[k].grad[:, :tables[k].dim].double().cpu().numpy(), want_g[k], k)


def test_15k_shape_batch_matches_float64_on_the_device(cuda_device):
    """Synthetic 15K: 800 attributes, 160 sampled, a batch of 5 000, d = 100."""
    _batch_against_float64(800, 100, 5000, 160, 15)


def test_large_vocabulary_batch_matches_float64_on_the_device(cuda_device):
    """20 000 classes, 4 000 sampled (32 column tiles), a batch of 5 000 (40 row tiles)."""
    _batch_against_float64(20000, 100, 5000, 4000, 20)


def test_raw_class_table_batch_matches_float64_on_the_device(cuda_device):
    _batch_against_float64(800, 75, 2000, 160, 7, norms={"in": True, "w": False})


def test_adagrad_steps_equal_dense_float64_steps(cuda_device):
    """20 steps, each on the pairs and sampled set the device drew, applied to the float64 state as well."""
    A, d, lr, B = 800, 100, 0.01, 1000
    rng, tabs = _case(3, A, d)
    pairs = rng.integers(0, A, (6000, 2)).astype(np.int32)
    tr, tables = _trainer(tabs, 160, lr)
    tr.set_pairs(pairs)
    st = ao.DenseState(dict(tabs), "Adagrad")
    for step in range(20):
        inputs, labels = tr.draw(B, 77, 1, step)
        tr.sample(1000 + step)
        sampled, tries = tr.sampled.cpu().numpy(), int(tr.num_tries.item())
        want = ao.step(st, BOTH, inputs.cpu().numpy(), labels.cpu().numpy(), sampled, tries, lr)
        tr.score_fed(inputs, labels)
        tr.apply()
        assert tr.read_loss() == pytest.approx(want, rel=1e-4)
    for k, tab in tables.items():
        np.testing.assert_allclose(tab.raw().cpu().numpy(), st.w[k].reshape(tab.rows, -1), rtol=1e-3, atol=2e-5,
                                   err_msg=k)


def test_one_seed_draws_the_same_steps_and_tables_agree_to_the_atomic_order_bound(cuda_device):
    """The pair draws and sampled sets of a seed are bit-identical; the tables are not, because the head's dX, dW and
    bias gradients are summed with atomics in an order that varies from run to run.  After 10 steps at the 15K shape
    they agree to 1e-6 absolute (parameters of norm ~0.1-1)."""
    A, d, B = 800, 100, 5000
    rng, tabs = _case(9, A, d)
    pairs = rng.integers(0, A, (40000, 2)).astype(np.int32)
    runs = []
    for _ in range(2):
        tr, tables = _trainer(tabs, 160)
        tr.set_pairs(pairs)
        draws = []
        for step in range(10):
            tr.step(B, 1234, 1, step)
            draws.append((tr._batch[:, :B].cpu().numpy().copy(), tr.sampled.cpu().numpy().copy()))
        runs.append((draws, {k: t.raw().cpu().numpy() for k, t in tables.items()}, tr.read_loss()))
    for (a_pairs, a_smp), (b_pairs, b_smp) in zip(runs[0][0], runs[1][0]):
        assert np.array_equal(a_pairs, b_pairs) and np.array_equal(a_smp, b_smp)
    for k in NAMES:
        assert np.abs(runs[0][1][k] - runs[1][1][k]).max() <= 1e-6, k
    assert runs[0][2] == pytest.approx(runs[1][2], rel=1e-6)


def test_attr2vec_through_main_from_args(cuda_device, tmp_path):
    """run/main_from_args.py with a JSON written from presets.attr2vec("15K") on the synthetic 15K dataset: it runs to
    the end, prints the reference's epoch lines, writes the results and attr_embeds.npy, and the loss falls."""
    from openea_b200 import presets
    from openea_b200.synth import write_dataset
    write_dataset(str(tmp_path / "data" / "SYN_15K") + "/", "15K")
    args = presets.attr2vec("15K")
    args.training_data, args.output = str(tmp_path / "data") + "/", str(tmp_path / "out") + "/"
    args.attr_max_epoch = 20
    path = tmp_path / "attr2vec_args.json"
    path.write_text(json.dumps(vars(args)))
    res = subprocess.run([sys.executable, os.path.join(ROOT, "run", "main_from_args.py"), str(path), "SYN_15K",
                          args.dataset_division], capture_output=True, text=True, timeout=1200,
                         cwd=os.path.join(ROOT, "run"))
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-3000:]
    losses = [float(x) for x in re.findall(r"epoch \d+, attribute loss: ([0-9.]+), cost time", res.stdout)]
    assert len(losses) == 20 and np.isfinite(losses).all()
    assert np.mean(losses[-3:]) < 0.95 * np.mean(losses[:3]), losses
    folder = re.search(r"results output folder: (\S+)", res.stdout).group(1)
    assert os.path.exists(folder + "attr_embeds.npy") and os.path.exists(folder + "alignment_results_12")
    assert "Total run time" in res.stdout
