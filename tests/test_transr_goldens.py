"""TransR against the reference's OWN graph code.  tests/golden/path_i_transr.npz was produced by executing the
reference's `TransR._define_variables` / `_define_embed_graph` and `session.run([triple_loss, triple_optimizer],
feed_dict)` on a TensorFlow-1 graph interpreter (oracle/tf1_shim.py, float64; scripts/make_golden_transr.py): the shipped
configuration (margin-based, L2, Adagrad, one negative), the limited loss with Adam and three negatives, the logistic
loss with the L1 score and SGD, un-normalised entities, and d = 10 (padding columns in every matrix row).  This
package's TransR, started from the same variables (the [R, d²] matrix as R·d rows of width d) and fed the same batches,
must reproduce every fetched loss within 2·10⁻⁴ and the variables after the last run, their movement included:

  * CPU: the kernels' sources on the warp emulator;
  * GPU (`-m gpu`): liboea.so.

tests/transr_oracle.py is pinned to the same file at float64 precision.
"""
import json
import os
import types

import numpy as np
import pytest
import torch

from openea_b200 import engine as eng
from tests import transr_oracle as tro
from tests.emu import build_emu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "path_i_transr.npz")
G = np.load(GOLDEN)
META = json.loads(bytes(G["meta"]).decode())
SLOT = {"ent_embeds": "ent", "rel_embeds": "rel", "rel_matrix": "mat"}


def _feed(case, i):
    prefix = "%s/run%d/feed/" % (case, i)
    return {k[len(prefix):]: G[k] for k in G.files if k.startswith(prefix)}


def _batch(case, i):
    f = _feed(case, i)
    pos = np.stack([f["pos_hs"], f["pos_rs"], f["pos_ts"]]).astype(np.int32)
    neg = np.stack([f["neg_hs"], f["neg_rs"], f["neg_ts"]]).astype(np.int32)
    return pos, neg


def replay(case, engine, device, monkeypatch):
    from openea_b200.models.trans import TransR
    from openea_b200.modules.base import initializers
    meta = META[case]
    monkeypatch.setattr(initializers, "_make", lambda values, norm, optimizer=None: engine.EmbeddingTable(
        values, bool(norm), optimizer or initializers._DEFAULT_OPT, device))
    model = TransR()
    model.args = types.SimpleNamespace(**meta["args"])
    model.kgs = types.SimpleNamespace(entities_num=40, relations_num=6)
    model._define_variables()
    model._define_embed_graph()
    d = meta["args"]["dim"]
    tables = {}
    for name in meta["variables"]:
        tab = getattr(model, name)
        start = G["%s/var0/%s" % (case, name)].reshape(-1, d)            # rel_matrix [R, d²] → R·d rows of width d
        assert tab.weight[:, :tab.dim].shape == start.shape, name
        tab.weight[:, :tab.dim] = torch.as_tensor(start, dtype=torch.float32, device=tab.weight.device)
        tables[name] = tab
    assert model.rel_matrix.l2_norm is False and model.rel_matrix.rows == 6 * d
    tr = model.triple_trainer
    for i, _ in enumerate(meta["runs"]):
        pos, neg = _batch(case, i)
        tr.score_fed(torch.from_numpy(pos).to(device), torch.from_numpy(neg).to(device))
        tr.apply()
        got = tr.read_loss()
        assert got == pytest.approx(float(G["%s/run%d/loss" % (case, i)]), rel=2e-4), (case, i)
    for name, tab in tables.items():
        want = G["%s/var_final/%s" % (case, name)].reshape(-1, d)
        start = G["%s/var0/%s" % (case, name)].reshape(-1, d)
        got = tab.raw().cpu().numpy()
        assert np.abs(want - start).max() > 0, name
        np.testing.assert_allclose(got - start, want - start, rtol=5e-3, atol=3e-6 + 2e-3 * np.abs(want - start).max(),
                                   err_msg="%s: %s" % (case, name))
        np.testing.assert_allclose(got, want, rtol=2e-4, atol=5e-6, err_msg="%s: %s" % (case, name))


@pytest.fixture()
def cpu_engine(monkeypatch):
    build_emu.patch_engine(monkeypatch, build_emu.load())
    return eng


def test_golden_file_covers_the_expected_cases():
    assert sorted(META) == ["transr", "transr_d10", "transr_limited_adam", "transr_logistic_l1_sgd",
                            "transr_raw_entities"]
    shipped = META["transr"]["args"]
    assert (shipped["loss"], shipped["loss_norm"], shipped["optimizer"], shipped["neg_triple_num"]) == \
        ("margin-based", "L2", "Adagrad", 1)
    assert META["transr_raw_entities"]["args"]["ent_l2_norm"] is False
    assert META["transr_d10"]["args"]["dim"] % 4 != 0
    for case, meta in META.items():
        assert meta["variables"] == ["ent_embeds", "rel_embeds", "rel_matrix"]
        d = meta["args"]["dim"]
        assert G["%s/var0/rel_matrix" % case].shape == (6, d * d)


@pytest.mark.parametrize("case", sorted(META))
def test_oracle_reproduces_the_reference_graph(case):
    """tests/transr_oracle.py, float64, on the golden's batches: every loss and the final variables to 1e-8."""
    meta = META[case]
    a = meta["args"]
    norms = {"ent": bool(a["ent_l2_norm"]), "rel": bool(a["rel_l2_norm"])}
    state = tro.DenseState({SLOT[v]: G["%s/var0/%s" % (case, v)] for v in meta["variables"]}, a["optimizer"])
    kw = {"margin-based": dict(margin=a["margin"]), "limited": dict(margin=a["pos_margin"], neg_margin=a["neg_margin"]),
          "logistic": {}}[a["loss"]]
    for i, _ in enumerate(meta["runs"]):
        pos, neg = _batch(case, i)
        val = tro.step(state, norms, pos, neg, a["loss"], a["learning_rate"], loss_norm=a["loss_norm"], **kw)
        assert val == pytest.approx(float(G["%s/run%d/loss" % (case, i)]), rel=1e-8), (case, i)
    for v in meta["variables"]:
        np.testing.assert_allclose(state.w[SLOT[v]], G["%s/var_final/%s" % (case, v)], rtol=1e-8, atol=1e-12)


@pytest.mark.parametrize("case", sorted(META))
def test_engine_on_the_emulator_reproduces_the_reference_graph(cpu_engine, monkeypatch, case):
    replay(case, cpu_engine, "cpu", monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(META))
def test_engine_on_the_gpu_reproduces_the_reference_graph(cuda_device, monkeypatch, case):
    from openea_b200 import engine
    replay(case, engine, "cuda", monkeypatch)
