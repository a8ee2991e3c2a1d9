"""Attr2Vec against the reference's OWN graph code.  tests/golden/path_i_attr2vec.npz was produced by executing the
reference's `Attr2Vec._define_variables` / `_define_embed_graph` and two `session.run([loss, optimizer], feed_dict)` per
case on a TensorFlow-1 graph interpreter (oracle/tf1_shim.py with scripts/tf1_shim_proje.py; float64;
scripts/make_golden_attr2vec.py), feeding the [B, 1] label reshape as the reference does: the shipped configuration
(d = 100) at A = 40, S = 8; every class sampled (S = A = 20); repeated inputs and labels with labels inside the sampled
set; and d = 10.  Each run records the sampled ids and num_tries it drew.  So the golden pins what a restatement could
get wrong: nce_loss over l2_normalize(var) for both tables, reduce_mean, and Adagrad through the normalisation.

  * tests/attr2vec_oracle.py reproduces every loss and the final variables to 1e-8;
  * the engine, started from the same variables and fed the same pairs and sampled sets, reproduces every loss within
    2·10⁻⁴ and the variables after the last run: the kernels' sources on the warp emulator (CPU) and liboea.so (`-m gpu`).
"""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from openea_b200 import lib as L
from tests import attr2vec_oracle as ao
from tests.test_emu_attr2vec import _run, emu  # noqa: F401  (emu: fixture)
from tests.test_emu_proje import HostTable

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "path_i_attr2vec.npz")
G = np.load(GOLDEN)
META = json.loads(bytes(G["meta"]).decode())
CASES = sorted(META)
NORMS = {"in": True, "w": True}
NAMES = ("in", "w", "b")


def _tables(case, stage):
    v = lambda n: G["%s/%s/%s" % (case, stage, n)]
    return {"in": v("attributeembeddings/attr_embed"), "w": v("nceembeddings/nce_weights"),
            "b": v("Variable").reshape(-1, 1)}


def _run_of(case, i):
    f = lambda k: G["%s/run%d/%s" % (case, i, k)]
    return (f("feed/inputs").astype(np.int32), f("feed/labels").astype(np.int32), f("sampled").astype(np.int32),
            int(f("num_tries")), float(f("loss")))


def _lr(case):
    return META[case]["learning_rate"]


def test_golden_covers_the_cases():
    assert CASES == ["attr2vec", "attr2vec_all_classes", "attr2vec_d10", "attr2vec_repeats"]
    assert META["attr2vec"]["dim"] == 100 and META["attr2vec_d10"]["dim"] == 10
    assert len(_run_of("attr2vec_all_classes", 0)[2]) == META["attr2vec_all_classes"]["attributes"]
    inputs, labels, sampled, _, _ = _run_of("attr2vec_repeats", 0)
    assert np.isin(labels, sampled).any() and len(set(labels)) < len(labels) and len(set(inputs)) < len(inputs)
    assert (inputs == labels).any()


@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_the_reference_graph(case):
    st = ao.DenseState(_tables(case, "var0"), "Adagrad")
    for i in range(2):
        inputs, labels, sampled, tries, want = _run_of(case, i)
        assert ao.step(st, NORMS, inputs, labels, sampled, tries, _lr(case)) == pytest.approx(want, rel=1e-8), (case, i)
    for k, want in _tables(case, "var_final").items():
        np.testing.assert_allclose(st.w[k], want, rtol=1e-8, atol=1e-12, err_msg="%s: %s" % (case, k))


def _check_final(case, got, start):
    """Final variables: the movement of every table within the suite's tolerances."""
    for k, want in _tables(case, "var_final").items():
        g, s, w = got[k], start[k], want.reshape(got[k].shape)
        np.testing.assert_allclose(g - s, w - s, rtol=5e-3, atol=3e-6 + 2e-3 * np.abs(w - s).max(),
                                   err_msg="%s: %s" % (case, k))


@pytest.mark.parametrize("case", CASES)
def test_emulated_engine_reproduces_the_reference_graph(emu, case):  # noqa: F811
    start = _tables(case, "var0")
    tables = {k: HostTable(v.astype(np.float32), NORMS.get(k, False)) for k, v in start.items()}
    for t in tables.values():
        t.s1[:] = 0.1                                     # TF's Adagrad accumulator starts at 0.1
        t.s1[:, t.d:] = 1.0
    cfg = L.OptCfg(L.OPT_ADAGRAD, _lr(case), 0.9, 0.999, 1e-8, 1)
    for i in range(2):
        inputs, labels, sampled, tries, want = _run_of(case, i)
        rc, got = _run(emu, tables, inputs, labels, sampled, tries, 1.0 / len(inputs))
        assert rc == 0 and got == pytest.approx(want, rel=2e-4), (case, i)
        for tab in tables.values():
            assert emu.oea_rowopt_apply(C.byref(tab.struct), C.byref(cfg), None) == 0
    _check_final(case, {k: t.weight[:, :t.d].astype(np.float64) for k, t in tables.items()}, start)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_engine_reproduces_the_reference_graph_on_the_gpu(cuda_device, case):
    from openea_b200 import engine as eng
    start = _tables(case, "var0")
    tabs = {k: eng.EmbeddingTable(v.astype(np.float32), NORMS.get(k, False), "Adagrad") for k, v in start.items()}
    tr = eng.NceTrainer(tuple(tabs[k] for k in NAMES), META[case]["num_sampled"], _lr(case))
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).cuda()
    for i in range(2):
        inputs, labels, sampled, tries, want = _run_of(case, i)
        tr.score_fed(dev(inputs), dev(labels), dev(sampled), dev([tries]))
        tr.apply()
        assert tr.read_loss() == pytest.approx(want, rel=2e-4), (case, i)
    _check_final(case, {k: t.raw().double().cpu().numpy() for k, t in tabs.items()}, start)
