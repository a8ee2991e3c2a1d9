"""ProjE against the reference's OWN graph code.  tests/golden/path_i_proje.npz was produced by executing the reference's
`ProjE._define_variables` / `_define_embed_graph` and two `session.run([triple_loss, triple_optimizer], feed_dict)` per
case on a TensorFlow-1 graph interpreter (oracle/tf1_shim.py with scripts/tf1_shim_proje.py: variable scopes with reuse,
contrib.layers.batch_norm, the unique log-uniform candidate sampler and nce_loss; float64; scripts/make_golden_proje.py):
the shipped configuration at E = 40, S = 12; d = 75 with E = 300, S = 64; a batch with repeated tails, tails inside the
sampled set and repeated heads; and a batch of one positive, where every batch norm sees a variance of 0.  Each run
records the sampled ids and num_tries it drew.  So the golden pins the readings of proje.py that a restatement could get
wrong: the beta the two input batch norms share, the one mlp_w returned twice, batch_norm's training-mode defaults, and
nce_loss's subtract_log_q with TF's expected counts.

  * tests/proje_oracle.py reproduces every loss and the final variables to 1e-8;
  * the engine, started from the same variables and fed the same batches and sampled sets, reproduces every loss within
    2·10⁻⁴ and the variables after the last run: the kernels' sources on the warp emulator (CPU) and liboea.so (`-m gpu`).
"""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from openea_b200 import lib as L
from tests import proje_oracle as po
from tests.test_emu_proje import HostTable, _run, emu  # noqa: F401  (emu: fixture)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "path_i_proje.npz")
G = np.load(GOLDEN)
META = json.loads(bytes(G["meta"]).decode())
CASES = sorted(META)
NORMS = {"ent": True, "rel": True}
NAMES = ("ent", "rel", "w", "b", "params")


def _tables(case, stage):
    """The golden's variables as the engine's five tables: entity_b as [E, 1]; params rows mlp_w, mlp_bias, the input
    beta, the output beta."""
    v = lambda n: G["%s/%s/%s" % (case, stage, n)]
    return {"ent": v("relationalembeddings/ent_embeds"), "rel": v("relationalembeddings/rel_embeds"),
            "w": v("probparameters/entity_w"), "b": v("probparameters/entity_b").reshape(-1, 1),
            "params": np.stack([v("mlp/mlp_w"), v("mlp/mlp_bias"), v("input_bn/bn/beta"), v("output_bn/bn/beta")])}


def _run_of(case, i):
    f = lambda k: G["%s/run%d/%s" % (case, i, k)]
    pos = np.stack([f("feed/pos_hs"), f("feed/pos_rs"), f("feed/pos_ts")]).astype(np.int32)
    return pos, f("sampled").astype(np.int32), int(f("num_tries")), float(f("loss"))


def _lr(case):
    return META[case]["args"]["learning_rate"]


def test_golden_covers_the_cases():
    assert CASES == ["proje", "proje_d75", "proje_one_positive", "proje_repeats"]
    assert _run_of("proje_one_positive", 0)[0].shape[1] == 1
    pos, sampled, _, _ = _run_of("proje_repeats", 0)
    assert np.isin(pos[2], sampled).any() and len(set(pos[2])) < pos.shape[1] and len(set(pos[0])) < pos.shape[1]
    assert any(_run_of(c, i)[2] > len(_run_of(c, i)[1]) for c in CASES for i in range(2))


@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_the_reference_graph(case):
    st = po.DenseState(_tables(case, "var0"), "Adam")
    for i in range(2):
        pos, sampled, tries, want = _run_of(case, i)
        assert po.step(st, NORMS, pos, sampled, tries, _lr(case)) == pytest.approx(want, rel=1e-8), (case, i)
    for k, want in _tables(case, "var_final").items():
        got = st.w[k]
        if k == "params":
            # mlp_bias and the input beta: gradients of 0 up to float64 rounding (~1e-14), which Adam's ε = 1e-8 keeps
            # to steps far below lr — but not below 1e-8 relative
            assert np.abs(got[1:3] - want[1:3]).max() < 1e-7, case
            got, want = got[[0, 3]], want[[0, 3]]
        np.testing.assert_allclose(got, want, rtol=1e-8, atol=1e-12, err_msg="%s: %s" % (case, k))


def test_oracle_expected_count_shortcut():
    """num_tries == S: q(c) = P(c)·S, not −expm1(S·log1p(−P))."""
    p = po.probability([0, 5], 40)
    np.testing.assert_array_equal(po.expected_count([0, 5], 40, 7, 7), p * np.float32(7))
    assert not np.allclose(po.expected_count([0, 5], 40, 7, 8), p * np.float32(7))


def _check_final(case, got, start):
    """Final variables: the movement of every table within the suite's tolerances.  mlp_bias and the input beta reach
    the loss only through the output batch norm, which cancels them, so their gradient is 0 up to rounding; in fp32
    Adam turns that rounding into steps of up to lr either way, so those two rows are held to that bound."""
    lr = _lr(case)
    for k, want in _tables(case, "var_final").items():
        g, s, w = got[k], start[k], want.reshape(got[k].shape)
        if k == "params":
            assert np.abs(g[1:3] - w[1:3]).max() <= 2 * 2 * lr + 1e-6, case
            g, s, w = g[[0, 3]], s[[0, 3]], w[[0, 3]]
        np.testing.assert_allclose(g - s, w - s, rtol=5e-3, atol=3e-6 + 2e-3 * np.abs(w - s).max(),
                                   err_msg="%s: %s" % (case, k))


@pytest.mark.parametrize("case", CASES)
def test_emulated_engine_reproduces_the_reference_graph(emu, case):  # noqa: F811
    start = _tables(case, "var0")
    tables = {k: HostTable(v.astype(np.float32), NORMS.get(k, False)) for k, v in start.items()}
    for i in range(2):
        pos, sampled, tries, want = _run_of(case, i)
        rc, got = _run(emu, tables, pos, sampled, tries)
        assert rc == 0 and got == pytest.approx(want, rel=2e-4), (case, i)
        for tab in tables.values():
            tab.adam_t += 1
            cfg = L.OptCfg(L.OPT_ADAM, _lr(case), 0.9, 0.999, 1e-8, tab.adam_t)
            assert emu.oea_rowopt_apply(C.byref(tab.struct), C.byref(cfg), None) == 0
    _check_final(case, {k: t.weight[:, :t.d].astype(np.float64) for k, t in tables.items()}, start)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_engine_reproduces_the_reference_graph_on_the_gpu(cuda_device, case):
    from openea_b200 import engine as eng
    start = _tables(case, "var0")
    tabs = {k: eng.EmbeddingTable(v.astype(np.float32), NORMS.get(k, False), "Adam") for k, v in start.items()}
    tr = eng.ProjETrainer(tuple(tabs[k] for k in NAMES), len(_run_of(case, 0)[1]), _lr(case))
    for i in range(2):
        pos, sampled, tries, want = _run_of(case, i)
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).cuda()
        tr.score_fed(dev(pos), dev(sampled), dev([tries]))
        tr.apply()
        assert tr.read_loss() == pytest.approx(want, rel=2e-4), (case, i)
    _check_final(case, {k: t.raw().double().cpu().numpy() for k, t in tabs.items()}, start)
