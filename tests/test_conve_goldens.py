"""ConvE against the reference's OWN graph code.  tests/golden/path_i_conve.npz was produced by executing the reference's
`ConvE._define_variables` / `_define_embed_graph` and two `session.run([triple_loss, triple_optimizer], feed_dict)` per
case on a TensorFlow-1 graph interpreter (oracle/tf1_shim.py with scripts/tf1_shim_proje.py and
scripts/tf1_shim_conve.py: layers.batch_normalization in inference mode on any axis, channels-first conv2d with 'same'
padding, contrib.layers.fully_connected, dropout from a recorded counter stream, the candidate sampler and nce_loss;
float64; scripts/make_golden_conve.py): the shipped configuration (d = 12, a 4 × 3 image, keep_prob 0.7); d = 7, a 1 × 7
image, keep_prob 1; d = 10 with keep_prob 0.5; and a sampled set of every class.  So the golden pins the readings of
conve.py a restatement could get wrong: each batch norm's axis, fully_connected's default ReLU, the stacking and the
channel-first flatten order, the kernel's layout, and dropout's scaling.

  * tests/conve_oracle.py, given the recorded masks, reproduces every loss and the final variables to 1e-8;
  * the recorded masks are the device's counter stream for the recorded seed;
  * the engine, started from the same variables and fed the same batches, sampled sets and dropout seeds, reproduces
    every loss and the variables after the last run: the kernels' sources on the warp emulator (CPU) and liboea.so
    (`-m gpu`).
"""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from openea_b200 import lib as L
from tests import conve_oracle as co
from tests.test_emu_conve import _run
from tests.test_emu_proje import HostTable, emu  # noqa: F401  (emu: fixture)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "path_i_conve.npz")
G = np.load(GOLDEN)
META = json.loads(bytes(G["meta"]).decode())
CASES = sorted(META)
NORMS = {"ent": True, "rel": True}


def _tables(case, stage):
    """The golden's variables as the engine's eight tables (include/oea.h oea_conve)."""
    v = lambda n: G["%s/%s/%s" % (case, stage, n)]
    k = v("cnn/conv2d/kernel")                                       # [3, 3, 1, F]
    F = k.shape[3]
    conv = np.concatenate([k[:, :, 0, :].transpose(2, 0, 1).reshape(F, 9), v("cnn/conv2d/bias")[:, None],
                           v("batch_normalization_1/gamma")[:, None], v("batch_normalization_1/beta")[:, None]], 1)
    return {"ent": v("relationalembeddings/ent_embeds"), "rel": v("relationalembeddings/rel_embeds"),
            "w": v("probparameters/entity_w"), "b": v("probparameters/entity_b").reshape(-1, 1), "conv": conv,
            "bn_in": np.stack([v("batch_normalization/gamma"), v("batch_normalization/beta")]),
            "fc_w": v("fully_connected/weights"),
            "fc_out": np.stack([v("fully_connected/biases"), v("batch_normalization_2/gamma"),
                                v("batch_normalization_2/beta")])}


def _args(case):
    return META[case]["args"]


def _run_of(case, i):
    f = lambda k: G["%s/run%d/%s" % (case, i, k)]
    pos = np.stack([f("feed/pos_hs"), f("feed/pos_rs"), f("feed/pos_ts")]).astype(np.int32)
    keep = _args(case)["output_keep_prob"]
    n, d, F = pos.shape[1], _args(case)["dim"], _args(case)["filter_num"]
    if keep < 1:
        m0, m1 = f("mask0"), f("mask1")
    else:
        m0, m1 = np.ones((n, 2 * d), bool), np.ones((n, 2 * F * d), bool)
    return pos, f("sampled").astype(np.int32), int(f("num_tries")), int(f("dropout_seed")), m0, m1, float(f("loss"))


def test_golden_covers_the_cases():
    assert CASES == ["conve", "conve_d10", "conve_every_class", "conve_prime"]
    assert co.dim_factorization(_args("conve_prime")["dim"])[0] == 1
    assert _args("conve")["output_keep_prob"] < 1 and _args("conve_prime")["output_keep_prob"] == 1
    assert len(_run_of("conve_every_class", 0)[1]) == META["conve_every_class"]["entities"]


@pytest.mark.parametrize("case", [c for c in CASES if META[c]["args"]["output_keep_prob"] < 1])
def test_recorded_masks_are_the_device_counter_stream(case):
    a = _args(case)
    for i in range(2):
        pos, _, _, seed, m0, m1, _ = _run_of(case, i)
        w0, w1 = co.masks(seed, pos.shape[1], a["dim"], a["filter_num"], a["output_keep_prob"])
        assert np.array_equal(m0, w0) and np.array_equal(m1, w1)
        assert 0 < m1.mean() < 1


@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_the_reference_graph(case):
    a = _args(case)
    st = co.DenseState(_tables(case, "var0"), "Adam")
    for i in range(2):
        pos, sampled, tries, _, m0, m1, want = _run_of(case, i)
        got = co.step(st, NORMS, pos, sampled, tries, a["output_keep_prob"], m0, m1, a["learning_rate"])
        assert got == pytest.approx(want, rel=1e-8), (case, i)
    for k, want in _tables(case, "var_final").items():
        np.testing.assert_allclose(st.w[k], want, rtol=1e-8, atol=1e-12, err_msg="%s: %s" % (case, k))


def _check_final(case, got, start):
    """Final variables: every table's movement within the suite's tolerance.  An element whose gradient is at the level
    of fp32 rounding may take an Adam step of up to lr either way, so each may differ by 2·lr per run."""
    lr = _args(case)["learning_rate"]
    for k, want in _tables(case, "var_final").items():
        g, s, w = got[k], start[k], want.reshape(got[k].shape)
        assert np.abs(g - w).max() <= 2 * 2 * lr + 1e-6, (case, k)
        close = np.abs((g - s) - (w - s)) <= 3e-6 + 5e-3 * np.abs(w - s) + 2e-3 * np.abs(w - s).max()
        assert close.mean() >= 0.99, (case, k, float(close.mean()))


def _lossrel(case):
    a = _args(case)
    pitch = (a["dim"] + 3) // 4 * 4
    from tests.test_emu_conve import gamma
    return 8 * gamma(2 * a["filter_num"] * a["dim"] + 9 * a["filter_num"] + a["dnn_neg_nums"] + pitch + 64)


@pytest.mark.parametrize("case", CASES)
def test_emulated_engine_reproduces_the_reference_graph(emu, case):  # noqa: F811
    a = _args(case)
    start = _tables(case, "var0")
    tables = {k: HostTable(v.astype(np.float32), NORMS.get(k, False)) for k, v in start.items()}
    for i in range(2):
        pos, sampled, tries, seed, _, _, want = _run_of(case, i)
        rc, got = _run(emu, tables, pos, sampled, tries, a["output_keep_prob"], seed)
        assert rc == 0 and got == pytest.approx(want, rel=_lossrel(case)), (case, i)
        for tab in tables.values():
            tab.adam_t += 1
            cfg = L.OptCfg(L.OPT_ADAM, a["learning_rate"], 0.9, 0.999, 1e-8, tab.adam_t)
            assert emu.oea_rowopt_apply(C.byref(tab.struct), C.byref(cfg), None) == 0
    _check_final(case, {k: t.weight[:, :t.d].astype(np.float64) for k, t in tables.items()}, start)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_engine_reproduces_the_reference_graph_on_the_gpu(cuda_device, case):
    from openea_b200 import engine as eng
    a = _args(case)
    start = _tables(case, "var0")
    tabs = {k: eng.EmbeddingTable(v.astype(np.float32), NORMS.get(k, False), "Adam") for k, v in start.items()}
    tr = eng.ConvETrainer(tuple(tabs[k] for k in co.NAMES), len(_run_of(case, 0)[1]), a["learning_rate"],
                          a["output_keep_prob"])
    for i in range(2):
        pos, sampled, tries, seed, _, _, want = _run_of(case, i)
        dev = lambda x: torch.from_numpy(np.ascontiguousarray(x, dtype=np.int32)).cuda()
        tr.score_fed(dev(pos), dev(sampled), dev([tries]), dropout_seed=seed)
        tr.apply()
        assert tr.read_loss() == pytest.approx(want, rel=_lossrel(case)), (case, i)
    _check_final(case, {k: t.raw().double().cpu().numpy() for k, t in tabs.items()}, start)
