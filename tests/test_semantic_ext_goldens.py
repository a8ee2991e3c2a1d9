"""RotatE, HolE and BootEA_RotatE against the reference's OWN graph code.  tests/golden/path_i_semantic_ext.npz was
produced by executing the reference's `_define_variables` / `_define_embed_graph` / `_define_alignment_graph` and
`session.run([loss, optimizer], feed_dict)` of the three classes on a TensorFlow-1 graph interpreter (oracle/tf1_shim.py
plus the ops added in scripts/make_golden_semantic_ext.py, float64).  The same classes of this package, started from the
same variables and fed the same batches, must reproduce every fetched loss (within 2·10⁻⁴) and the variables after the
last run, their movement included:

  * CPU: the kernels' sources on the warp emulator;
  * GPU (`-m gpu`): liboea.so.

The tests/semantic_ext_oracle.py restatement of the graphs is pinned to the same file at float64 precision.
"""
import json
import os

import numpy as np
import pytest
import torch

from tests import semantic_ext_oracle as so
from tests.test_emu_triple_core import cpu_engine      # noqa: F401  (fixture: the engine over the emulated library)
from tests.test_reference_graph_goldens import replay as _replay_path_i
import tests.test_reference_graph_goldens as golden_path_i

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "path_i_semantic_ext.npz")
G = np.load(GOLDEN)
META = json.loads(bytes(G["meta"]).decode())


def replay(case, engine, device, monkeypatch):
    """The path (i) replay of tests/test_reference_graph_goldens.py, pointed at this file's cases."""
    monkeypatch.setattr(golden_path_i, "G", G)
    monkeypatch.setattr(golden_path_i, "META", META)
    _replay_path_i(case, engine, device, monkeypatch)


def test_golden_file_covers_the_expected_cases():
    assert sorted(META) == ["bootea_rotate", "hole_k1", "hole_k3", "rotate"]
    assert [r["kind"] for r in META["bootea_rotate"]["runs"]] == ["triple", "align", "triple"]
    assert [r["k"] for r in META["rotate"]["runs"]] == [3, 3, 3]
    assert META["hole_k1"]["args"]["neg_triple_num"] == 1 and META["hole_k3"]["args"]["neg_triple_num"] == 3


@pytest.mark.parametrize("case", sorted(META))
def test_engine_on_the_emulator_reproduces_the_reference_graph(cpu_engine, monkeypatch, case):
    replay(case, cpu_engine, "cpu", monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(META))
def test_engine_on_the_gpu_reproduces_the_reference_graph(cuda_device, monkeypatch, case):
    from openea_b200 import engine
    replay(case, engine, "cuda", monkeypatch)


@pytest.mark.parametrize("case", sorted(META))
def test_oracle_reproduces_the_reference_graph(case):
    """tests/semantic_ext_oracle.py, float64, on the golden's batches: every loss to 1e-9 and the final variables."""
    meta = META[case]
    a = meta["args"]
    model = "HolE" if meta["class"].endswith("HolE") else "RotatE"
    names = {"re_ent_embeds": "re_ent", "im_ent_embeds": "im_ent", "rel_embeds": "rel", "ent_embeds": "ent"}
    norms = {names[v]: bool(a["rel_l2_norm"] if v == "rel_embeds" else a["ent_l2_norm"]) for v in meta["variables"]}
    w = {names[v]: G["%s/var0/%s" % (case, v)] for v in meta["variables"]}
    triple = so.DenseState(w, a["optimizer"])
    align = so.DenseState(w, a["optimizer"])          # BootEA_RotatE: the alignment optimiser owns its slots
    for i, run in enumerate(meta["runs"]):
        f = {k.rsplit("/", 1)[1]: G[k] for k in G.files if k.startswith("%s/run%d/feed/" % (case, i))}
        if run["kind"] == "triple":
            pos = np.stack([f["pos_hs"], f["pos_rs"], f["pos_ts"]])
            neg = np.stack([f["neg_hs"], f["neg_rs"], f["neg_ts"]])
            kw = dict(margin=a["margin"]) if model == "HolE" else dict(
                gamma=a["gamma"], neg_weight=1.0 / a["neg_triple_num"] if case == "rotate" else 1.0)
            state = triple
        else:
            pos, neg = np.stack([f["new_h"], f["new_r"], f["new_t"]]), None
            kw, state = dict(gamma=a["gamma"]), align
        val, grads = so.fwd_bwd(model, state.w, norms, pos, neg, **kw)
        assert val == pytest.approx(float(G["%s/run%d/loss" % (case, i)]), rel=1e-9), (case, i)
        state.apply(grads, a["learning_rate"])
        other = align if state is triple else triple
        for k in other.w:                              # both optimisers update the same variables
            other.w[k] = state.w[k]
    for v in meta["variables"]:
        np.testing.assert_allclose(triple.w[names[v]], G["%s/var_final/%s" % (case, v)], rtol=1e-9, atol=1e-12)


def test_fft_correlation_of_the_golden_rows_is_the_direct_sum():
    e = torch.as_tensor(G["hole_k3/var0/ent_embeds"])
    np.testing.assert_allclose(so.ccorr(e[:5], e[5:10]).numpy(), so.ccorr_direct(e[:5].numpy(), e[5:10].numpy()),
                               rtol=1e-10, atol=1e-12)
