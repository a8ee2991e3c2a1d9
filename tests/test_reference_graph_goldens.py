"""Path (i) against the reference's OWN graph code.  tests/golden/path_i_reference_graphs.npz was produced by executing
the reference's `_define_variables` / `_define_embed_graph` / `_define_alignment_graph` / mapping module and
`session.run([loss, optimizer], feed_dict)` for 15 model classes on a TensorFlow-1 graph interpreter
(oracle/tf1_shim.py, float64; scripts/make_golden_path_i.py).  Here the SAME classes of this package are built with the
same hyper-parameters, started from the same variables, fed the same batches through the engine's entry points, and
must reproduce every fetched loss and all variables after the last run:

  * CPU: the kernels' sources on the warp emulator (the whole suite runs where no GPU exists);
  * GPU (`-m gpu`): liboea.so.

What this pins: which variables exist and which are normalised, every loss expression and its constants (e.g. that
get_loss_func's limited loss ignores neg_margin_balance while AlignE's passes it), sums vs means, which optimiser
instance owns which slots.  What it cannot pin offline: TensorFlow's op and optimiser semantics, restated in the shim.
"""
import json
import os
import types

import numpy as np
import pytest
import torch

from tests.test_emu_triple_core import cpu_engine      # noqa: F401  (fixture: the engine over the emulated library)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "path_i_reference_graphs.npz")
G = np.load(GOLDEN)
META = json.loads(bytes(G["meta"]).decode())

ATTR = {"mapping_matrix": "mapping_mat", "mapping_matrix_1": "mapping_mat_1", "mapping_matrix_2": "mapping_mat_2"}


def _class(path):
    import importlib
    module, name = path.rsplit(".", 1)
    return getattr(importlib.import_module(module.replace("openea.", "openea_b200.", 1)), name)


def _feed(case, i):
    prefix = "%s/run%d/feed/" % (case, i)
    return {k[len(prefix):]: G[k] for k in G.files if k.startswith(prefix)}


def _hrt(feed, keys, device):
    return torch.from_numpy(np.stack([feed[k] for k in keys]).astype(np.int32)).to(device)


def replay(case, engine, device, monkeypatch):
    from openea_b200.modules.base import initializers
    meta = META[case]
    monkeypatch.setattr(initializers, "_make", lambda values, norm, optimizer=None: engine.EmbeddingTable(
        values, bool(norm), optimizer or initializers._DEFAULT_OPT, device))
    model = _class(meta["class"])()
    model.args = types.SimpleNamespace(**meta["args"])
    model.kgs = types.SimpleNamespace(entities_num=40, relations_num=6)
    for name in meta["defines"]:
        if hasattr(model, name):
            getattr(model, name)()
    tables = {}
    for name in meta["variables"]:
        tab = getattr(model, ATTR.get(name, name))
        start = G["%s/var0/%s" % (case, name)]
        assert tab.weight[:, :tab.dim].shape == start.shape, name
        tab.weight[:, :tab.dim] = torch.as_tensor(start, dtype=torch.float32, device=tab.weight.device)
        tables[name] = tab
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    losses = []
    for i, run in enumerate(meta["runs"]):
        f = _feed(case, i)
        kind = run["kind"]
        if kind in ("triple", "label"):
            tr = model.triple_trainer
            if kind == "label":
                n_pos = int((f["label"] > 0).sum())
                both = np.stack([f["hs"], f["rs"], f["ts"]]).astype(np.int32)
                pos, neg = dev(both[:, :n_pos]), dev(both[:, n_pos:])
            else:
                pos = _hrt(f, ("pos_hs", "pos_rs", "pos_ts"), device)
                neg = _hrt(f, ("neg_hs", "neg_rs", "neg_ts"), device) if "neg_hs" in f else None
            tr.score_fed(pos, neg)
            tr.apply()
            losses.append(tr.read_loss())
        elif kind == "align":
            tr = model.alignment_trainer
            tr.score_fed(_hrt(f, ("new_h", "new_r", "new_t"), device))
            tr.apply()
            losses.append(tr.read_loss())
        elif kind == "mapping":
            losses.append(model.mapping_trainer.step(f["seed_entities1"], f["seed_entities2"]))
        elif kind == "ptranse":
            tr = model.triple_trainer
            tr.score_fed(_hrt(f, ("pos_hs", "pos_rs", "pos_ts"), device), _hrt(f, ("neg_hs", "neg_rs", "neg_ts"), device))
            tr.score_margin_weighted(_hrt(f, ("pos_rx", "pos_ry", "pos_r"), device), _hrt(f, ("neg_rx", "neg_ry", "neg_r"), device),
                                     dev(f["path_weight"]), reciprocal=True, scale=model.args.path_parm, paths=True)
            tr.apply()
            losses.append(tr.read_loss())
        elif kind == "ipt_align":
            tr = model.alignment_trainer
            tr.score_margin_weighted(_hrt(f, ("new_ph", "new_pr", "new_pt"), device), _hrt(f, ("new_nh", "new_nr", "new_nt"), device),
                                     dev(f["tr_weight"]))
            tr.apply()
            losses.append(tr.read_loss())
        elif kind == "sea_map":
            model.mapping_trainer.step(f["labeled_entities1"], f["labeled_entities2"], f["unlabeled_entities1"],
                                       f["unlabeled_entities2"])
            losses.append(model.mapping_trainer.read_loss())
        elif kind == "imuse_align":
            tr = model.alignment_trainer
            tr.score_pairs(f["aligned_ents1"], f["aligned_ents2"])
            tr.apply()
            losses.append(tr.read_loss())
        else:
            raise AssertionError(kind)
    for i, got in enumerate(losses):
        assert got == pytest.approx(float(G["%s/run%d/loss" % (case, i)]), rel=2e-4), (case, i, meta["runs"][i])
    for name, tab in tables.items():
        want = G["%s/var_final/%s" % (case, name)]
        start = G["%s/var0/%s" % (case, name)]
        got = tab.raw().cpu().numpy()
        assert np.abs(want - start).max() > 0, name                 # every variable of the case was trained
        # compare the MOVEMENT too: a wrong update direction hides behind the start values at rtol alone
        np.testing.assert_allclose(got - start, want - start, rtol=5e-3, atol=3e-6 + 2e-3 * np.abs(want - start).max(),
                                   err_msg="%s: %s" % (case, name))
        np.testing.assert_allclose(got, want, rtol=2e-4, atol=5e-6, err_msg="%s: %s" % (case, name))


@pytest.mark.parametrize("case", sorted(META))
def test_engine_on_the_emulator_reproduces_the_reference_graph(cpu_engine, monkeypatch, case):
    from openea_b200.approaches import imuse, iptranse, sea
    for mod in (imuse, iptranse, sea):
        monkeypatch.setattr(mod, "load_session", lambda: None, raising=False)
    replay(case, cpu_engine, "cpu", monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(META))
def test_engine_on_the_gpu_reproduces_the_reference_graph(cuda_device, monkeypatch, case):
    from openea_b200 import engine
    replay(case, engine, "cuda", monkeypatch)


def test_golden_file_covers_the_expected_cases():
    assert set(META) >= {"aligne_limited", "bootea", "mtranse", "transe_margin_adam", "transh", "transd", "distmult",
                         "simple", "bootea_transh", "iptranse", "sea", "imuse"}
    for case, meta in META.items():
        assert meta["class"].startswith("openea.") and len(meta["runs"]) >= 2


ORACLE_CASES = {     # case → (loss, loss_norm, normalised?, optimiser, kwargs of the C oracle's step)
    "aligne_limited": ("limited", "L2", True, "Adagrad", dict(margin=0.01, neg_margin=2.0, balance=0.2)),
    "transe_limited_d75": ("limited", "L2", True, "Adagrad", dict(margin=0.01, neg_margin=2.0, balance=1.0)),
    "transe_margin_l1_sgd": ("margin-based", "L1", True, "SGD", dict(margin=1.5)),
    "transe_margin_adam": ("margin-based", "L2", True, "Adam", dict(margin=1.5)),
}


@pytest.mark.parametrize("case", sorted(ORACLE_CASES))
def test_c_oracle_reproduces_the_reference_graph(case):
    """The CPU oracle (oracle/oea_oracle.c, what the GPU parity tests and bench.py's CPU leg use) is itself pinned to the
    goldens: losses of every run and the variables after the last one."""
    from oracle import triple as orc
    loss, loss_norm, norm, opt, kw = ORACLE_CASES[case]
    meta = META[case]
    st = orc.DenseState(G[case + "/var0/ent_embeds"].astype(np.float32), G[case + "/var0/rel_embeds"].astype(np.float32), opt)
    for i, run in enumerate(meta["runs"]):
        f = _feed(case, i)
        pos = np.stack([f["pos_hs"], f["pos_rs"], f["pos_ts"]]).astype(np.int32)
        neg = np.stack([f["neg_hs"], f["neg_rs"], f["neg_ts"]]).astype(np.int32)
        got = orc.step(st, pos, neg, loss, loss_norm, norm, norm, meta["args"]["learning_rate"], **kw)
        assert got == pytest.approx(float(G["%s/run%d/loss" % (case, i)]), rel=2e-4), (case, i)
    np.testing.assert_allclose(st.ent, G[case + "/var_final/ent_embeds"], rtol=2e-4, atol=5e-6)
    np.testing.assert_allclose(st.rel, G[case + "/var_final/rel_embeds"], rtol=2e-4, atol=5e-6)


# ---- path (ii): GCN-Align's unit, from the reference's GCN_Align_Unit / align_loss / construct_feed_dict ------------
GCN = np.load(os.path.join(os.path.dirname(GOLDEN), "path_ii_gcn_align.npz"))


def replay_gcn_align(engine, device, branch):
    import scipy.sparse as sp
    from openea_b200 import gnn
    from openea_b200.approaches.gcn_align import GCNAlignUnit
    n, n_feat, dim, t, k = (int(x) for x in GCN["dims"])
    coo = lambda name, shape: sp.coo_matrix((GCN[name + "/values"], (GCN[name + "/coords"][:, 0], GCN[name + "/coords"][:, 1])),
                                            shape=shape)
    support = gnn.DeviceCsr(coo("support", (n, n)), device)
    features = None if branch == "se" else gnn.DeviceCsr(coo("features", (n, n_feat)), device)
    table = engine.EmbeddingTable(GCN[branch + "/var0"].astype(np.float32), True, "SGD", device)
    unit = GCNAlignUnit(support, table, features, GCN["ill"], float(GCN["gamma"]), k, float(GCN["lr"]))
    for step in range(3):
        neg = [torch.as_tensor(GCN["%s/run%d/%s" % (branch, step, key)], dtype=torch.int32, device=device)
               for key in ("neg_left", "neg_right", "neg2_left", "neg2_right")]
        loss = float(unit.train_step(*neg).item())
        assert loss == pytest.approx(float(GCN["%s/run%d/loss" % (branch, step)]), rel=2e-4), (branch, step)
    want, start = GCN[branch + "/var_final"], GCN[branch + "/var0"]
    got = table.raw().cpu().numpy()
    np.testing.assert_allclose(got - start, want - start, rtol=5e-3, atol=2e-3 * np.abs(want - start).max())
    np.testing.assert_allclose(unit.forward()[:, :dim].cpu().numpy(), GCN[branch + "/outputs_final"], rtol=5e-4, atol=1e-5)


@pytest.mark.parametrize("branch", ["se", "ae"])
def test_gcn_align_unit_on_the_emulator_reproduces_the_reference_unit(cpu_engine, branch):
    replay_gcn_align(cpu_engine, "cpu", branch)


@pytest.mark.gpu
@pytest.mark.parametrize("branch", ["se", "ae"])
def test_gcn_align_unit_on_the_gpu_reproduces_the_reference_unit(cuda_device, branch):
    from openea_b200 import engine
    replay_gcn_align(engine, "cuda", branch)


# ---- path (ii): RDGCN's whole layer, from the reference's Layer.build() + AdamOptimizer ---------------------------------
RD = np.load(os.path.join(os.path.dirname(GOLDEN), "path_ii_rdgcn.npz"))
RD_NAMES = sorted(k[len("var0/"):] for k in RD.files if k.startswith("var0/"))


def _rdgcn_to_param(name, ref):
    """Reference variable → this package's parameter layout (approaches/rdgcn.py: conv kernels without the leading 1,
    1-filter kernels and their biases replicated to 4 columns for the 16-byte row optimiser, vectors as [1, d])."""
    a = np.asarray(ref, dtype=np.float32)
    if a.ndim == 3:
        a = a[0]
    if a.ndim == 1:
        a = a[None, :]
    if name.endswith((".f1.w", ".f2.w")) or name in ("sp1.w", "sp2.w"):
        a = np.repeat(a, 4, axis=1)
    if name.endswith((".f1.b", ".f2.b")) or name in ("sp1.b", "sp2.b"):
        a = np.repeat(a, 4, axis=1)
    return a


def replay_rdgcn(device):
    from openea_b200.approaches.alinet import DenseAdam
    from openea_b200.approaches.rdgcn import RDGCNLayer
    n_ent, n_rel, dim, t, k = (int(x) for x in RD["dims"])
    as_list = lambda a: [tuple(int(v) for v in row) for row in a]
    kgs = types.SimpleNamespace(train_links=as_list(RD["links"]), relations_num=n_rel, entities_num=n_ent,
                                kg1=types.SimpleNamespace(relation_triples_list=as_list(RD["triples1"])),
                                kg2=types.SimpleNamespace(relation_triples_list=as_list(RD["triples2"])))
    args = types.SimpleNamespace(dim=dim, dropout=0.0, gamma=float(RD["gamma"]), neg_triple_num=k, alpha=float(RD["alpha"]),
                                 beta=float(RD["beta"]), learning_rate=float(RD["lr"]))
    layer = RDGCNLayer(args, kgs, RD["var0/X0"].astype(np.float32), torch.device(device))
    assert sorted(layer.params) == RD_NAMES
    with torch.no_grad():
        for name in RD_NAMES:
            want = _rdgcn_to_param(name, RD["var0/" + name])
            assert tuple(layer.params[name].shape) == want.shape, (name, tuple(layer.params[name].shape), want.shape)
            layer.params[name].copy_(torch.as_tensor(want, device=device))
    opt = DenseAdam(list(layer.params.values()), args.learning_rate)
    for step in range(3):
        negs = tuple(torch.as_tensor(RD["run%d/%s" % (step, key)], dtype=torch.int32, device=device)
                     for key in ("neg_left", "neg_right", "neg2_left", "neg2_right"))
        loss = layer.loss(layer.forward(), negs)
        loss.backward()
        opt.step()
        assert float(loss.detach()) == pytest.approx(float(RD["run%d/loss" % step]), rel=2e-4), step
    for name in RD_NAMES:
        start, want = _rdgcn_to_param(name, RD["var0/" + name]), _rdgcn_to_param(name, RD["var_final/" + name])
        got = layer.params[name].detach().cpu().numpy()
        col = slice(0, 1) if want.shape[1] == 4 and name != "X0" and "." in name and name.split(".")[-1] in ("w", "b") \
            and (name.startswith(("sp", "self.f", "dual.f"))) else slice(None)
        move = np.abs(want - start).max()
        if move == 0.0:
            # a bias added to every logit of a softmax row has a mathematically zero gradient (sp1.b / sp2.b): float64
            # keeps it at exactly 0, in fp32 Adam normalises the rounding noise of that gradient (whose size depends on
            # the order of the atomic adds) into a drift of at most its step bound, lr per step
            assert np.abs(got - start).max() <= 3 * args.learning_rate * 1.01, name
            continue
        np.testing.assert_allclose((got - start)[:, col], (want - start)[:, col], rtol=2e-2, atol=3e-2 * move + 1e-7, err_msg=name)
    with torch.no_grad():
        np.testing.assert_allclose(layer.forward()[:, :dim].cpu().numpy(), RD["outputs_final"], rtol=2e-3, atol=2e-5)


def test_rdgcn_layer_on_the_emulator_reproduces_the_reference_layer(cpu_engine):
    replay_rdgcn("cpu")


@pytest.mark.gpu
def test_rdgcn_layer_on_the_gpu_reproduces_the_reference_layer(cuda_device):
    replay_rdgcn("cuda")


# ---- path (ii): AliNet's whole graph, from the reference's _get_variable / _generate_rel_graph + AdamOptimizer ---------
AL = np.load(os.path.join(os.path.dirname(GOLDEN), "path_ii_alinet.npz"))
AL_NAMES = {"init_embedding": "init_embedding", "gcn_0_kernel_0": "gcn0.kernel", "gcn_0_bias": "gcn0.bias",
            "batch_normalization/gamma": "gcn0.bn_gamma", "batch_normalization/beta": "gcn0.bn_beta",
            "alinet_0_kernel": "gat0.kernel", "alinet_0_kernel_1": "gat0.kernel1", "alinet_0_kernel_2": "gat0.kernel2",
            "batch_normalization_1/gamma": "gat0.bn_gamma", "batch_normalization_1/beta": "gat0.bn_beta",
            "highwaykernel": "hw0.kernel", "batch_normalization_2/gamma": "hw0.bn_gamma",
            "batch_normalization_2/beta": "hw0.bn_beta", "gcn_1_kernel_0": "gcn1.kernel", "gcn_1_bias": "gcn1.bias",
            "batch_normalization_3/gamma": "gcn1.bn_gamma", "batch_normalization_3/beta": "gcn1.bn_beta"}


def replay_alinet(device):
    import scipy.sparse as sp
    from openea_b200 import gnn
    from openea_b200.approaches.alinet import AliNetModel, DenseAdam
    n, win = int(AL["dims"][0]), int(AL["dims"][-1])
    dims = [int(x) for x in AL["dims"][1:-1]]
    coo = lambda name: sp.coo_matrix((AL[name + "/values"], (AL[name + "/coords"][:, 0], AL[name + "/coords"][:, 1])), shape=(n, n))
    model = AliNetModel(n, dims, gnn.DeviceCsr(coo("one"), device), gnn.DeviceCsr(coo("two"), device), torch.device(device))
    assert sorted(model.params) == sorted(AL_NAMES.values())
    as2d = lambda a: np.asarray(a, dtype=np.float32).reshape(1, -1) if np.ndim(a) == 1 else np.asarray(a, dtype=np.float32)
    with torch.no_grad():
        for ref, mine in AL_NAMES.items():
            want = as2d(AL["var0/" + ref])
            assert tuple(model.params[mine].shape) == want.shape, (ref, mine)
            model.params[mine].copy_(torch.as_tensor(want, device=device))
    opt = DenseAdam(list(model.params.values()), float(AL["lr"]))
    idx = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.long, device=device)
    for step in range(3):
        outs = model.forward()
        loss = model.loss(outs, idx(AL["run%d/pos" % step]), idx(AL["run%d/neg" % step]), float(AL["neg_margin"]),
                          float(AL["balance"]), hs=idx(AL["run%d/hs" % step]), ts=idx(AL["run%d/ts" % step]), rel_win=win,
                          rel_param=float(AL["rel_param"]))
        loss.backward()
        opt.step()
        assert float(loss.detach()) == pytest.approx(float(AL["run%d/loss" % step]), rel=2e-4), step
    for ref, mine in AL_NAMES.items():
        start, want = as2d(AL["var0/" + ref]), as2d(AL["var_final/" + ref])
        got = model.params[mine].detach().cpu().numpy()
        move = np.abs(want - start).max()
        assert move > 0, ref
        np.testing.assert_allclose(got - start, want - start, rtol=2e-2, atol=3e-2 * move, err_msg=ref)
    with torch.no_grad():
        for i, out in enumerate(model.forward()):
            np.testing.assert_allclose(out[:, :dims[i + 1]].cpu().numpy(), AL["outputs_final/%d" % i], rtol=2e-3, atol=2e-5)


def test_alinet_model_on_the_emulator_reproduces_the_reference_graph(cpu_engine):
    replay_alinet("cpu")


@pytest.mark.gpu
def test_alinet_model_on_the_gpu_reproduces_the_reference_graph(cuda_device):
    replay_alinet("cuda")


# ---- AttrE: structure + character-level + joint losses, from the reference's _define_embed_graph ----------------------
AT = np.load(os.path.join(os.path.dirname(GOLDEN), "path_i_attre.npz"))


def replay_attre(engine, device, monkeypatch):
    from openea_b200.approaches.attre import AttrE, ngram_weights
    from openea_b200.modules.base import initializers
    n_attr, n_val, n_char, lit, batch, dim = (int(x) for x in AT["dims"])
    monkeypatch.setattr(initializers, "_make", lambda values, norm, optimizer=None: engine.EmbeddingTable(
        values, bool(norm), optimizer or initializers._DEFAULT_OPT, device))
    model = AttrE()
    model.args = types.SimpleNamespace(dim=dim, init="normal", ent_l2_norm=True, rel_l2_norm=True, attr_l2_norm=True,
                                       char_l2_norm=True, loss="margin-based", loss_norm="L2", margin=1.5, learning_rate=0.01,
                                       optimizer="SGD", batch_size=batch, neg_triple_num=1, literal_len=lit)
    model.kgs = types.SimpleNamespace(entities_num=40, relations_num=6, attributes_num=n_attr)
    model.value_id_char_ids, model.char_list_size = AT["chars"], n_char
    model._define_variables()
    model._define_embed_graph()
    names = sorted(k[len("var0/"):] for k in AT.files if k.startswith("var0/"))
    for name in names:
        tab = getattr(model, name)
        tab.weight[:, :dim] = torch.as_tensor(AT["var0/" + name], dtype=torch.float32, device=tab.weight.device)
    # the composition weights are the suffix-mean sum of attre.py:89-107 written out
    np.testing.assert_allclose(ngram_weights(4), [1 / 4 + 1 / 3 + 1 / 2 + 1, 1 / 4 + 1 / 3 + 1 / 2, 1 / 4 + 1 / 3, 1 / 4], rtol=1e-6)
    i = 0
    while "run%d/loss" % i in AT.files:
        kind = bytes(AT["run%d/kind" % i]).decode()
        f = {k[len("run%d/feed/" % i):]: AT[k] for k in AT.files if k.startswith("run%d/feed/" % i)}
        dev = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.int32, device=device)
        if kind == "triple":
            tr = model.triple_trainer
            tr.score_fed(_hrt(f, ("pos_hs", "pos_rs", "pos_ts"), device), _hrt(f, ("neg_hs", "neg_rs", "neg_ts"), device))
            tr.apply()
            got = tr.read_loss()
        elif kind == "ce":
            got = float(model.ce_step(_hrt(f, ("pos_es", "pos_as", "pos_vs"), device), _hrt(f, ("neg_es", "neg_as", "neg_vs"), device)))
        else:
            got = float(model.joint_step(dev(f["joint_ents"])))
        assert got == pytest.approx(float(AT["run%d/loss" % i]), rel=2e-4), (i, kind)
        i += 1
    for name in names:
        start, want = AT["var0/" + name], AT["var_final/" + name]
        got = getattr(model, name).raw().cpu().numpy()
        move = np.abs(want - start).max()
        assert move > 0, name
        np.testing.assert_allclose(got - start, want - start, rtol=5e-3, atol=3e-6 + 2e-3 * move, err_msg=name)


def test_attre_on_the_emulator_reproduces_the_reference_graph(cpu_engine, monkeypatch):
    import ctypes as C
    from openea_b200.modules.base import losses
    monkeypatch.setattr(losses, "_stream_ptr", lambda: C.c_void_p(0))
    replay_attre(cpu_engine, "cpu", monkeypatch)


@pytest.mark.gpu
def test_attre_on_the_gpu_reproduces_the_reference_graph(cuda_device, monkeypatch):
    from openea_b200 import engine
    replay_attre(engine, "cuda", monkeypatch)


# ---- the other oracles, held to the same goldens -------------------------------------------------------------------
EXT_CASES = {   # case → (model of oracle.triple_ext, {oracle slot: reference variable}, loss, kwargs, mean loss?)
    "transh": ("TransH", {"ent": "ent_embeds", "rel": "rel_embeds", "normal": "normal_vector"}, "margin-based", dict(margin=1.5), False),
    "transd": ("TransD", {"ent": "ent_embeds", "rel": "rel_embeds", "ent_transfer": "ent_transfer", "rel_transfer": "rel_transfer"},
               "margin-based", dict(margin=1.5), False),
    "simple": ("SimplE", {"head_ent": "head_ent_embeds", "rel1": "rel_embeds1", "tail_ent": "tail_ent_embeds", "rel2": "rel_embeds2"},
               "logistic", {}, False),
    "distmult": ("DistMult", {"ent": "ent_embeds", "rel": "rel_embeds"}, "logistic", {}, True),
}


@pytest.mark.parametrize("case", sorted(EXT_CASES))
def test_score_family_oracle_reproduces_the_reference_graph(case):
    """oracle/triple_ext.py (the float64 restatement the score-family kernels are tested against on the GPU)."""
    from oracle import triple_ext as ox
    model, slots, loss, kw, mean = EXT_CASES[case]
    meta = META[case]
    st = ox.DenseState({slot: G["%s/var0/%s" % (case, name)] for slot, name in slots.items()}, "Adagrad")
    norms = {slot: True for slot in slots}
    for i, run in enumerate(meta["runs"]):
        f = _feed(case, i)
        if run["kind"] == "label":
            n_pos = int((f["label"] > 0).sum())
            both = np.stack([f["hs"], f["rs"], f["ts"]]).astype(np.int32)
            pos, neg = both[:, :n_pos], both[:, n_pos:]
        else:
            pos = np.stack([f["pos_hs"], f["pos_rs"], f["pos_ts"]]).astype(np.int32)
            neg = np.stack([f["neg_hs"], f["neg_rs"], f["neg_ts"]]).astype(np.int32)
        scale = 1.0 / (pos.shape[1] + neg.shape[1]) if mean else 1.0
        got = ox.step(st, model, norms, pos, neg, loss, meta["args"]["learning_rate"], scale=scale, **kw)
        assert got == pytest.approx(float(G["%s/run%d/loss" % (case, i)]), rel=1e-9), (case, i)
    for slot, name in slots.items():
        np.testing.assert_allclose(st.w[slot], G["%s/var_final/%s" % (case, name)], rtol=1e-9, atol=1e-12, err_msg=name)


@pytest.mark.parametrize("branch", ["se", "ae"])
def test_gcn_align_oracle_reproduces_the_reference_unit(branch):
    """oracle/gnn.py's GCN-Align unit (what tests/test_gnn_gpu.py checks the kernels against)."""
    import scipy.sparse as sp
    from oracle import gnn as og
    n, n_feat, dim, t, k = (int(x) for x in GCN["dims"])
    coo = lambda name, shape: sp.coo_matrix((GCN[name + "/values"], (GCN[name + "/coords"][:, 0], GCN[name + "/coords"][:, 1])),
                                            shape=shape).tocsr()
    support = coo("support", (n, n))
    features = None if branch == "se" else coo("features", (n, n_feat))
    W = GCN[branch + "/var0"]
    for step in range(3):
        negs = [GCN["%s/run%d/%s" % (branch, step, key)] for key in ("neg_left", "neg_right", "neg2_left", "neg2_right")]
        loss, W, out = og.unit_train_step(support, W, features, GCN["ill"], float(GCN["gamma"]), k, negs, float(GCN["lr"]),
                                          dtype=torch.float64)
        assert loss == pytest.approx(float(GCN["%s/run%d/loss" % (branch, step)]), rel=1e-9)
    np.testing.assert_allclose(W, GCN[branch + "/var_final"], rtol=1e-9, atol=1e-12)
