"""CPU: the general sampled-NCE step and the pair draw (openea_b200/csrc/oea_proje.cu) on the warp emulator of
tests/emu, against the float64 oracle of tests/attr2vec_oracle.py (row widths 4-128, batches of 1-500, sampled sets from
one class to every class, repeated ids, accidental hits, TF's expected-count shortcut, raw and normalised tables), whole
Adagrad steps against dense TF Adagrad, the argument checks; Attr2Vec's training pairs and entity vectors against the
reference's own functions (recorded in tests/golden/reference_attr2vec.pkl.xz); and the Attr2Vec lifecycle with torch's
CUDA surface faked (tests/emu/fake_cuda.py)."""
import collections
import ctypes as C
import math
import os
import subprocess
import sys
import types

import numpy as np
import pytest

from openea_b200 import lib as L
from tests import attr2vec_oracle as ao
from tests import proje_oracle as po
from tests.emu import build_emu
from tests.test_emu_proje import HostTable, L_ERR, _aligned

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu():
    return build_emu.load()


NAMES = ("in", "w", "b")


def _case(seed, A, d):
    rng = np.random.default_rng(seed)
    sd = math.sqrt(1.3 * 2 / (A + d))
    tabs = {"in": rng.standard_normal((A, d)) * sd, "w": rng.standard_normal((A, d)) * sd,
            "b": rng.standard_normal((A, 1)) * 0.1}
    return rng, {k: v.astype(np.float32) for k, v in tabs.items()}


def _tables(tabs, norms):
    return {k: HostTable(v, norms.get(k, False)) for k, v in tabs.items()}


def _run(lib, tables, inputs, labels, sampled, num_tries, scale, ws_bytes=None, num_sampled=None, null=None):
    n = 0 if inputs is None else len(inputs)
    S = len(sampled) if num_sampled is None else num_sampled
    d, Cn = tables["in"].d, tables["w"].weight.shape[0]
    need = lib.oea_nce_workspace_bytes(n, max(1, S), d, Cn)
    raw, base = _aligned(need)
    m = L.Nce(*[C.pointer(tables[k].struct) for k in NAMES])
    out = np.zeros(1, dtype=np.float64)
    smp = np.ascontiguousarray(sampled, dtype=np.int32)
    nt = np.array([num_tries], dtype=np.int32)
    ii = None if inputs is None else np.ascontiguousarray(inputs, dtype=np.int32)
    ll = None if labels is None else np.ascontiguousarray(labels, dtype=np.int32)
    vp = lambda a: C.c_void_p(0 if a is None else a.ctypes.data)
    args = [vp(ii), vp(ll), n, vp(smp), vp(nt), S, scale, C.c_void_p(base), need if ws_bytes is None else ws_bytes, vp(out)]
    if null is not None:
        args[null] = C.c_void_p(0)
    rc = lib.oea_nce_score_fed(C.byref(m), *args, None)
    return rc, float(out[0])


def _check(tables, want_g, rtol=2e-4):
    for k, tab in tables.items():
        got, want = tab.grad[:, :tab.d], want_g[k].reshape(tab.grad.shape[0], -1)
        np.testing.assert_allclose(got, want, rtol=rtol, atol=1e-4 * max(1e-6, np.abs(want).max()), err_msg=k)
        assert not tab.grad[:, tab.d:].any(), "padding columns must stay zero"
        assert (np.abs(want).sum(1)[tab.touched == 0] == 0).all(), "untouched rows must have zero oracle gradient"


BOTH = {"in": True, "w": True}


def _compare(emu, d, n, A=60, S=12, seed=0, norms=BOTH, tweak=None, shortcut=False, scale=None):
    rng, tabs = _case(seed + 31 * d + n, A, d)
    inputs, labels = rng.integers(0, A, n), rng.integers(0, A, n)
    sampled, tries = po.sample_unique(seed + 11, A, S)
    if shortcut:
        tries = S
    if tweak is not None:
        inputs, labels = tweak(inputs, labels, sampled)
    scale = 1.0 / n if scale is None else scale
    want_loss, want_g = ao.fwd_bwd(tabs, norms, inputs, labels, sampled, tries, scale)
    tables = _tables(tabs, norms)
    rc, got = _run(emu, tables, inputs, labels, sampled, tries, scale)
    assert rc == 0
    assert got == pytest.approx(want_loss, rel=2e-5)
    _check(tables, want_g)


@pytest.mark.parametrize("d", [4, 10, 75, 100, 128])
def test_emulated_nce_step_matches_oracle_at_every_width(emu, d):
    _compare(emu, d, 37)


@pytest.mark.parametrize("n", [1, 2, 37, 500])
def test_emulated_nce_step_matches_oracle_at_every_batch(emu, n):
    """500 rows: four row tiles and sixteen splits of the batch on the emulator's grid."""
    _compare(emu, 20, n, S=40 if n == 500 else 12)


@pytest.mark.parametrize("S", [1, 2, 33, 60])
def test_emulated_nce_step_matches_oracle_for_sampled_sets_from_one_to_every_class(emu, S):
    _compare(emu, 12, 21, S=S, seed=S)


def test_emulated_nce_step_with_the_expected_count_shortcut(emu):
    _compare(emu, 20, 17, S=16, shortcut=True)


def test_emulated_nce_step_with_repeats_and_accidental_hits(emu):
    """Repeated inputs, repeated labels, labels inside the sampled set, an input equal to its label."""
    def tweak(inputs, labels, sampled):
        inputs, labels = inputs.copy(), labels.copy()
        labels[:6] = labels[0]
        labels[6:12] = sampled[:6]
        inputs[3:9] = inputs[3]
        inputs[12] = labels[12]
        return inputs, labels
    _compare(emu, 16, 29, S=20, tweak=tweak)


@pytest.mark.parametrize("norms", [{"in": True, "w": False}, {"in": False, "w": True}, {"in": False, "w": False}],
                         ids=["raw-classes", "raw-inputs", "both-raw"])
def test_emulated_nce_step_with_raw_tables(emu, norms):
    _compare(emu, 24, 19, S=15, norms=norms, scale=0.37)


def test_emulated_adagrad_steps_match_dense_tf_adagrad(emu):
    A, d, lr, n = 50, 20, 0.01, 23
    rng, tabs = _case(3, A, d)
    tables = _tables(tabs, BOTH)
    for t in tables.values():
        t.s1[:] = 0.1
        t.s1[:, t.d:] = 1.0
    st = ao.DenseState(dict(tabs), "Adagrad")
    for step in range(3):
        inputs, labels = rng.integers(0, A, n), rng.integers(0, A, n)
        sampled, tries = po.sample_unique(50 + step, A, 10)
        want = ao.step(st, BOTH, inputs, labels, sampled, tries, lr)
        rc, got = _run(emu, tables, inputs, labels, sampled, tries, 1.0 / n)
        assert rc == 0 and got == pytest.approx(want, rel=2e-5)
        cfg = L.OptCfg(L.OPT_ADAGRAD, lr, 0.9, 0.999, 1e-8, 1)
        for tab in tables.values():
            assert emu.oea_rowopt_apply(C.byref(tab.struct), C.byref(cfg), None) == 0
    for k, tab in tables.items():
        np.testing.assert_allclose(tab.weight[:, :tab.d], st.w[k].reshape(tab.weight.shape[0], -1), rtol=1e-4,
                                   atol=2e-6, err_msg=k)


def test_emulated_nce_argument_checks(emu):
    A, d, n = 30, 12, 6
    rng, tabs = _case(1, A, d)
    inputs, labels = rng.integers(0, A, n), rng.integers(0, A, n)
    sampled, tries = po.sample_unique(1, A, 8)
    tables = _tables(tabs, BOTH)
    run = lambda tabs_, **kw: _run(emu, tabs_, inputs, labels, sampled, tries, 1.0 / n, **kw)[0]
    need = emu.oea_nce_workspace_bytes(n, 8, d, A)
    assert need >= 4 * A and emu.oea_nce_workspace_bytes(n, 0, d, A) == 0
    assert run(tables, ws_bytes=need - 1) == L_ERR["WORKSPACE"]
    assert run(tables, num_sampled=0) == L_ERR["RANGE"]
    assert _run(emu, tables, inputs, labels, np.arange(A + 1), tries, 1.0)[0] == L_ERR["RANGE"]
    wide = {k: HostTable(np.zeros((A, 132 if k != "b" else 1), np.float32), k != "b") for k in NAMES}
    assert run(wide) == L_ERR["DIM"]                                                      # pitch 132 > 128
    assert run(dict(tables, w=HostTable(tabs["w"], True, pitch=16))) == L_ERR["DIM"]     # pitches disagree
    assert run(dict(tables, w=HostTable(tabs["w"][:, :8], True))) == L_ERR["DIM"]        # dims disagree
    assert run(dict(tables, b=HostTable(tabs["b"][:-1], False))) == L_ERR["SHAPE"]
    assert run(dict(tables, b=HostTable(np.zeros((A, 2)), False))) == L_ERR["SHAPE"]
    for slot in (0, 1, 3, 4, 9):                                                          # inputs, labels, sampled, tries, loss
        assert run(tables, null=slot) == L_ERR["NULL"], slot
    assert emu.oea_nce_score_fed(None, None, None, 0, None, None, 0, 1.0, None, 0, None, None) == L_ERR["NULL"]
    assert _run(emu, tables, None, None, sampled, tries, 1.0)[0] == 0                    # an empty batch is a no-op
    assert not any(t.grad.any() for t in tables.values())


# ---- the pair draw -------------------------------------------------------------------------------------------------
def _draw(lib, pairs, batch, seed, epoch, step, null=None):
    first, second = np.full(max(1, batch), -1, np.int32), np.full(max(1, batch), -1, np.int32)
    ptrs = [C.c_void_p(pairs.ctypes.data), C.c_void_p(first.ctypes.data), C.c_void_p(second.ctypes.data)]
    if null is not None:
        ptrs[null] = C.c_void_p(0)
    rc = lib.oea_pairs_draw(ptrs[0], len(pairs), batch, seed, epoch, step, ptrs[1], ptrs[2], None)
    return rc, first[:batch], second[:batch]


@pytest.mark.parametrize("n,batch", [(1, 1), (7, 7), (1000, 5), (1000, 999), (5000, 4096)])
def test_emulated_pair_draws_are_distinct_rows_and_a_function_of_the_key(emu, n, batch):
    pairs = np.stack([np.arange(n), np.arange(n) + 10 ** 6], axis=1).astype(np.int32)     # row r = (r, r + 10⁶)
    rc, a, b = _draw(emu, pairs, batch, 12345, 3, 17)
    assert rc == 0
    assert a.min() >= 0 and a.max() < n and np.array_equal(b, a + 10 ** 6)
    assert len(set(a.tolist())) == batch
    again = _draw(emu, pairs, batch, 12345, 3, 17)[1]
    assert np.array_equal(a, again)
    if batch < n:
        others = [_draw(emu, pairs, batch, *key)[1] for key in ((12346, 3, 17), (12345, 4, 17), (12345, 3, 18))]
        assert all(not np.array_equal(a, o) for o in others)


def test_emulated_pair_draw_argument_checks(emu):
    pairs = np.zeros((10, 2), np.int32)
    assert _draw(emu, pairs, 11, 0, 0, 0)[0] == L_ERR["RANGE"]
    assert _draw(emu, pairs, -1, 0, 0, 0)[0] == L_ERR["RANGE"]
    assert _draw(emu, pairs, 0, 0, 0, 0)[0] == 0
    for slot in range(3):
        assert _draw(emu, pairs, 4, 0, 0, 0, null=slot)[0] == L_ERR["NULL"]


# ---- training pairs and entity vectors against the reference's own functions -------------------------------------
def _reference_helpers():
    """get_kgs_popular_attributes, generate_training_data, get_ent_embeds_from_attributes of approaches/attr2vec.py."""
    import itertools
    import time
    from oracle import reference_source as ref_src
    from openea_b200.modules.utils.util import merge_dic
    preprocessing = types.SimpleNamespace(normalize=lambda m: m / np.maximum(np.linalg.norm(m, axis=1, keepdims=True),
                                                                                 np.finfo(m.dtype).tiny))
    row_stack = getattr(np, "row_stack", np.vstack)
    npx = types.SimpleNamespace(**{k: getattr(np, k) for k in dir(np) if not k.startswith("__")})
    npx.row_stack = row_stack
    return ref_src.extract("approaches/attr2vec.py", ["get_kg_popular_attributes", "get_kgs_popular_attributes",
                                                       "generate_training_data", "get_ent_embeds_from_attributes"],
                           {"np": npx, "itertools": itertools, "time": time, "merge_dic": merge_dic,
                            "preprocessing": preprocessing, "print": lambda *a, **k: None, "KG": object,
                            "KGs": object})


def _kgs(kind):
    from openea_b200.modules.load.kgs import read_kgs_from_folder
    from openea_b200.synth import write_dataset
    import tempfile
    folder = write_dataset(tempfile.mkdtemp() + "/%s/" % kind, kind)
    return read_kgs_from_folder(folder, "721_5fold/1/", "sharing", True)


def test_training_pairs_and_entity_vectors_equal_the_reference_source(cpu_engine_attr2vec):
    from openea_b200.approaches import attr2vec as a2v
    from openea_b200 import engine as eng
    from tests.helpers import ReferenceRecording
    ref = ReferenceRecording("reference_attr2vec", _reference_helpers)
    for kind, thresholds in (("micro", (0.9, 0.5, 1.0)), ("tiny", (0.9, 0.3))):
        kgs = _kgs(kind)
        for th in thresholds:
            want = ref("get_kgs_popular_attributes", kgs, th)
            assert tuple(set(x) for x in want) == a2v.get_kgs_popular_attributes(kgs, th)
            want_pairs = ref("generate_training_data", kgs, th)
            got = a2v.generate_training_data(kgs, th)
            canon = lambda ps: collections.Counter(tuple(sorted((int(a), int(b)))) for a, b in ps)
            assert canon(want_pairs) == canon(got.tolist()) and len(got) == len(want_pairs)
        rng = np.random.default_rng(7)
        attr = rng.standard_normal((kgs.attributes_num, 10)).astype(np.float32)
        selected = a2v.get_kgs_popular_attributes(kgs, 0.9)[2]
        table = eng.EmbeddingTable(attr, True, "Adagrad", "cpu")
        normed = table.lookup().numpy()
        want = ref("get_ent_embeds_from_attributes", kgs, normed, selected)
        from openea_b200 import gnn
        got = a2v.entity_vectors(table, gnn.DeviceCsr(a2v.mean_attribute_matrix(kgs, selected), "cpu")).numpy()
        assert got.shape == want.shape == (kgs.entities_num, 10)
        np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-6)
        assert (np.abs(want).sum(1) == 0).sum() == (np.abs(got).sum(1) == 0).sum()
    ref.save()


@pytest.fixture()
def cpu_engine_attr2vec(monkeypatch):
    build_emu.patch_engine(monkeypatch, build_emu.load())


# ---- configuration, guards and the lifecycle -----------------------------------------------------------------------
def test_attr2vec_preset_is_japes_configuration():
    from openea_b200 import presets
    for scale, batch in (("15K", 5000), ("100K", 20000)):
        a = presets.attr2vec(scale)
        assert a.embedding_module == "Attr2Vec" and a.batch_size == batch
        assert (a.dim, a.learning_rate, a.optimizer, a.attr_max_epoch, a.top_attr_threshold, a.eval_metric, a.csls) == \
            (100, 0.01, "Adagrad", 200, 0.9, "inner", 10)


def _model(monkeypatch, tmp_path, **over):
    from openea_b200 import engine as eng
    from openea_b200 import presets
    from openea_b200.approaches import Attr2Vec
    from openea_b200.modules.base import initializers
    from openea_b200.modules.load.kgs import read_kgs_from_folder
    from openea_b200.synth import write_dataset
    build_emu.patch_engine(monkeypatch, build_emu.load())
    monkeypatch.setattr(initializers, "_make", lambda values, norm, optimizer=None: eng.EmbeddingTable(
        values, bool(norm), optimizer or "Adagrad", "cpu"))
    folder = write_dataset(str(tmp_path) + "/micro/", "micro")
    args = presets.attr2vec("15K")
    args.training_data, args.output = folder, str(tmp_path) + "/out/"
    args.batch_size, args.attr_max_epoch, args.dim = 16, 2, 16
    for k, v in over.items():
        setattr(args, k, v)
    model = Attr2Vec()
    model.set_args(args)
    model.set_kgs(read_kgs_from_folder(folder, args.dataset_division, "sharing", args.ordered))
    return model


@pytest.mark.parametrize("over,msg", [(dict(top_attr_threshold=0.01), "fewer than 5"), (dict(dim=132), "dim <= 128")])
def test_attr2vec_guards(monkeypatch, tmp_path, over, msg):
    model = _model(monkeypatch, tmp_path, **over)
    with pytest.raises(ValueError, match=msg):
        model.init()


def test_attr2vec_rejects_several_ranks(monkeypatch, tmp_path):
    from openea_b200 import parallel as par
    model = _model(monkeypatch, tmp_path)
    monkeypatch.setattr(par, "world", lambda: (0, 2))
    with pytest.raises(NotImplementedError, match="Attr2Vec runs on one GPU"):
        model.init()


LIFECYCLE = r"""
import os, re, sys
sys.path.insert(0, {root!r})
from tests.emu import fake_cuda
fake_cuda.install()
from openea_b200 import presets
from openea_b200.approaches import Attr2Vec
from openea_b200.modules.load.kgs import read_kgs_from_folder
from openea_b200.synth import write_dataset
folder = {folder!r}
data = write_dataset(os.path.join(folder, "micro") + "/", "micro")
args = presets.attr2vec("15K")
args.training_data, args.output = data, os.path.join(folder, "out") + "/"
args.batch_size, args.attr_max_epoch, args.dim = 16, 3, 16
model = Attr2Vec()
model.set_args(args)
model.set_kgs(read_kgs_from_folder(data, args.dataset_division, "sharing", args.ordered))
model.init()
model.run()
print("valid", model.valid())
model.test()
model.save()
print("sim", model.eval_sim_mat().shape, model.eval_kg1_ent_embeddings().shape, model.eval_kg2_ent_embeddings().shape)
print("out", model.out_folder)
"""


def test_attr2vec_lifecycle_on_the_emulator(tmp_path):
    if build_emu.build() is None:
        pytest.skip("no CUDA headers for the emulator build")
    res = subprocess.run([sys.executable, "-c", LIFECYCLE.format(root=ROOT, folder=str(tmp_path))], capture_output=True,
                         text=True, timeout=900, cwd=ROOT)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-3000:]
    out = res.stdout
    import re
    losses = [float(x) for x in re.findall(r"epoch \d+, attribute loss: ([0-9.]+), cost time: [0-9.]+s", out)]
    assert len(losses) == 3 and all(np.isfinite(losses)) and losses[0] > 0
    for line in ("total attributes:", "selected attributes", "total selected attributes", "entity attribute dict",
                 "training data of attribute correlations", "get entity embeddings from attributes"):
        assert line in out, line
    assert re.search(r"valid [0-9.]+", out)
    assert "sim (" in out
    folder = re.search(r"^out (.+)$", out, re.M).group(1)
    attr = np.load(folder + "attr_embeds.npy")
    assert np.allclose(np.linalg.norm(attr, axis=1), 1.0, atol=1e-5)
    for name in ("alignment_results_12", "kg1_attr_ids", "kg1_attr_embeds_txt"):
        assert any(f.startswith(name) for f in os.listdir(folder)), name
