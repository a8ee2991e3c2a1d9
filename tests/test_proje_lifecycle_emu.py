"""CPU: ProjE's configuration and initialisation, and set_args / set_kgs / init / run / save on the micro synthetic
dataset with the engine's entry points on the warp-emulator library of tests/emu/build_emu_proje.py (in-process, as
tests/test_jape.py runs JAPE)."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch

from openea_b200 import engine as eng
from openea_b200 import lib as L
from openea_b200 import presets
from tests.emu import build_emu_proje

SHIPPED = {  # run/args/proje_args_15K.json and proje_args_100K.json, the keys the engine reads
    "15K": dict(embedding_module="ProjE", alignment_module="sharing", dim=100, init="xavier", ent_l2_norm=True,
                rel_l2_norm=True, learning_rate=0.001, optimizer="Adam", max_epoch=2000, batch_size=500,
                dnn_neg_nums=4096, batch_threads_num=2, test_threads_num=2, start_valid=100, eval_freq=10,
                stop_metric="hits1", eval_metric="inner", csls=10, top_k=[1, 5, 10, 50], eval_norm=True),
    "100K": dict(embedding_module="ProjE", alignment_module="sharing", dim=100, init="xavier", ent_l2_norm=True,
                 rel_l2_norm=True, learning_rate=0.001, optimizer="Adam", max_epoch=2000, batch_size=5000,
                 dnn_neg_nums=4096, batch_threads_num=3, test_threads_num=10, start_valid=300, eval_freq=10,
                 stop_metric="hits1", eval_metric="inner", csls=10, top_k=[1, 5, 10, 50], eval_norm=True),
}


@pytest.mark.parametrize("scale", ["15K", "100K"])
def test_proje_preset_is_the_shipped_configuration(scale):
    a = presets.proje(scale)
    for k, v in SHIPPED[scale].items():
        assert getattr(a, k) == v, k


def test_xavier_on_a_one_dimensional_shape():
    """entity_b = init_embeddings([E], 'xavier'): fan_in = fan_out = E, σ = sqrt(1.3/E), truncated at 2σ."""
    from openea_b200.modules.base import initializers
    n = 20000
    initializers.set_seed(5)
    v = initializers.init_values([n], "xavier")
    sigma = math.sqrt(1.3 / n)
    assert tuple(v.shape) == (n,)
    assert float(v.std()) == pytest.approx(0.8796 * sigma, rel=0.03)        # a normal truncated at ±2σ
    assert float(v.abs().max()) <= 2 * sigma + 1e-7


@pytest.fixture()
def proje_engine(monkeypatch):
    so = build_emu_proje.build()
    if so is None:
        pytest.skip("no CUDA headers for the emulator build")
    lib = C.CDLL(so)
    for name, (res, args) in L.SIGNATURES.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    monkeypatch.setattr(L, "load", lambda: lib)
    monkeypatch.setattr(eng, "_stream_ptr", lambda: C.c_void_p(0))
    return eng


def _model(cpu_engine, monkeypatch, tmp_path, **over):
    from openea_b200.models.neural import ProjE
    from openea_b200.models.neural import proje as pj
    from openea_b200.modules.base import initializers
    from openea_b200.modules.load.kgs import read_kgs_from_folder
    from openea_b200.synth import write_dataset
    monkeypatch.setattr(initializers, "_make", lambda values, norm, optimizer=None: cpu_engine.EmbeddingTable(
        values, bool(norm), optimizer or "Adagrad", "cpu"))
    monkeypatch.setattr(pj, "load_session", lambda: None)
    folder = write_dataset(str(tmp_path) + "/micro/", "micro")
    args = presets.proje("15K")
    args.training_data, args.output = folder, str(tmp_path) + "/out/"
    # validation and test rank on the GPU's similarity kernels: the emulated run trains and saves
    args.batch_size, args.max_epoch, args.start_valid, args.dim, args.dnn_neg_nums = 64, 3, 1000, 16, 8
    args.learning_rate = 0.01
    for k, v in over.items():
        setattr(args, k, v)
    kgs = read_kgs_from_folder(folder, args.dataset_division, "sharing", args.ordered)
    model = ProjE()
    model.set_args(args)
    model.set_kgs(kgs)
    return model


def test_proje_lifecycle_on_the_emulator(proje_engine, monkeypatch, tmp_path, capsys):
    model = _model(proje_engine, monkeypatch, tmp_path)
    model.init()
    assert tuple(model.entity_b.weight.shape) == (model.kgs.entities_num, 4) and model.entity_b.dim == 1
    assert tuple(model.proje_params.raw().shape) == (4, 16) and not model.proje_params.raw()[2:].any()
    before = {k: getattr(model, k).weight.clone() for k in ("ent_embeds", "rel_embeds", "entity_w", "entity_b", "proje_params")}
    model.run()
    model.save()
    out = capsys.readouterr().out
    losses = [float(x) for x in re.findall(r"avg\. triple loss: (-?[0-9.]+)", out)]
    assert len(losses) == 3 and all(np.isfinite(losses)) and "Training ends" in out
    for k, w in before.items():
        now = getattr(model, k).weight
        assert torch.isfinite(now).all() and not torch.equal(w, now), k
    assert os.path.exists(model.out_folder + "ent_embeds.npy")


@pytest.mark.parametrize("over,msg", [(dict(optimizer="Adagrad"), "Adam"), (dict(dnn_neg_nums=1), "dnn_neg_nums"),
                                      (dict(dnn_neg_nums=10 ** 6), "range is too small"), (dict(init="normal"), "xavier")])
def test_proje_guards(proje_engine, monkeypatch, tmp_path, over, msg):
    model = _model(proje_engine, monkeypatch, tmp_path, **over)
    with pytest.raises(ValueError, match=msg):
        model.init()
