"""CPU: ConvE's configuration, its init guards, and set_args / set_kgs / init / run / save on the micro synthetic
dataset with the engine's entry points on the warp-emulator library of tests/emu."""
import os
import re

import numpy as np
import pytest
import torch

from openea_b200 import engine as eng
from openea_b200 import presets
from tests.emu import build_emu

SHIPPED = {  # run/args/conve_args_15K.json and conve_args_100K.json, the keys the engine reads
    "15K": dict(embedding_module="ConvE", alignment_module="sharing", dim=100, init="xavier", ent_l2_norm=True,
                rel_l2_norm=True, learning_rate=0.001, optimizer="Adam", max_epoch=2000, batch_size=500,
                dnn_neg_nums=4096, output_keep_prob=0.7, filter_num=32, batch_threads_num=2, test_threads_num=2,
                start_valid=100, eval_freq=10, stop_metric="hits1", eval_metric="inner", csls=10,
                top_k=[1, 5, 10, 50], eval_norm=True),
    "100K": dict(embedding_module="ConvE", alignment_module="sharing", dim=100, init="xavier", ent_l2_norm=True,
                 rel_l2_norm=True, learning_rate=0.001, optimizer="Adam", max_epoch=2000, batch_size=5000,
                 dnn_neg_nums=4096, output_keep_prob=0.7, filter_num=32, batch_threads_num=3, test_threads_num=10,
                 start_valid=300, eval_freq=10, stop_metric="hits1", eval_metric="inner", csls=10,
                 top_k=[1, 5, 10, 50], eval_norm=True),
}


@pytest.mark.parametrize("scale", ["15K", "100K"])
def test_conve_preset_is_the_shipped_configuration(scale):
    a = presets.conve(scale)
    for k, v in SHIPPED[scale].items():
        assert getattr(a, k) == v, k


@pytest.mark.parametrize("d,xy", [(100, (10, 10)), (75, (5, 15)), (12, (4, 3)), (10, (2, 5)), (7, (1, 7)),
                                  (97, (1, 97)), (128, (8, 16))])
def test_dim_factorization(d, xy):
    from openea_b200.models.neural.conve import dim_factorization
    assert dim_factorization(d) == xy


@pytest.fixture()
def conve_engine(monkeypatch):
    build_emu.patch_engine(monkeypatch, build_emu.load())
    return eng


def _model(cpu_engine, monkeypatch, tmp_path, **over):
    from openea_b200.models.neural import ConvE
    from openea_b200.models.neural import proje as pj
    from openea_b200.modules.base import initializers
    from openea_b200.modules.load.kgs import read_kgs_from_folder
    from openea_b200.synth import write_dataset
    monkeypatch.setattr(initializers, "_make", lambda values, norm, optimizer=None: cpu_engine.EmbeddingTable(
        values, bool(norm), optimizer or "Adagrad", "cpu"))
    monkeypatch.setattr(pj, "load_session", lambda: None)
    folder = write_dataset(str(tmp_path) + "/micro/", "micro")
    args = presets.conve("15K")
    args.training_data, args.output = folder, str(tmp_path) + "/out/"
    args.batch_size, args.max_epoch, args.start_valid, args.dim, args.dnn_neg_nums = 64, 3, 1000, 12, 8
    args.filter_num, args.learning_rate = 3, 0.01
    for k, v in over.items():
        setattr(args, k, v)
    kgs = read_kgs_from_folder(folder, args.dataset_division, "sharing", args.ordered)
    model = ConvE()
    model.set_args(args)
    model.set_kgs(kgs)
    return model


def test_conve_lifecycle_on_the_emulator(conve_engine, monkeypatch, tmp_path, capsys):
    model = _model(conve_engine, monkeypatch, tmp_path)
    model.init()
    assert model.proje_params is None
    assert tuple(model.conv.raw().shape) == (3, 12) and tuple(model.bn_in.raw().shape) == (2, 3)
    assert tuple(model.fc_w.raw().shape) == (72, 12) and tuple(model.fc_out.raw().shape) == (3, 12)
    assert (model.conv.raw()[:, 10] == 1).all() and not model.conv.raw()[:, [9, 11]].any()
    assert float(model.conv.raw()[:, :9].abs().max()) <= (6 / 36) ** 0.5
    names = ("ent_embeds", "rel_embeds", "entity_w", "entity_b", "conv", "bn_in", "fc_w", "fc_out")
    assert set(names) == set(model._checkpoint_tables())
    before = {k: getattr(model, k).weight.clone() for k in names}
    model.run()
    model.save()
    out = capsys.readouterr().out
    losses = [float(x) for x in re.findall(r"avg\. triple loss: (-?[0-9.]+)", out)]
    assert len(losses) == 3 and all(np.isfinite(losses)) and "Training ends" in out
    for k, w in before.items():
        now = getattr(model, k).weight
        assert torch.isfinite(now).all() and not torch.equal(w, now), k
    assert os.path.exists(model.out_folder + "ent_embeds.npy")


@pytest.mark.parametrize("over,msg", [(dict(optimizer="Adagrad"), "ConvE needs optimizer 'Adam'"),
                                      (dict(dnn_neg_nums=1), "dnn_neg_nums"), (dict(init="normal"), "xavier"),
                                      (dict(dnn_neg_nums=10 ** 6), "range is too small"),
                                      (dict(alignment_module="mapping"), "sharing"),
                                      (dict(eval_metric="L2"), "inner"), (dict(rel_l2_norm=False), "rel_l2_norm"),
                                      (dict(output_keep_prob=0.0), "output_keep_prob"),
                                      (dict(output_keep_prob=1.5), "output_keep_prob"),
                                      (dict(filter_num=0), "filter_num"), (dict(dim=132), "dim <= 128")])
def test_conve_guards(conve_engine, monkeypatch, tmp_path, over, msg):
    model = _model(conve_engine, monkeypatch, tmp_path, **over)
    with pytest.raises(ValueError, match=msg):
        model.init()


def test_conve_runs_on_one_gpu(conve_engine, monkeypatch, tmp_path):
    from openea_b200 import parallel as par
    model = _model(conve_engine, monkeypatch, tmp_path)
    monkeypatch.setattr(par, "world", lambda: (0, 2))
    with pytest.raises(NotImplementedError, match="ConvE runs on one GPU"):
        model.init()
