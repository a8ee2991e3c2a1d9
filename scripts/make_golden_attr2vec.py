"""Generates tests/golden/path_i_attr2vec.npz by EXECUTING the reference's own graph code for Attr2Vec
(approaches/attr2vec.py) — `_define_variables`, `_define_embed_graph` and two `session.run([loss, optimizer],
feed_dict)` per case, feeding `train_labels` (the [B, 1] reshape the reference feeds, not its placeholder) — on
oracle/tf1_shim.py with the ops of scripts/tf1_shim_proje.py installed (variable scopes, the unique log-uniform
candidate sampler, nce_loss).  All arithmetic is float64.  Every run records its feeds, the sampled ids and num_tries
the sampler drew, and its loss; every case its start and final variables under their scoped names.  Runs only where
the reference exists; the fixture it writes is what travels.

    python scripts/make_golden_attr2vec.py                   # writes the golden
    python scripts/make_golden_attr2vec.py --check-existing  # the other path (i) goldens, regenerated with the
                                                             # extension installed, compared with the committed files
"""
import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.dont_write_bytecode = True          # never write into the reference tree
import make_golden_path_i as base  # noqa: E402
import make_golden_proje  # noqa: E402
import tf1_shim_proje as ext  # noqa: E402
from oracle import tf1_shim as tf  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "path_i_attr2vec.npz")


def _uniform(rng, n_attr, batch):
    return rng.integers(0, n_attr, batch).astype(np.int32), rng.integers(0, n_attr, batch).astype(np.int32)


def _repeats(rng, n_attr, batch):
    """Repeated inputs, repeated labels, labels among the low ids a sampled set very likely holds, and an input that is
    its own label."""
    inputs, labels = _uniform(rng, n_attr, batch)
    labels[:5] = labels[0]
    labels[5:11] = np.arange(6)
    inputs[2:8] = inputs[2]
    inputs[12] = labels[12]
    return inputs, labels


# case → (dim, learning rate, attributes, num_sampled, batch, batch maker).  The shipped configuration is JAPE's JSON
# (d = 100, lr 0.01, Adagrad) at a golden's size; num_sampled = S = A draws every class.
CASES = {
    "attr2vec": (100, 0.01, 40, 8, 16, _uniform),
    "attr2vec_all_classes": (24, 0.05, 20, 20, 12, _uniform),
    "attr2vec_repeats": (32, 0.05, 40, 14, 21, _repeats),
    "attr2vec_d10": (10, 0.05, 60, 12, 9, _uniform),
}


def generate():
    out, meta = {}, {}
    ext.install(tf)
    for case, (dim, lr, n_attr, num_sampled, batch_size, batch) in CASES.items():
        tf.reset_default_graph()
        mod = base.import_reference("openea.approaches.attr2vec")
        model = mod.Attr2Vec()
        model.args = types.SimpleNamespace(dim=dim, learning_rate=lr, batch_size=batch_size)
        model.kgs = types.SimpleNamespace(attributes_num=n_attr)
        model.num_sampled_negs = num_sampled
        defines = ["_define_variables", "_define_embed_graph"]
        for name in defines:
            getattr(model, name)()
        session = tf.Session()
        rng = np.random.default_rng(sum(map(ord, case)))
        variables = tf.trainable_variables()
        names = [getattr(v, "scoped_name", v.name) for v in variables]
        assert len(set(names)) == len(names), names
        for v, name in zip(variables, names):
            shape = tuple(v.value.shape)
            scale = 0.1 if len(shape) == 1 else 2.0 / np.sqrt(shape[-1])
            start = (rng.standard_normal(shape) * scale).astype(np.float32).astype(np.float64)
            v.assign_numpy(start)
            out["%s/var0/%s" % (case, name)] = start
        for i in range(2):
            inputs, labels = batch(rng, n_attr, batch_size)
            loss, _ = session.run([model.loss, model.optimizer],
                                  feed_dict={model.train_inputs: inputs, model.train_labels: labels.reshape(-1, 1)})
            assert len(ext.SAMPLED) == i + 1, "one sampler draw per session.run"
            sampled, tries = ext.SAMPLED[i]
            out["%s/run%d/loss" % (case, i)] = np.float64(loss)
            out["%s/run%d/sampled" % (case, i)] = sampled
            out["%s/run%d/num_tries" % (case, i)] = np.int32(tries)
            out["%s/run%d/feed/inputs" % (case, i)] = inputs
            out["%s/run%d/feed/labels" % (case, i)] = labels
            if batch is _repeats:
                assert np.isin(labels, sampled).any(), "the case must hold a label inside the sampled set"
        for v, name in zip(variables, names):
            out["%s/var_final/%s" % (case, name)] = v.value.detach().numpy().copy()
        meta[case] = {"class": "openea.approaches.attr2vec.Attr2Vec", "dim": dim, "learning_rate": lr,
                      "attributes": n_attr, "num_sampled": num_sampled, "batch_size": batch_size, "defines": defines,
                      "variables": names}
        print("%-22s %s  losses %s" % (case, names, ["%.6g" % float(out["%s/run%d/loss" % (case, i)]) for i in range(2)]))
    out["meta"] = np.frombuffer(json.dumps(meta, sort_keys=True).encode(), dtype=np.uint8)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    if not os.path.isdir(base.REF_SRC):
        sys.exit("the reference is not present: goldens can only be generated where it exists")
    if "--check-existing" in sys.argv:
        sys.exit(0 if make_golden_proje.check_existing() else 1)
    generate()
