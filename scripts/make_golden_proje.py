"""Generates tests/golden/path_i_proje.npz by EXECUTING the reference's own graph code for ProjE
(models/neural/proje.py) — `_define_variables`, `_define_embed_graph` and two
`session.run([triple_loss, triple_optimizer], feed_dict)` per case — on oracle/tf1_shim.py with the ops of
scripts/tf1_shim_proje.py installed.  All arithmetic is float64.  Every run records its feeds, the sampled ids and
num_tries the candidate sampler drew, and its loss; every case its start and final variables under their scoped names.
Runs only where the reference exists; the fixture it writes is what travels.

    python scripts/make_golden_proje.py                   # writes the golden
    python scripts/make_golden_proje.py --check-existing  # the other path (i) goldens, regenerated with the extension
                                                          # installed, compared array by array with the committed files
"""
import importlib
import json
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.dont_write_bytecode = True          # never write into the reference tree
import make_golden_path_i as base  # noqa: E402
import tf1_shim_proje as ext  # noqa: E402
from oracle import tf1_shim as tf  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "path_i_proje.npz")
N_REL = 6


def _shipped(**kw):
    # run/args/proje_args_15K.json (lr 0.001, Adam, xavier, both tables normalised), at a golden's size
    a = dict(dim=12, init="xavier", alignment_module="sharing", optimizer="Adam", eval_metric="inner",
             ent_l2_norm=True, rel_l2_norm=True, learning_rate=0.001, dnn_neg_nums=12)
    a.update(kw)
    return a


def _uniform(rng, n_ent, n):
    return np.stack([rng.integers(0, n_ent, n), rng.integers(0, N_REL, n), rng.integers(0, n_ent, n)]).astype(np.int32)


def _repeats(rng, n_ent, n):
    """Repeated tails, repeated heads, and tails that a sampled set of a third of the classes very likely holds
    (the low ids carry most of the log-uniform mass)."""
    pos = _uniform(rng, n_ent, n)
    pos[2, :5] = pos[2, 0]
    pos[2, 5:12] = np.arange(7)
    pos[0, 3:9] = pos[0, 3]
    return pos


# case → (args, entities, positives per run, batch maker)
CASES = {
    "proje": (_shipped(), 40, 16, _uniform),
    "proje_d75": (_shipped(dim=75, dnn_neg_nums=64, learning_rate=0.01), 300, 37, _uniform),
    "proje_repeats": (_shipped(dnn_neg_nums=14, learning_rate=0.01), 40, 21, _repeats),
    "proje_one_positive": (_shipped(learning_rate=0.01), 40, 1, _uniform),
}


def generate():
    out, meta = {}, {}
    ext.install(tf)
    for case, (args, n_ent, n_pos, batch) in CASES.items():
        tf.reset_default_graph()
        mod = base.import_reference("openea.models.neural.proje")
        model = mod.ProjE()
        model.args = types.SimpleNamespace(**args)
        model.kgs = types.SimpleNamespace(entities_num=n_ent, relations_num=N_REL)
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
            start = (rng.standard_normal(shape) * 2.0 / np.sqrt(shape[-1])).astype(np.float32).astype(np.float64)
            v.assign_numpy(start)
            out["%s/var0/%s" % (case, name)] = start
        for i in range(2):
            pos = batch(rng, n_ent, n_pos)
            feed = {"pos_hs": pos[0], "pos_rs": pos[1], "pos_ts": pos[2]}
            loss, _ = session.run([model.triple_loss, model.triple_optimizer],
                                  feed_dict={getattr(model, k): v for k, v in feed.items()})
            assert len(ext.SAMPLED) == i + 1, "one sampler draw per session.run"
            sampled, tries = ext.SAMPLED[i]
            out["%s/run%d/loss" % (case, i)] = np.float64(loss)
            out["%s/run%d/sampled" % (case, i)] = sampled
            out["%s/run%d/num_tries" % (case, i)] = np.int32(tries)
            for k, v in feed.items():
                out["%s/run%d/feed/%s" % (case, i, k)] = v
            if batch is _repeats:
                assert np.isin(pos[2], sampled).any(), "the case must hold a tail inside the sampled set"
        for v, name in zip(variables, names):
            out["%s/var_final/%s" % (case, name)] = v.value.detach().numpy().copy()
        meta[case] = {"class": "openea.models.neural.proje.ProjE", "args": args, "entities": n_ent,
                      "relations": N_REL, "defines": defines, "variables": names}
        print("%-20s %s  losses %s" % (case, names, ["%.6g" % float(out["%s/run%d/loss" % (case, i)]) for i in range(2)]))
    out["meta"] = np.frombuffer(json.dumps(meta, sort_keys=True).encode(), dtype=np.uint8)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


def check_existing():
    """Regenerate the committed path (i) goldens of make_golden_path_i.py, make_golden_semantic_ext.py and
    make_golden_transr.py with the extension installed, into a temporary directory, and compare them array by array."""
    ext.install(tf)
    ok = True
    with tempfile.TemporaryDirectory() as tmp:
        for script, entry in (("make_golden_path_i", ("generate",)),
                              ("make_golden_semantic_ext", ("generate",)), ("make_golden_transr", ("generate",))):
            m = importlib.import_module(script)
            outs = [n for n in vars(m) if n.startswith("OUT")]
            committed = {n: getattr(m, n) for n in outs}
            for n in outs:
                setattr(m, n, os.path.join(tmp, os.path.basename(committed[n])))
            for fn in entry:
                if hasattr(m, fn):
                    getattr(m, fn)()
            for n in outs:
                new, old = np.load(getattr(m, n)), np.load(committed[n])
                same = set(new.files) == set(old.files) and all(np.array_equal(new[k], old[k]) for k in old.files)
                print("%-40s %s" % (os.path.basename(committed[n]), "identical" if same else "DIFFERS"))
                ok = ok and same
    return ok


if __name__ == "__main__":
    if not os.path.isdir(base.REF_SRC):
        sys.exit("the reference is not present: goldens can only be generated where it exists")
    if "--check-existing" in sys.argv:
        sys.exit(0 if check_existing() else 1)
    generate()
