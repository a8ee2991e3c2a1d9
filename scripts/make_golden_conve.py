"""Generates tests/golden/path_i_conve.npz by EXECUTING the reference's own graph code for ConvE
(models/neural/conve.py) — `_define_variables`, `_define_embed_graph` and two
`session.run([triple_loss, triple_optimizer], feed_dict)` per case — on oracle/tf1_shim.py with the ops of
scripts/tf1_shim_proje.py and scripts/tf1_shim_conve.py installed.  All arithmetic is float64.  Every run records its
feeds, the sampled ids and num_tries the candidate sampler drew, the dropout seed and both dropout masks, and its loss;
every case its start and final variables under their scoped names.  Runs only where the reference exists; the fixture
it writes is what travels.

    python scripts/make_golden_conve.py                   # writes the golden
    python scripts/make_golden_conve.py --check-existing  # the other path (i) goldens regenerated with and without both
                                                          # extensions installed, compared array by array
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
import tf1_shim_conve as cext  # noqa: E402
import tf1_shim_proje as ext  # noqa: E402
from oracle import tf1_shim as tf  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "path_i_conve.npz")
N_REL = 6


def _shipped(**kw):
    # run/args/conve_args_15K.json (lr 0.001, Adam, xavier, both tables normalised, keep 0.7), at a golden's size
    a = dict(dim=12, init="xavier", alignment_module="sharing", optimizer="Adam", eval_metric="inner",
             ent_l2_norm=True, rel_l2_norm=True, learning_rate=0.001, dnn_neg_nums=12, output_keep_prob=0.7,
             filter_num=4)
    a.update(kw)
    return a


def _uniform(rng, n_ent, n):
    return np.stack([rng.integers(0, n_ent, n), rng.integers(0, N_REL, n), rng.integers(0, n_ent, n)]).astype(np.int32)


# case → (args, entities, positives per run)
CASES = {
    "conve": (_shipped(), 40, 16),                                                  # 4 × 3 image, keep 0.7
    "conve_prime": (_shipped(dim=7, output_keep_prob=1.0, learning_rate=0.01), 40, 9),   # d = 7: a 1 × 7 image
    "conve_d10": (_shipped(dim=10, filter_num=3, output_keep_prob=0.5, learning_rate=0.01), 40, 11),   # 2 × 5
    "conve_every_class": (_shipped(dnn_neg_nums=16, learning_rate=0.01), 16, 13),  # S = E
}


def generate():
    out, meta = {}, {}
    ext.install(tf)
    cext.install(tf)
    for case, (args, n_ent, n_pos) in CASES.items():
        tf.reset_default_graph()
        mod = base.import_reference("openea.models.neural.conve")
        model = mod.ConvE()
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
            if "batch_normalization" in name and name.endswith("gamma"):
                start = 1.0 + 0.2 * start                   # gammas near their initial 1
            v.assign_numpy(start)
            out["%s/var0/%s" % (case, name)] = start
        for i in range(2):
            pos = _uniform(rng, n_ent, n_pos)
            feed = {"pos_hs": pos[0], "pos_rs": pos[1], "pos_ts": pos[2]}
            tf.dropout_new_run()
            loss, _ = session.run([model.triple_loss, model.triple_optimizer],
                                  feed_dict={getattr(model, k): v for k, v in feed.items()})
            assert len(ext.SAMPLED) == i + 1, "one sampler draw per session.run"
            sampled, tries = ext.SAMPLED[i]
            dseed, masks = cext.DROPOUT[i]
            assert len(masks) == (2 if args["output_keep_prob"] < 1 else 0), "two dropout calls per session.run"
            out["%s/run%d/loss" % (case, i)] = np.float64(loss)
            out["%s/run%d/sampled" % (case, i)] = sampled
            out["%s/run%d/num_tries" % (case, i)] = np.int32(tries)
            out["%s/run%d/dropout_seed" % (case, i)] = np.uint64(dseed)
            for j, m in enumerate(masks):
                out["%s/run%d/mask%d" % (case, i, j)] = m.reshape(n_pos, -1)
            for k, v in feed.items():
                out["%s/run%d/feed/%s" % (case, i, k)] = v
        for v, name in zip(variables, names):
            out["%s/var_final/%s" % (case, name)] = v.value.detach().numpy().copy()
        meta[case] = {"class": "openea.models.neural.conve.ConvE", "args": args, "entities": n_ent,
                      "relations": N_REL, "defines": defines, "variables": names}
        print("%-20s %s  losses %s" % (case, names, ["%.6g" % float(out["%s/run%d/loss" % (case, i)]) for i in range(2)]))
    out["meta"] = np.frombuffer(json.dumps(meta, sort_keys=True).encode(), dtype=np.uint8)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


GENERATORS = ("make_golden_path_i", "make_golden_semantic_ext", "make_golden_transr", "make_golden_proje",
              "make_golden_attr2vec")


def regenerate(into, with_extensions):
    """Regenerate every other path (i) golden into the directory `into`, with or without both extensions installed."""
    if with_extensions:
        ext.install(tf)
        cext.install(tf)
    for script in GENERATORS:
        m = importlib.import_module(script)
        for n in [n for n in vars(m) if n.startswith("OUT")]:
            setattr(m, n, os.path.join(into, os.path.basename(getattr(m, n))))
        m.generate()


def check_existing():
    """The other path (i) goldens regenerated in two fresh processes, once on the plain shim and once with both
    extensions installed, must be equal array by array: installing the extensions changes nothing they compute.  Each
    is also compared with its committed file (the largest relative difference is printed: a different torch or NumPy
    build may move the last bits of the committed float64 values)."""
    import subprocess
    ok = True
    with tempfile.TemporaryDirectory() as tmp:
        dirs = {flag: os.path.join(tmp, flag or "plain") for flag in ("", "--with-extensions")}
        for flag, d in dirs.items():
            os.makedirs(d)
            cmd = [sys.executable, os.path.abspath(__file__), "--regenerate-into", d] + ([flag] if flag else [])
            subprocess.run(cmd, check=True, stdout=subprocess.DEVNULL)
        for name in sorted(os.listdir(dirs[""])):
            plain, withx = np.load(os.path.join(dirs[""], name)), np.load(os.path.join(dirs["--with-extensions"], name))
            same = set(plain.files) == set(withx.files) and all(np.array_equal(plain[k], withx[k]) for k in plain.files)
            old = np.load(os.path.join(ROOT, "tests", "golden", name))
            dev = max((float(np.max(np.abs(plain[k] - old[k]) / np.maximum(np.abs(old[k]), 1e-300)))
                       for k in old.files if old[k].dtype.kind == "f" and old[k].size), default=0.0)
            print("%-32s %s; largest relative difference from the committed file %.1e"
                  % (name, "identical with the extensions" if same else "DIFFERS with the extensions", dev))
            ok = ok and same
    return ok


if __name__ == "__main__":
    if not os.path.isdir(base.REF_SRC):
        sys.exit("the reference is not present: goldens can only be generated where it exists")
    if "--regenerate-into" in sys.argv:
        regenerate(sys.argv[sys.argv.index("--regenerate-into") + 1], "--with-extensions" in sys.argv)
        sys.exit(0)
    if "--check-existing" in sys.argv:
        sys.exit(0 if check_existing() else 1)
    generate()
