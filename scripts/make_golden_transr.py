"""Generates tests/golden/path_i_transr.npz by EXECUTING the reference's own graph code for TransR
(models/trans/transr.py) — `_define_variables`, `_define_embed_graph` and `session.run([triple_loss, triple_optimizer],
feed_dict)` — on oracle/tf1_shim.py, as scripts/make_golden_path_i.py does for the other path (i) models.  The shim needs
no op beyond its own.  All arithmetic is float64.  Runs only where the reference exists; the fixture it writes is what
travels.

    python scripts/make_golden_transr.py
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
from oracle import tf1_shim as tf  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "path_i_transr.npz")

# case → (args overrides, runs); a run is (kind, number of negatives per positive)
CASES = {
    # run/args/transr_args_15K.json: margin-based, L2, Adagrad, one negative
    "transr": (dict(loss="margin-based", loss_norm="L2", optimizer="Adagrad", neg_triple_num=1, margin=1.5),
               [("triple", 1), ("triple", 1)]),
    "transr_limited_adam": (dict(loss="limited", loss_norm="L2", optimizer="Adam", neg_triple_num=3),
                            [("triple", 3), ("triple", 3)]),
    "transr_logistic_l1_sgd": (dict(loss="logistic", loss_norm="L1", optimizer="SGD", neg_triple_num=3, learning_rate=0.1),
                               [("triple", 3), ("triple", 3)]),
    "transr_raw_entities": (dict(loss="margin-based", loss_norm="L2", optimizer="Adagrad", neg_triple_num=1,
                                 ent_l2_norm=False), [("triple", 1), ("triple", 1)]),
    "transr_d10": (dict(loss="margin-based", loss_norm="L2", optimizer="Adagrad", neg_triple_num=1, dim=10),
                   [("triple", 1), ("triple", 1)]),
}


def generate():
    out, meta = {}, {}
    for case, (overrides, runs) in CASES.items():
        tf.reset_default_graph()
        mod = base.import_reference("openea.models.trans.transr")
        args = dict(base.BASE)
        args.update(overrides)
        model = mod.TransR()
        model.args = types.SimpleNamespace(**args)
        model.kgs = types.SimpleNamespace(entities_num=base.N_ENT, relations_num=base.N_REL)
        defines = ["_define_variables", "_define_embed_graph"]
        for name in defines:
            getattr(model, name)()
        session = tf.Session()
        rng = np.random.default_rng(sum(map(ord, case)))
        variables = tf.trainable_variables()
        names = [v.name for v in variables]
        assert len(set(names)) == len(names), names
        for v in variables:
            shape = tuple(v.value.shape)
            start = (rng.standard_normal(shape) * 2.0 / np.sqrt(shape[1])).astype(np.float32).astype(np.float64)
            v.assign_numpy(start)
            out["%s/var0/%s" % (case, v.name)] = start
        run_meta = []
        for i, (kind, k) in enumerate(runs):
            fetch, feed = base.make_run(kind, k, rng, model)
            loss, _ = session.run([getattr(model, fetch[0]), getattr(model, fetch[1])],
                                  feed_dict={getattr(model, key): val for key, val in feed.items()})
            out["%s/run%d/loss" % (case, i)] = np.float64(loss)
            for key, val in feed.items():
                out["%s/run%d/feed/%s" % (case, i, key)] = val
            run_meta.append({"kind": kind, "k": k, "fetch": list(fetch)})
        for v in variables:
            out["%s/var_final/%s" % (case, v.name)] = v.value.detach().numpy().copy()
        meta[case] = {"class": "openea.models.trans.transr.TransR", "args": args, "defines": defines, "runs": run_meta,
                      "variables": names}
        print("%-24s %s  losses %s" % (case, names, ["%.6g" % float(out["%s/run%d/loss" % (case, i)]) for i in range(len(runs))]))
    out["meta"] = np.frombuffer(json.dumps(meta, sort_keys=True).encode(), dtype=np.uint8)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    if not os.path.isdir(base.REF_SRC):
        sys.exit("the reference is not present: goldens can only be generated where it exists")
    generate()
