"""Generates tests/golden/path_i_semantic_ext.npz by EXECUTING the reference's own graph code for RotatE
(models/semantic/rotate.py), HolE (models/semantic/hole.py) and BootEA_RotatE (approaches/bootea_rotate.py) —
`_define_variables`, `_define_embed_graph`, `_define_alignment_graph` and `session.run([loss, optimizer], feed_dict)` —
on oracle/tf1_shim.py, as scripts/make_golden_path_i.py does for the other path (i) models.  The ops these two graphs
need beyond the shim's (cos, sin, norm, the FFT, conj, real, the complex cast) are added to the shim here, from the
TF 1.x op definitions, before the reference is imported.  All arithmetic is float64, the FFT's complex64 included.
Runs only where the reference exists; the fixture it writes is what travels.

    python scripts/make_golden_semantic_ext.py
"""
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.dont_write_bytecode = True          # never write into the reference tree
import make_golden_path_i as base  # noqa: E402
from oracle import tf1_shim as tf  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "path_i_semantic_ext.npz")

# case → (module, class, args overrides, graph-definition calls, runs); a run is (kind, number of negatives per positive)
CASES = {
    "rotate": ("openea.models.semantic.rotate", "RotatE",
               dict(init="uniform", optimizer="Adam", gamma=12.0, neg_triple_num=3, learning_rate=0.01),
               ["_define_variables", "_define_embed_graph"], [("triple", 3), ("triple", 3), ("triple", 3)]),
    "hole_k1": ("openea.models.semantic.hole", "HolE", dict(init="xavier", margin=0.2, neg_triple_num=1),
                ["_define_variables", "_define_embed_graph"], [("triple", 1), ("triple", 1)]),
    "hole_k3": ("openea.models.semantic.hole", "HolE", dict(init="xavier", margin=0.3, neg_triple_num=3),
                ["_define_variables", "_define_embed_graph"], [("triple", 3), ("triple", 3)]),
    "bootea_rotate": ("openea.approaches.bootea_rotate", "BootEA_RotatE",
                      dict(init="normal", optimizer="Adam", gamma=12.0, neg_triple_num=3, rel_l2_norm=False,
                           learning_rate=0.01),
                      ["_define_variables", "_define_embed_graph", "_define_alignment_graph"],
                      [("triple", 3), ("align", 0), ("triple", 3)]),
}


def extend_shim():
    """tf.cos / sin / norm / fft / ifft / conj / real and the complex cast, float64 (complex128) throughout."""
    def unary(f, name):
        return lambda x, name_=None, **kw: tf.Tensor(f, (tf._wrap(x),), name)
    tf.cos, tf.sin = unary(torch.cos, "cos"), unary(torch.sin, "sin")
    tf.conj, tf.real = unary(torch.conj, "conj"), unary(torch.real, "real")
    tf.fft, tf.ifft = unary(torch.fft.fft, "fft"), unary(torch.fft.ifft, "ifft")      # innermost axis, as tf.fft
    tf.complex64, tf.complex128 = "complex64", "complex128"
    real_cast = tf.cast

    def cast(x, dtype=None, name=None):
        if dtype in ("complex64", "complex128"):
            return tf.Tensor(lambda a: a.to(torch.complex128), (tf._wrap(x),), "cast")
        return real_cast(x, dtype, name)
    tf.cast = cast

    def norm(tensor, ord="euclidean", axis=None, keepdims=None, name=None, keep_dims=None):
        """tf.norm, Euclidean: sqrt(reduce_sum(x²)) over `axis` (all elements when None)."""
        keep = bool(keepdims or keep_dims)
        return tf.Tensor(lambda a: torch.sqrt((a * a).sum() if axis is None else (a * a).sum(dim=axis, keepdim=keep)),
                         (tf._wrap(tensor),), "norm")
    tf.norm = norm


def generate():
    extend_shim()
    out, meta = {}, {}
    for case, (module, cls, overrides, defines, runs) in CASES.items():
        tf.reset_default_graph()
        mod = base.import_reference(module)
        args = dict(base.BASE)
        args.update(overrides)
        model = getattr(mod, cls)()
        model.args = types.SimpleNamespace(**args)
        model.kgs = types.SimpleNamespace(entities_num=base.N_ENT, relations_num=base.N_REL)
        if hasattr(model, "epsilon"):            # what init() sets before the graph definition (rotate.py:37)
            model.embedding_range = (args["gamma"] + model.epsilon) / args["dim"]
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
        meta[case] = {"class": module + "." + cls, "args": args, "defines": defines, "runs": run_meta, "variables": names}
        print("%-16s %s  losses %s" % (case, names, ["%.6g" % float(out["%s/run%d/loss" % (case, i)]) for i in range(len(runs))]))
    out["meta"] = np.frombuffer(json.dumps(meta, sort_keys=True).encode(), dtype=np.uint8)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    if not os.path.isdir(base.REF_SRC):
        sys.exit("the reference is not present: goldens can only be generated where it exists")
    generate()
