#!/usr/bin/env python
"""Generates tests/golden/hits_aligne_15k_oracle.json: the CPU ORACLE's end-to-end accuracy on the synthetic 15K KG.

The oracle loop (oracle/train_loop.py) is the reference's own Python sampler (modules/train/batch.py imported from
/root/reference) + the C restatement of the dense TF step + the NumPy evaluation of modules/finding; AlignE/BootEA triple
training configuration of run/args/bootea_args_15K.json (dim 100, batch 5000, 10 negatives, limited loss, ε = 0.9 truncated
sampling refreshed every 10 epochs, Adagrad 0.01).  Run HERE (CPU container, several minutes per seed); the GPU-side test
(tests/test_hits_parity_gpu.py) trains the engine on the same KG for the same epochs and compares mean ± σ over seeds.

    python scripts/make_hits_golden.py [--epochs 100] [--seeds 1 2 3 4] [--threads 2]
"""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ProcessPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
EVAL_AT = (10, 20, 50, 100)


def one_seed(job):
    seed, epochs, threads = job
    import numpy as np
    from oracle import train_loop as tl, triple as orc
    from openea_b200.synth import synth_id_arrays
    orc.set_num_threads(threads)
    arr = dict(synth_id_arrays("15K"))
    # The reference trains its FIRST epoch on the triple lists in load order (they are shuffled only after every epoch,
    # models/basic_model.py:234-235) — on the real datasets that is Python-set order, i.e. effectively random, but
    # synth_id_arrays emits np.unique-SORTED triples: an epoch of batches with contiguous head ids inflates Adagrad's
    # accumulators early and leaves the run several epochs behind for good.  The oracle therefore starts from a seeded random order, as real data would.
    prng = np.random.default_rng(1000 + seed)
    arr["triples1"] = arr["triples1"][prng.permutation(len(arr["triples1"]))]
    arr["triples2"] = arr["triples2"][prng.permutation(len(arr["triples2"]))]
    curve, losses = {}, []

    def on_epoch(epoch, st):
        if epoch in EVAL_AT or epoch == epochs:
            hits, mr, mrr = tl.test_hits(st, arr)
            chits, cmr, cmrr = tl.test_hits(st, arr, csls_k=10)
            curve[str(epoch)] = {"hits": hits, "mr": mr, "mrr": mrr, "csls_hits": chits, "csls_mrr": cmrr}
    t0 = time.time()
    tl.train_triples(arr, 100, 5000, 10, epochs, truncated_eps=0.9, seed=seed,
                     log=lambda s: losses.append(float(s.split(":")[-1])), on_epoch=on_epoch)
    return {"seed": seed, "curve": curve, "loss": losses, "seconds": time.time() - t0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=100)
    ap.add_argument("--seeds", type=int, nargs="+", default=[1, 2, 3, 4])
    ap.add_argument("--threads", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "hits_aligne_15k_oracle.json"))
    args = ap.parse_args()
    from oracle import ref_adapter
    with ProcessPoolExecutor(max_workers=len(args.seeds)) as pool:
        runs = list(pool.map(one_seed, [(s, args.epochs, args.threads) for s in args.seeds]))
    out = {"what": "CPU oracle (reference sampler + dense TF-style step), AlignE/BootEA triple training on synth_id_arrays('15K'), triple lists in a seeded random initial order",
           "sampler": "reference modules/train/batch.py" if ref_adapter.available() else "behavioural port",
           "config": {"dim": 100, "batch": 5000, "neg": 10, "loss": "limited(0.01, 2.0, 0.2)", "lr": 0.01, "eps": 0.9,
                      "truncated_freq": 10, "epochs": args.epochs, "top_k": [1, 5, 10, 50]},
           "runs": runs}
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
