"""Times Attr2Vec on the synthetic 15K and 100K datasets (openea_b200/synth.py; 800 attributes, presets.attr2vec: d = 100,
batch 5 000 / 20 000, S = len(selected) // 5) — one training step with CUDA events over many steps and an L2 flush
before each (the pair draw, the sampler, oea_nce_score_fed, Adagrad on the three tables), whole training epochs of
Attr2Vec (launch_training_1epo, the epoch loop of run()) and, apart, run()'s one-off host build of the pairs — and, on
the same data and the same GPU, the training epochs of JAPE's torch auxiliary (jape.attribute_similarity, its one-off
set-up measured by a run of zero epochs and subtracted) as the comparison point.  A separate torch.profiler run splits the step into its kernels.  Prints the card and its power limit.
Needs a GPU.

    python scripts/bench_attr2vec.py [--steps 200] [--epochs 5] [--shapes 15K,100K]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openea_b200 import presets  # noqa: E402
from openea_b200.approaches import Attr2Vec  # noqa: E402
from openea_b200.approaches import jape  # noqa: E402
from openea_b200.modules.load.kgs import read_kgs_from_folder  # noqa: E402
from openea_b200.synth import write_dataset  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def run_shape(name, steps, epochs, root):
    folder = write_dataset(os.path.join(root, name) + "/", name)
    args = presets.attr2vec(name)
    args.training_data, args.output = folder, os.path.join(root, "out") + "/"
    kgs = read_kgs_from_folder(folder, args.dataset_division, args.alignment_module, args.ordered)
    model = Attr2Vec()
    model.set_args(args)
    model.set_kgs(kgs)
    model.init()
    from openea_b200.approaches.attr2vec import PAIR_THRESHOLD, generate_training_data
    pairs = generate_training_data(kgs, PAIR_THRESHOLD)
    tr, B = model.trainer, args.batch_size
    tr.set_pairs(pairs)
    flush = torch.empty(128 << 20, dtype=torch.uint8, device="cuda")       # larger than the 50 MB L2
    for i in range(10):                                                     # warm-up: modules, workspace
        tr.step(B, 1, 0, i)
    torch.cuda.synchronize()

    def timed(fn):
        total = 0.0
        for i in range(steps):
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn(i)
            e.record()
            e.synchronize()
            total += s.elapsed_time(e)
        return total / steps

    inputs, labels = tr.draw(B, 1, 0, 0)
    t_draw = timed(lambda i: tr.draw(B, 1, 1, i))
    t_sample = timed(lambda i: tr.sample(1000 + i))
    t_score = timed(lambda i: tr.score_fed(inputs, labels))
    t_opt = timed(lambda i: tr.apply())
    t_step = timed(lambda i: tr.step(B, 1, 2, i))
    tr.read_loss()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(20):
            tr.step(B, 1, 3, i)
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        if ev.device_time_total > 0 and not ev.key.startswith("Memset") and not ev.key.startswith("Memcpy"):
            k = ev.key.split("(")[0].split("<")[0].replace("void ", "").replace("oea::", "")
            per[k] = per.get(k, 0.0) + ev.device_time_total / 20.0         # µs per step
    S, d = tr.num_sampled, args.dim
    head_flop = 3 * 2.0 * B * S * d

    # whole epochs of run(), without its one-off host build of the pairs (timed on its own)
    t0 = time.perf_counter()
    generate_training_data(kgs, PAIR_THRESHOLD)
    t_pairs = time.perf_counter() - t0
    steps_per_epoch = len(pairs) // B
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for epoch in range(1, epochs + 1):
        model.launch_training_1epo(epoch, steps_per_epoch)
    torch.cuda.synchronize()
    t_run = (time.perf_counter() - t0) / epochs

    def torch_aux(n_epochs):
        t0 = time.perf_counter()
        jape.attribute_similarity(kgs, args, torch.device("cuda"), epochs=n_epochs)
        torch.cuda.synchronize()
        return time.perf_counter() - t0
    t_torch_setup = torch_aux(0)
    t_torch = (torch_aux(epochs) - t_torch_setup) / epochs
    return {"shape": name, "attributes": kgs.attributes_num, "pairs": int(len(pairs)), "batch": B, "num_sampled": S,
            "dim": d, "steps_per_epoch": int(len(pairs) // B), "timed_steps": steps,
            "pair_draw_ms": round(t_draw, 4), "sampler_ms": round(t_sample, 4), "nce_score_fed_ms": round(t_score, 4),
            "adagrad_ms": round(t_opt, 4), "step_ms": round(t_step, 4),
            "profiled_kernels_us": {k: round(v, 1) for k, v in sorted(per.items())},
            "head_gflop": round(head_flop / 1e9, 3), "head_fp32_datasheet_floor_us": round(head_flop / 67e12 * 1e6, 2),
            "pair_build_s": round(t_pairs, 4), "run_epoch_s": round(t_run, 4),
            "torch_auxiliary_epoch_s": round(t_torch, 4), "torch_auxiliary_setup_s": round(t_torch_setup, 4),
            "epochs_timed": epochs}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--shapes", default="15K,100K")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_attr2vec needs a GPU")
    c = card()
    with tempfile.TemporaryDirectory() as root:
        for name in a.shapes.split(","):
            print(json.dumps(dict(card=c, **run_shape(name, a.steps, a.epochs, root))), flush=True)


if __name__ == "__main__":
    main()
