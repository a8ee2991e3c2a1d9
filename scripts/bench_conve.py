"""Times ConvE's step at the shipped shapes — 15K: B = 500, E = 30 000; 100K: B = 5 000, E = 200 000; both S = 4 096,
d = 100, F = 32, keep_prob 0.7 — with CUDA events over many steps and an L2 flush before each: the device sampler,
oea_conve_score_fed (the convolution tower and the NCE head), Adam on the eight tables, and the whole step.  A separate
torch.profiler run splits oea_conve_score_fed into the tower's kernels and the head's.  Prints the card and its power
limit, and the dense layer's three GEMMs' FLOP rate against the FP32 data-sheet bound.  Needs a GPU.

    python scripts/bench_conve.py [--steps 100] [--shapes 15K,100K]
"""
import argparse
import json
import math
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openea_b200 import engine as eng  # noqa: E402
from scripts.bench_proje import SHAPES, card  # noqa: E402

# the head's dX and dW kernels also run the dense layer's forward and dW: their template argument tells them apart
HEAD = ("k_nce_logq", "k_nce_logits", "k_nce_dx<oea::GatheredW>", "k_nce_dw<oea::GatheredW>", "k_nce_true")
FC = ("k_nce_dx<oea::StagedW>", "k_nce_dw<oea::StagedW>", "k_conve_fc_dx")
TOWER = FC + ("k_conve_conv_fwd", "k_conve_fc_out", "k_conve_fc_out_bwd", "k_conve_conv_dw", "k_conve_conv_dx")


def run_shape(name, steps, S=4096, d=100, F=32, keep=0.7):
    B, E, R = SHAPES[name]
    rng = np.random.default_rng(0)
    K, y = 2 * F * d, 10
    xav = lambda rows, cols: (rng.standard_normal((rows, cols)) * math.sqrt(2.6 / (rows + cols))).astype(np.float32)
    conv = np.concatenate([rng.uniform(-0.14, 0.14, (F, 9)), np.zeros((F, 1)), np.ones((F, 1)), np.zeros((F, 1))], 1)
    tabs = (eng.EmbeddingTable(xav(E, d), True, "Adam"), eng.EmbeddingTable(xav(R, d), True, "Adam"),
            eng.EmbeddingTable(xav(E, d), False, "Adam"), eng.EmbeddingTable(xav(E, 1), False, "Adam"),
            eng.EmbeddingTable(conv.astype(np.float32), False, "Adam"),
            eng.EmbeddingTable(np.stack([np.ones(y), np.zeros(y)]).astype(np.float32), False, "Adam"),
            eng.EmbeddingTable(rng.uniform(-0.03, 0.03, (K, d)).astype(np.float32), False, "Adam"),
            eng.EmbeddingTable(np.stack([np.zeros(d), np.ones(d), np.zeros(d)]).astype(np.float32), False, "Adam"))
    tr = eng.ConvETrainer(tabs, S, 0.001, keep)
    data = [torch.from_numpy(np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)])
                             .astype(np.int32)).cuda() for _ in range(8)]
    flush = torch.empty(128 << 20, dtype=torch.uint8, device="cuda")       # larger than the 50 MB L2
    for i in range(5):                                                      # warm-up: modules, workspace
        tr.sample(i)
        tr.score_fed(data[i % len(data)], dropout_seed=i)
        tr.apply()
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

    t_sample = timed(lambda i: tr.sample(1000 + i))
    t_score = timed(lambda i: tr.score_fed(data[i % len(data)], dropout_seed=i))
    t_adam = timed(lambda i: tr.apply())
    t_step = timed(lambda i: (tr.sample(2000 + i), tr.score_fed(data[i % len(data)], dropout_seed=i), tr.apply()))
    tr.read_loss()
    # per-kernel device times in a separate run (tracing slows the host; the times above are taken without it)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(20):
            tr.sample(3000 + i)
            tr.score_fed(data[i % len(data)], dropout_seed=i)
            tr.apply()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        # whole names (followed by their argument list or template arguments): k_conve_fc_out is a prefix of
        # k_conve_fc_out_bwd
        key = next((k for k in TOWER + HEAD + ("k_logu_sample",) if k + "(" in ev.key or k + "<" in ev.key), None)
        if key:
            per[key] = per.get(key, 0.0) + ev.device_time_total / 20.0       # µs per step
    head_us = sum(per.get(k, 0.0) for k in HEAD)
    tower_us = sum(per.get(k, 0.0) for k in TOWER)
    fc_us = sum(per.get(k, 0.0) for k in FC)
    fc_flop = 3 * 2.0 * B * K * d
    return {"shape": name, "batch": B, "entities": E, "num_sampled": S, "dim": d, "filters": F, "steps": steps,
            "workspace_mb": round(tr._workspace(B).numel() / 1e6, 1),
            "sampler_ms": round(t_sample, 4), "score_fed_ms": round(t_score, 4), "adam_ms": round(t_adam, 4),
            "step_ms": round(t_step, 4), "profiled_tower_us": round(tower_us, 1), "profiled_head_us": round(head_us, 1),
            "profiled_kernels_us": {k: round(v, 1) for k, v in sorted(per.items())},
            "fc_gflop": round(fc_flop / 1e9, 3),
            "fc_tflops": round(fc_flop / (fc_us * 1e-6) / 1e12, 2) if fc_us else None,
            "fc_fp32_datasheet_floor_us": round(fc_flop / 67e12 * 1e6, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--shapes", default="15K,100K")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_conve needs a GPU")
    c = card()
    for name in a.shapes.split(","):
        print(json.dumps(dict(card=c, **run_shape(name, a.steps))))


if __name__ == "__main__":
    main()
