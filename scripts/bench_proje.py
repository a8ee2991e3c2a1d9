"""Times ProjE's step at the shipped shapes — 15K: B = 500, E = 30 000; 100K: B = 5 000, E = 200 000; both S = 4 096,
d = 100 — with CUDA events over many steps and an L2 flush before each: the device sampler, oea_proje_score_fed (the
projection layer and the NCE head), Adam on the five tables, and the whole step.  A separate torch.profiler run splits
oea_proje_score_fed into the projection layer's kernels and the head's.  Prints the card and its power limit, the head's
FLOP rate against the FP32 data-sheet bound and Adam's bytes against HBM.  Needs a GPU.

    python scripts/bench_proje.py [--steps 100] [--shapes 15K,100K]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openea_b200 import engine as eng  # noqa: E402

SHAPES = {"15K": (500, 30000, 1000), "100K": (5000, 200000, 1500)}     # (batch, entities, relations)
HEAD = ("k_nce_logits", "k_nce_dx", "k_nce_dw", "k_nce_true")
PROJ = ("k_proje_gather", "k_proje_columns_fwd", "k_proje_columns_bwd", "k_proje_push")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def run_shape(name, steps, S=4096, d=100):
    B, E, R = SHAPES[name]
    rng = np.random.default_rng(0)
    xav = lambda rows, cols: (rng.standard_normal((rows, cols)) * math.sqrt(2.6 / (rows + cols))).astype(np.float32)
    tabs = (eng.EmbeddingTable(xav(E, d), True, "Adam"), eng.EmbeddingTable(xav(R, d), True, "Adam"),
            eng.EmbeddingTable(xav(E, d), False, "Adam"), eng.EmbeddingTable(xav(E, 1), False, "Adam"),
            eng.EmbeddingTable(rng.uniform(-0.17, 0.17, (4, d)).astype(np.float32), False, "Adam"))
    tr = eng.ProjETrainer(tabs, S, 0.001)
    data = [torch.from_numpy(np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)])
                             .astype(np.int32)).cuda() for _ in range(8)]
    flush = torch.empty(128 << 20, dtype=torch.uint8, device="cuda")       # larger than the 50 MB L2
    for i in range(5):                                                      # warm-up: modules, workspace
        tr.sample(i)
        tr.score_fed(data[i % len(data)])
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
    t_score = timed(lambda i: tr.score_fed(data[i % len(data)]))
    t_adam = timed(lambda i: tr.apply())
    t_step = timed(lambda i: (tr.sample(2000 + i), tr.score_fed(data[i % len(data)]), tr.apply()))
    tr.read_loss()
    # per-kernel device times in a separate run (tracing slows the host; the times above are taken without it)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(20):
            tr.sample(3000 + i)
            tr.score_fed(data[i % len(data)])
            tr.apply()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        key = next((k for k in HEAD + PROJ + ("k_logu_sample",) if k in ev.key), None)
        if key:
            per[key] = per.get(key, 0.0) + ev.device_time_total / 20.0       # µs per step
    head_us = sum(per.get(k, 0.0) for k in HEAD)
    proj_us = sum(per.get(k, 0.0) for k in PROJ)
    head_flop = 3 * 2.0 * B * S * d
    # dense Adam reads weight, grad, m, v and writes weight, m, v (and zeroes grad): 8 passes of 4 bytes per element
    adam_bytes = 8 * 4.0 * sum(t.rows * t.pitch for t in tabs)
    return {"shape": name, "batch": B, "entities": E, "num_sampled": S, "dim": d, "steps": steps,
            "sampler_ms": round(t_sample, 4), "score_fed_ms": round(t_score, 4), "adam_ms": round(t_adam, 4),
            "step_ms": round(t_step, 4), "profiled_projection_us": round(proj_us, 1), "profiled_head_us": round(head_us, 1),
            "profiled_kernels_us": {k: round(v, 1) for k, v in sorted(per.items())},
            "head_gflop": round(head_flop / 1e9, 3),
            "head_tflops": round(head_flop / (head_us * 1e-6) / 1e12, 2) if head_us else None,
            "head_fp32_datasheet_floor_us": round(head_flop / 67e12 * 1e6, 1),
            "adam_mb": round(adam_bytes / 1e6, 1), "adam_tb_per_s": round(adam_bytes / (t_adam * 1e-3) / 1e12, 2),
            "adam_hbm_floor_us": round(adam_bytes / 3.35e12 * 1e6, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--shapes", default="15K,100K")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_proje needs a GPU")
    c = card()
    for name in a.shapes.split(","):
        print(json.dumps(dict(card=c, **run_shape(name, a.steps))))


if __name__ == "__main__":
    main()
