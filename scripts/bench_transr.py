"""Times TransR's fed step at the 15K shape (5 000 positives + 5 000 uniform negatives, ≈ 450 relations with Zipf
frequencies, d = 100, the shipped margin loss and Adagrad): oea_transr_score_fed alone, and the whole step (score + the
three row optimisers), with CUDA events over many steps and an L2 flush before each.  Prints the card, its power limit,
the times and the FLOP rate on the roofline of DESIGN §4 (12·d² FLOP per scored triple).  Needs a GPU.

    python scripts/bench_transr.py [--steps 200] [--dim 100]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openea_b200 import engine as eng  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def batches(rng, n_ent, n_rel, n_pos, count):
    p = 1.0 / np.arange(1, n_rel + 1) ** 1.1
    out = []
    for _ in range(count):
        rel = rng.choice(n_rel, size=n_pos, p=p / p.sum())
        pos = np.stack([rng.integers(0, n_ent, n_pos), rel, rng.integers(0, n_ent, n_pos)]).astype(np.int32)
        neg = pos.copy()
        side = rng.random(n_pos) < 0.5
        neg[0, side] = rng.integers(0, n_ent, int(side.sum()))
        neg[2, ~side] = rng.integers(0, n_ent, int((~side).sum()))
        out.append((torch.from_numpy(pos).cuda(), torch.from_numpy(neg).cuda()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--dim", type=int, default=100)
    ap.add_argument("--n-pos", type=int, default=5000)
    ap.add_argument("--profile", default=None, help="also write per-kernel device times (torch.profiler) to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_transr needs a GPU")
    d, n_ent, n_rel = a.dim, 30000, 450
    rng = np.random.default_rng(0)
    ent = eng.EmbeddingTable(rng.standard_normal((n_ent, d)).astype(np.float32) / np.sqrt(d), True, "Adagrad", "cuda")
    rel = eng.EmbeddingTable(rng.standard_normal((n_rel, d)).astype(np.float32) / np.sqrt(d), True, "Adagrad", "cuda")
    mat = eng.EmbeddingTable(rng.standard_normal((n_rel * d, d)).astype(np.float32) / d, False, "Adagrad", "cuda")
    tr = eng.ModelTrainer("TransR", (ent, rel, None, mat), eng.loss_cfg("margin-based", "L2", margin=1.5), 0.01)
    data = batches(rng, n_ent, n_rel, a.n_pos, 16)
    flush = torch.empty(128 << 20, dtype=torch.uint8, device="cuda")       # larger than the 50 MB L2
    for i in range(10):                                                     # warm-up: modules, workspace
        tr.score_fed(*data[i % len(data)])
        tr.apply()
    torch.cuda.synchronize()

    def timed(step):
        total = 0.0
        for i in range(a.steps):
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            step(data[i % len(data)])
            e.record()
            e.synchronize()
            total += s.elapsed_time(e)
        return total / a.steps

    t_score = timed(lambda b: tr.score_fed(*b))
    for tab in (ent, rel, mat):                                           # leave the tables between steps clean
        tab.apply(0.0)
    t_step = timed(lambda b: (tr.score_fed(*b), tr.apply()))
    n = 2 * a.n_pos
    flop = 12.0 * d * d * n
    if a.profile:                     # a separate run: tracing slows the host, the times above are taken without it
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(50):
                tr.score_fed(*data[i % len(data)])
                tr.apply()
            torch.cuda.synchronize()
        with open(a.profile, "w") as f:
            f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=20))
    print(json.dumps({"card": card(), "dim": d, "scored_triples": n, "relations": n_rel, "steps": a.steps,
                      "score_ms": round(t_score, 4), "step_ms": round(t_step, 4),
                      "score_tflops": round(flop / (t_score * 1e-3) / 1e12, 2),
                      "fp32_datasheet_bound_us": round(flop / 67e12 * 1e6, 1)}))


if __name__ == "__main__":
    main()
