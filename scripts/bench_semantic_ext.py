"""Device-timed launches of the RotatE and HolE scorers (oea_model_score_fed, OEA_MODEL_ROTATE / OEA_MODEL_HOLE) at the
shipped 15K / 100K batch shapes (rotate_args / hole_args: 5000 / 20000 positives, k = 10 for RotatE, 1 for HolE,
d = 100): kernel time from CUDA events on the launching stream (L2 flushed between launches), algorithmic bytes per
scored triple (rows read + gradient rows reduced) · pitch · 4 — RotatE 5 + 5, HolE 3 + 3 — and, for HolE's O(d²)
correlation, FLOP/s against the FP32 peak.  Prints one JSON line per case, the GPU's name and power limit first.

    python scripts/bench_semantic_ext.py [out.jsonl]
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openea_b200 import engine as eng  # noqa: E402

HBM_PEAK_GBS = 3350.0          # H100 SXM data sheet
FP32_PEAK_TFLOPS = 67.0        # H100 SXM data sheet, dense FP32 (an FMA counts 2)
ROWS = {"RotatE": 10, "HolE": 6}


def hole_flops(d, n_pos, k):
    """Executed FLOPs of k_hole_margin when every pair is active: forward 2d² per triple (the correlation), backward 6d²
    per triple (correlation again, ∂ĥ, ∂t̂), plus one more forward of each negative before its backward."""
    return n_pos * (1 + k) * 8 * d * d + n_pos * k * 2 * d * d


def device_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def main(out_path=None):
    if not torch.cuda.is_available():
        raise SystemExit("bench_semantic_ext needs a GPU")
    info = dict(device=torch.cuda.get_device_name(0), nvidia_smi=device_info())
    print(json.dumps(info), flush=True)
    lines = [info]
    flush = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")
    d = 100
    for shape, n_ent, n_rel, B in (("15K", 30000, 450, 5000), ("100K", 200000, 600, 20000)):
        for model, k in (("RotatE", 10), ("HolE", 1)):
            rng = np.random.default_rng(0)
            mk = lambda rows: eng.EmbeddingTable((rng.standard_normal((rows, d)) / 10).astype(np.float32), True)
            if model == "RotatE":
                tabs = (mk(n_ent), mk(n_rel), mk(n_ent))
                tr = eng.ModelTrainer("RotatE", tabs, eng.loss_cfg("logistic", "L2"), 0.1, gamma=12.0, neg_weight=1.0 / k)
            else:
                tabs = (mk(n_ent), mk(n_rel))
                tr = eng.ModelTrainer("HolE", tabs, eng.loss_cfg("margin-based", "L2", margin=0.2), 0.01)
            pos = torch.from_numpy(np.stack([rng.integers(0, n_ent, B), rng.integers(0, n_rel, B),
                                             rng.integers(0, n_ent, B)]).astype(np.int32)).cuda()
            neg = pos.repeat_interleave(k, dim=1).clone()
            side = torch.from_numpy(rng.random(B * k) < 0.5).cuda()
            repl = torch.from_numpy(rng.integers(0, n_ent, B * k).astype(np.int32)).cuda()
            neg[0] = torch.where(side, repl, neg[0])
            neg[2] = torch.where(side, neg[2], repl)
            times = []
            for it in range(23):
                flush.fill_(it & 1)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                tr.score_fed(pos, neg)
                e1.record()
                torch.cuda.synchronize()
                if it >= 3:
                    times.append(e0.elapsed_time(e1))
                loss = tr.read_loss()
                for t in tr.live:
                    t.grad.zero_()
                    t.touched.zero_()
            ms = float(np.median(times))
            triples = B * (1 + k)
            nbytes = ROWS[model] * tabs[0].pitch * 4 * triples
            row = dict(shape=shape, model=model, d=d, n_pos=B, k=k, ms=ms, ms_min=float(np.min(times)),
                       ms_max=float(np.max(times)), scored_triples_per_s=triples / ms * 1e3,
                       algorithmic_gb=nbytes / 1e9, algorithmic_gbs=nbytes / ms / 1e6,
                       frac_of_hbm_peak=nbytes / ms / 1e6 / HBM_PEAK_GBS, loss=loss)
            if model == "RotatE":
                row["launches"] = 2          # positives and negatives at their own weights
            else:
                fl = hole_flops(d, B, k)
                row.update(flops_if_all_active=fl, tflops=fl / ms / 1e9, frac_of_fp32_peak=fl / ms / 1e9 / FP32_PEAK_TFLOPS)
                t_mem, t_fl = nbytes / (HBM_PEAK_GBS * 1e9), fl / (FP32_PEAK_TFLOPS * 1e12)
                row["roofline_bound"] = "fp32" if t_fl > t_mem else "hbm"
            print(json.dumps(row), flush=True)
            lines.append(row)
    if out_path:
        with open(out_path, "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")
    return lines


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
