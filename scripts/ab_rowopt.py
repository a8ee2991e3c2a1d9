#!/usr/bin/env python
"""A/B of the one-launch step's row optimiser against a previous commit, on the bench.

    build (no GPU needed):  python scripts/ab_rowopt.py build [REV]     REV defaults to HEAD; use the parent of the change
    run (on the GPU):       python scripts/ab_rowopt.py run [RUNS] [OUT_DIR]
                            RUNS (default 5) bench runs per library; OUT_DIR (default: a new temporary directory)

`build` extracts REV's sources with `git archive` into a temporary directory, builds its liboea.so there and copies it
to openea_b200/_lib/ab_parent/ (git-ignored).  `run` alternates `bench.py --no-cpu-baseline` between that library
(OEA_LIB_PATH) and the tree's own, times TripleTrainer.apply() (k_rowopt_pair) after a real 100K sampled score with L2
flushed, compares table digests after a seeded apply() and a fed step without reordered atomics (`bitwise`),
and compares `bench.py --dump-outputs` (parent twice, new once) at both workloads.  Results go to
OUT_DIR/ab_rowopt.json and a table to OUT_DIR/ab_rowopt.txt, with the card's name, power limit and max SM clock."""
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PARENT_DIR = os.path.join(ROOT, "openea_b200", "_lib", "ab_parent")
PARENT_LIB = os.path.join(PARENT_DIR, "liboea.so")
FIELDS = [("value", lambda d: d["value"]), ("ms_per_step", lambda d: d["ms_per_step"]),
          ("kernel_ms_median", lambda d: d["roofline"]["kernel_ms_median"]),
          ("score_alone_ms_median", lambda d: d["roofline"]["score_kernel_alone"]["ms_median"]),
          ("optimiser_phase_ms", lambda d: d["roofline"]["kernel_ms_median"] - d["roofline"]["score_kernel_alone"]["ms_median"]),
          ("touched_rows_per_step", lambda d: d["roofline"]["touched_rows_per_step"]),
          ("bootea_15k.value", lambda d: d["bootea_15k"]["value"]), ("e2e.value", lambda d: d["e2e"]["value"])]


def build(rev="HEAD"):
    sha = subprocess.check_output(["git", "-C", ROOT, "rev-parse", rev], text=True).strip()
    with tempfile.TemporaryDirectory() as tmp:
        archive = subprocess.run(["git", "-C", ROOT, "archive", sha], check=True, capture_output=True).stdout
        subprocess.run(["tar", "-x", "-C", tmp], input=archive, check=True)
        lib = subprocess.check_output([sys.executable, "-c", "from openea_b200 import build; print(build.build_cuda())"],
                                      cwd=tmp, text=True).strip().splitlines()[-1]
        os.makedirs(PARENT_DIR, exist_ok=True)
        shutil.copy(lib, PARENT_LIB)
    with open(os.path.join(PARENT_DIR, "REV"), "w") as f:
        f.write(sha + "\n")
    print("parent %s -> %s" % (sha, PARENT_LIB))


def _env(arm):
    e = dict(os.environ)
    e.pop("OEA_LIB_PATH", None)
    if arm == "parent":
        e["OEA_LIB_PATH"] = PARENT_LIB
    return e


def _bench(arm, extra=()):
    res = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--no-cpu-baseline"] + list(extra),
                         capture_output=True, text=True, env=_env(arm), timeout=1200)
    if res.returncode != 0:
        raise RuntimeError("bench.py (%s) failed: %s" % (arm, res.stderr[-2000:]))
    return json.loads(res.stdout.strip().splitlines()[-1])


def apply_timing(reps=40):
    """Device time of TripleTrainer.apply() (k_rowopt_pair) after a real sampled score at the 100K shape, L2 flushed
    before each score."""
    import torch
    sys.path.insert(0, ROOT)
    import bench
    W = bench.build_workload("bootea_100k", 0, torch.device("cuda:0"))
    tr, cfg = W["trainer"], W["cfg"]
    flush = torch.empty(bench.L2_FLUSH_BYTES // 4, dtype=torch.float32, device="cuda")
    ms = []
    for i in range(8 + reps):
        flush.fill_(float(i))
        tr.score_sampled(W["kg1"], W["kg2"], W["tset"], cfg["batch"], cfg["k"], i, 0xAB + i)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        tr.apply()
        b.record()
        torch.cuda.synchronize()
        if i >= 8:
            ms.append(a.elapsed_time(b))
    print(json.dumps({"apply_ms_median": float(np.median(ms)), "apply_ms_min": float(np.min(ms)), "apply_ms_max": float(np.max(ms))}))


def bitwise():
    """Digests of the tables after (1) TripleTrainer.apply() on a seeded placed state at the bench's 200 000 + 600 rows
    and (2) one one-launch fed step (duo scorer) on a batch in which every row is written by at most one scorer
    contribution, so no float atomics are reordered: two libraries with the same arithmetic give the same digests."""
    import hashlib
    import torch
    sys.path.insert(0, ROOT)
    from openea_b200 import engine as eng
    n_ent, n_rel, d, lr = 200000, 600, 100, 0.01
    digests = {}
    for case in ("apply", "fed_step"):
        rng = np.random.default_rng(7)
        tabs = []
        for n in (n_ent, n_rel):
            t = eng.EmbeddingTable(rng.standard_normal((n, d), dtype=np.float32), True, "Adagrad", device="cuda")
            f = rng.random(n) < 0.15
            g = np.zeros((n, t.pitch), np.float32)
            g[f, :d] = rng.standard_normal((int(f.sum()), d), dtype=np.float32)
            t.grad.copy_(torch.from_numpy(g))
            t.touched.copy_(torch.from_numpy(f.astype(np.int32)))
            t.state1[:, :d] = torch.from_numpy(rng.uniform(0.1, 2.0, (n, d)).astype(np.float32)).cuda()
            tabs.append(t)
        tr = eng.TripleTrainer(tabs[0], tabs[1], eng.loss_cfg("limited", "L2", 0.01, 2.0, 0.2), lr)
        if case == "apply":
            tr.apply()
        else:
            n_pos, k = 128, 3
            ents = rng.permutation(n_ent)[: n_pos * (2 + k)].astype(np.int32)
            pos = np.stack([ents[:n_pos], rng.permutation(n_rel)[:n_pos].astype(np.int32), ents[n_pos:2 * n_pos]])
            neg = np.repeat(pos, k, axis=1)
            neg[0, ::2] = ents[2 * n_pos:2 * n_pos + neg[0, ::2].shape[0]]
            neg[2, 1::2] = ents[2 * n_pos + neg[0, ::2].shape[0]:2 * n_pos + neg.shape[1]]
            tr.step_fed_grouped(torch.from_numpy(pos).cuda(), torch.from_numpy(np.ascontiguousarray(neg)).cuda())
        torch.cuda.synchronize()
        h = hashlib.sha256()
        for t in tabs:
            for x in (t.weight, t.state1, t.grad, t.touched):
                h.update(x.cpu().numpy().tobytes())
        digests[case] = h.hexdigest()
    print(json.dumps(digests))


def _dump_diff(a, b):
    out = {}
    for name in sorted(os.listdir(a)):
        x, y = np.load(os.path.join(a, name)), np.load(os.path.join(b, name))
        out[name[:-4]] = float(np.max(np.abs(x.astype(np.float64) - y.astype(np.float64)))) if x.size else 0.0
    return out


def run(runs=5, out=None):
    out = out or tempfile.mkdtemp(prefix="ab_rowopt_")
    os.makedirs(out, exist_ok=True)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    report = {"gpu": smi, "parent_rev": open(os.path.join(PARENT_DIR, "REV")).read().strip(), "runs": {"parent": [], "new": []}}
    for i in range(runs):
        for arm in (("parent", "new") if i % 2 == 0 else ("new", "parent")):
            d = _bench(arm)
            report["runs"][arm].append({k: f(d) for k, f in FIELDS})
            print(arm, report["runs"][arm][-1], flush=True)
    report["apply"] = {}
    for arm in ("parent", "new"):
        res = subprocess.run([sys.executable, os.path.abspath(__file__), "apply_timing"], capture_output=True, text=True,
                             env=_env(arm), timeout=1200)
        report["apply"][arm] = json.loads(res.stdout.strip().splitlines()[-1]) if res.returncode == 0 else res.stderr[-1000:]
    report["bitwise"] = {}
    for arm in ("parent", "new"):
        res = subprocess.run([sys.executable, os.path.abspath(__file__), "bitwise"], capture_output=True, text=True,
                             env=_env(arm), timeout=1200)
        report["bitwise"][arm] = json.loads(res.stdout.strip().splitlines()[-1]) if res.returncode == 0 else res.stderr[-1000:]
    report["bitwise"]["identical"] = report["bitwise"]["parent"] == report["bitwise"]["new"]
    report["dumps"] = {}
    with tempfile.TemporaryDirectory() as tmp:
        for wl in ("bootea_100k", "bootea_15k"):
            dirs = {}
            for tag, arm in (("parent_a", "parent"), ("parent_b", "parent"), ("new", "new")):
                dirs[tag] = os.path.join(tmp, wl, tag)
                _bench(arm, ["--workload", wl, "--no-secondary", "--dump-outputs", dirs[tag]])
            report["dumps"][wl] = {"parent_vs_parent": _dump_diff(dirs["parent_a"], dirs["parent_b"]),
                                   "new_vs_parent": _dump_diff(dirs["new"], dirs["parent_a"]),
                                   "loss_last_step": {t: float(np.load(os.path.join(p, "loss_last_step.npy"))[0]) for t, p in dirs.items()}}
    lines = ["GPU: " + smi, "parent: " + report["parent_rev"], "%-24s %-40s %-40s" % ("field", "parent median [min, max]", "new median [min, max]")]
    for k, _ in FIELDS:
        cols = []
        for arm in ("parent", "new"):
            v = np.array([r[k] for r in report["runs"][arm]], dtype=np.float64)
            cols.append("%.6g [%.6g, %.6g]" % (np.median(v), v.min(), v.max()))
        lines.append("%-24s %-40s %-40s" % (k, cols[0], cols[1]))
    lines.append("apply(): " + json.dumps(report["apply"]))
    lines.append("bitwise: " + json.dumps(report["bitwise"]))
    for wl, d in report["dumps"].items():
        lines.append("dumps %s: %s" % (wl, json.dumps(d)))
    with open(os.path.join(out, "ab_rowopt.json"), "w") as f:
        json.dump(report, f, indent=1)
    with open(os.path.join(out, "ab_rowopt.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    cmd = sys.argv[1] if len(sys.argv) > 1 else "run"
    if cmd == "build":
        build(*sys.argv[2:3])
    elif cmd == "apply_timing":
        apply_timing()
    elif cmd == "bitwise":
        bitwise()
    else:
        run(int(sys.argv[2]) if len(sys.argv) > 2 else 5, sys.argv[3] if len(sys.argv) > 3 else None)
