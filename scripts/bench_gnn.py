#!/usr/bin/env python
"""Path (ii) at BASELINE.json configs 4 and 5 (model level, synthetic 100K-shape graphs), one process per GPU:

    python -m torch.distributed.run --nproc-per-node 4 --master-addr 127.0.0.1 --master-port P scripts/bench_gnn.py --config alinet
    python -m torch.distributed.run --nproc-per-node 8 ...                                    scripts/bench_gnn.py --config rdgcn

 alinet (config 4): AliNet's graph (approaches/alinet.py:784-826, layer dims 500/400/300) with the entity rows sharded
        over the ranks (parallel_gnn.ShardedAliNetModel): one training step = forward, loss on 20 000 positive + 200 000
        negative links, backward, gradient sync, TF-Adam — the reference's one step per epoch at 100K.  The one-hop adjacency
        is the symmetric 0/1 matrix of the synthetic D_*_100K-shape triples; the two-hop matrix is a random sparse pattern with
        the real dataset's order of nnz (SURVEY Appendix B: 1.4-2.6·10⁶) because the Zipf hubs of the synthetic graph make its
        true two-hop neighbourhood far denser than D_Y_100K's.
 rdgcn  (config 5): the RDGCN layer (approaches/rdgcn.py:162-338, d = 300) row-sharded (parallel_gnn.ShardedRDGCNLayer) on the
        100K V2-shape graph (600 000 triples per KG), one training step, plus the 100 000 × 100 000 CSLS evaluation
        (manhattan... the reference's eval metric is inner on d = 300 here) row-sharded over the same ranks.
Times are CUDA events, max over ranks, median of the timed steps; rank 0 prints one JSON line."""
import argparse
import json
import os
import sys
import time
from types import SimpleNamespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def timed_steps(fn, steps, warm, device, dist):
    import torch
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(steps):
        if dist.is_initialized():
            dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1)], dtype=torch.float64, device=device)
        if dist.is_initialized():
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ts.append(float(t.item()))
    return float(np.median(ts)), ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", required=True, choices=["alinet", "rdgcn"])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--shape", default="100K")
    args = ap.parse_args()
    os.environ.setdefault("NCCL_DEBUG", "WARN")
    import scipy.sparse as sp
    import torch
    import torch.distributed as dist
    from openea_b200 import finding as F, gnn, parallel as par, parallel_gnn as pg
    from openea_b200.synth import SHAPES, synth_id_arrays
    rank, local_rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    peak = 6577.7
    pk = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(pk):
        peak = json.load(open(pk))["hbm_gbs"]
    t0 = time.time()
    out = {"config": args.config, "n_gpus": world, "shape": args.shape}
    if args.config == "alinet":
        arr = synth_id_arrays(args.shape, swapping=False)
        n = arr["n_ent"]
        tri = np.concatenate([arr["triples1"], arr["triples2"]])
        h, t = tri[:, 0].astype(np.int64), tri[:, 2].astype(np.int64)
        a1 = sp.csr_matrix((np.ones(2 * len(h), np.float32), (np.concatenate([h, t]), np.concatenate([t, h]))), shape=(n, n))
        a1.data[:] = 1.0
        a1 = gnn.preprocess_adj(a1) if hasattr(gnn, "preprocess_adj") else a1
        rng = np.random.default_rng(7)
        nnz2 = 2_600_000 if args.shape == "100K" else 400_000
        r2, c2 = rng.integers(0, n, nnz2), rng.integers(0, n, nnz2)
        a2 = sp.csr_matrix((np.ones(nnz2, np.float32), (r2, c2)), shape=(n, n)) + sp.eye(n, dtype=np.float32, format="csr")
        a2 = sp.csr_matrix(a2); a2.data[:] = 1.0
        dims = [500, 400, 300]
        shard = pg.RowShard(n)
        from openea_b200.approaches.alinet import AliNetModel, DenseAdam
        model = pg.ShardedAliNetModel(n, dims, a1, a2, dev, seed=3, shard=shard) if world > 1 else \
            AliNetModel(n, dims, gnn.DeviceCsr(a1, dev), gnn.DeviceCsr(a2, dev), dev, seed=3)
        opt = DenseAdam(list(model.params.values()), 0.001)
        links = arr["train_links"].astype(np.int64)
        B, k = min(20000, len(links)), 10
        g = torch.Generator().manual_seed(1)
        pos = torch.as_tensor(links[:B], device=dev)
        neg = torch.stack([pos[:, 0].repeat_interleave(k), torch.randint(0, n, (B * k,), generator=g).to(dev)], 1)
        out["build_s"] = round(time.time() - t0, 1)

        def step():
            outs = model.forward()
            loss = model.loss(outs, pos, neg, 1.5, 0.1)
            loss.backward()
            if hasattr(model, "sync_grads"):
                model.sync_grads()
            opt.step()
        ms, all_ms = timed_steps(step, args.steps, args.warmup, dev, dist)
        # dense flops of one forward (alinet.py:784-826): layer 0 X·W (500→400), X·K (500→400), X·K1, X·K2 (500→500), highway
        # (400→400); layer 1 X·W (400→300); backward ≈ 2× forward
        fwd = 2.0 * n * (500 * 400 * 2 + 500 * 500 * 2 + 400 * 400 + 400 * 300)
        spmm_bytes = (a1.nnz * 8 + (n + 1) * 4 + 2 * n * 400 * 4) + (a1.nnz * 8 + (n + 1) * 4 + 2 * n * 300 * 4) + (a2.nnz * 8 + (n + 1) * 4 + 2 * n * 400 * 4)
        out.update({"entities": n, "layer_dims": dims, "adj1_nnz": int(a1.nnz), "adj2_nnz": int(a2.nnz), "pos_links": B, "neg_links": B * k,
                    "ms_per_step": ms, "steps_ms": all_ms, "epochs_per_s": 1e3 / ms,
                    "dense_tflops_fwd_bwd_whole_job": 3.0 * fwd / (ms * 1e-3) / 1e12,
                    "spmm_compulsory_bytes_fwd": spmm_bytes,
                    "note": "one step = one epoch at this batch size (alinet.py:1041: steps = len(sup_ent2) // batch_size)"})
    else:
        arr = synth_id_arrays(args.shape, swapping=False)
        if args.shape == "100K":     # V2 density: twice the triples (SURVEY 8d)
            rng = np.random.default_rng(9)
            extra = lambda tri, ents: np.stack([rng.choice(ents, len(tri)), tri[:, 1], rng.choice(ents, len(tri))], 1).astype(np.int32)
            arr = dict(arr)
            arr["triples1"] = np.unique(np.concatenate([arr["triples1"], extra(arr["triples1"], arr["entities1"])]), axis=0)
            arr["triples2"] = np.unique(np.concatenate([arr["triples2"], extra(arr["triples2"], arr["entities2"])]), axis=0)
        n, r = arr["n_ent"], arr["n_rel"]
        d, k = 300, 10
        links = arr["train_links"]
        kgs = SimpleNamespace(kg1=SimpleNamespace(relation_triples_list=[tuple(x) for x in arr["triples1"].tolist()]),
                              kg2=SimpleNamespace(relation_triples_list=[tuple(x) for x in arr["triples2"].tolist()]),
                              entities_num=n, relations_num=r, train_links=[(int(a), int(b)) for a, b in links.tolist()])
        margs = SimpleNamespace(dim=d, alpha=0.1, beta=0.3, gamma=1.0, neg_triple_num=k)
        rng = np.random.default_rng(2)
        emb = rng.standard_normal((n, d)).astype(np.float32)
        from openea_b200.approaches.rdgcn import RDGCNLayer
        from openea_b200.approaches.alinet import DenseAdam
        shard = pg.RowShard(n)
        layer = pg.ShardedRDGCNLayer(margs, kgs, emb, dev, seed=5, shard=shard) if world > 1 else RDGCNLayer(margs, kgs, emb, dev, seed=5)
        t = len(links)
        negs = tuple(torch.as_tensor(x, dtype=torch.int32, device=dev) for x in
                     (np.repeat(links[:, 0], k), rng.integers(0, n, t * k), rng.integers(0, n, t * k), np.repeat(links[:, 1], k)))
        opt = DenseAdam([p for p in layer.params.values() if p.dim() == 2 and p.shape[1] % 4 == 0], 0.001)
        out["build_s"] = round(time.time() - t0, 1)

        def step():
            o = layer.forward()
            loss = layer.loss(o, negs)
            loss.backward()
            if hasattr(layer, "sync_grads"):
                layer.sync_grads()
            opt.step()
            for p in layer.params.values():
                p.grad = None
        ms, all_ms = timed_steps(step, args.steps, args.warmup, dev, dist)
        out.update({"entities": n, "relations": r, "triples": int(len(arr["triples1"]) + len(arr["triples2"])), "dim": d,
                    "seed_links": t, "neg_per_link": k, "ms_per_step": ms, "steps_ms": all_ms, "epochs_per_s": 1e3 / ms})
        # the 100 000 x 100 000 CSLS evaluation of config 5, E1 rows sharded over the ranks
        m = 100000 if args.shape == "100K" else 10500
        g = torch.Generator().manual_seed(99)
        e2 = torch.randn(m, d, generator=g)
        e1 = (e2 + 0.5 * torch.randn(m, d, generator=g)).to(dev)
        e2 = e2.to(dev)
        if world > 1:
            par.mark_replicas_in_sync(True)

        def ev():
            if world > 1:
                return F.eval_alignment_sharded(e1, e2, [1, 5, 10, 50], "inner", False, 10)
            return F.eval_alignment(e1, e2, [1, 5, 10, 50], "inner", False, 10)
        ems, e_all = timed_steps(ev, 3, 1, dev, dist)
        out["csls"] = {"n1": m, "n2": m, "dim": d, "ms": ems, "all_ms": e_all, "pairs_per_s": float(m) * m / (ems * 1e-3),
                       "fp32_tflops_contraction": 2.0 * m * m * d / (ems * 1e-3) / 1e12}
    if rank == 0:
        print(json.dumps(out))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
