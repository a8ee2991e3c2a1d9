"""GPU, >= 2 devices: the sharded CSLS evaluation over NCCL equals the single-GPU evaluation; the seed-row sync
moves the owners' rows between replicas.  Skipped on machines with fewer than two GPUs."""
import os
import socket

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from openea_b200 import finding as F, parallel as par
        rng = np.random.default_rng(0)
        e2 = rng.standard_normal((3000, 100)).astype(np.float32)
        e1 = (e2[:2500] + 0.5 * rng.standard_normal((2500, 100))).astype(np.float32)
        for metric, csls in (("inner", 10), ("manhattan", 5), ("inner", 0)):
            hits, mr, mrr, (lo, hi, top1, rk) = F.eval_alignment_sharded(e1, e2, [1, 5, 10], metric, metric == "inner", csls)
            wtop1, wrk, whits, wmr, wmrr = F.eval_alignment(e1, e2, [1, 5, 10], metric, metric == "inner", csls)
            assert hits == whits and abs(mr - wmr) < 1e-9 and abs(mrr - wmrr) < 1e-12, (metric, csls, hits, whits)
            assert torch.equal(top1, wtop1[lo:hi]) and torch.equal(rk, wrk[lo:hi])
        w = torch.full((101, 8), float(rank + 1), device="cuda")
        par.SeedRowSync(w, np.array([3, 4, 10, 11, 50]), rank, world).sync()
        assert float(w[3, 0]) == 3 % world + 1 and float(w[4, 0]) == 4 % world + 1 and float(w[5, 0]) == rank + 1
        out.put((rank, "ok"))
    except Exception as e:
        out.put((rank, "FAIL: %r" % (e,)))
    finally:
        dist.destroy_process_group()


def test_sharded_eval_equals_single_gpu():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    res = [out.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res


def _xchg_worker(rank, world, port, out):
    """Seed-row exchange transports: own kernels over peer memory ('p2p'), pack + ncclAllGather + unpack ('nccl')."""
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from openea_b200 import parallel as par
        rng = np.random.default_rng(5)
        rows, pitch = 4001, 100
        seeds = rng.permutation(rows)[:1500]
        owner = seeds % world
        modes = {}
        for mode in ("p2p", "nccl"):
            w = torch.zeros(rows, pitch, device="cuda")
            x = par.SeedRowSync(w, seeds, rank, world, mode=mode)
            modes[mode] = x.mode
            for epoch in range(1, 6):        # five epochs: both parities of the double buffer are reused
                # every rank's replica: row r holds (epoch, rank, r) patterns; after the exchange a seed row must hold its
                # OWNER's pattern, every other row this rank's own
                base = torch.arange(rows, device="cuda", dtype=torch.float32)[:, None] + torch.arange(pitch, device="cuda")[None, :] / 128.0
                w.copy_(base + 10000.0 * epoch + 1000000.0 * rank)
                x.push()
                w[0, 0] += 0.0               # an unrelated kernel between push and pull (the training step's place)
                x.pull()
                torch.cuda.synchronize()
                want = (base + 10000.0 * epoch + 1000000.0 * rank).clone()
                so = torch.as_tensor(seeds, device="cuda"), torch.as_tensor(owner, device="cuda", dtype=torch.float32)
                want[so[0]] = base[so[0]] + 10000.0 * epoch + 1000000.0 * so[1][:, None]
                assert torch.equal(w, want), (mode, epoch, int((w != want).sum()))
            assert x.status() == 0
            x.close()
        out.put((rank, "ok " + modes["p2p"]))
    except Exception as e:
        import traceback
        out.put((rank, "FAIL: %r\n%s" % (e, traceback.format_exc())))
    finally:
        dist.destroy_process_group()


def test_seed_row_exchange_transports():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_xchg_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    res = [out.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    # the peer-memory transport must actually have been used on a P2P-capable box (no silent fallback)
    assert sorted(res) == [(0, "ok p2p"), (1, "ok p2p")], res


def _exact_setup(seed=11):
    from openea_b200 import engine as eng
    from tests.helpers import make_tables
    rng = np.random.default_rng(seed)
    n_ent, n_rel, d = 3000, 24, 100
    ent, rel = make_tables(rng, n_ent, n_rel, d)
    ents1, ents2 = np.arange(0, n_ent, 2, dtype=np.int32), np.arange(1, n_ent, 2, dtype=np.int32)

    def mk(ents, n, lo, hi):
        tri = np.stack([rng.choice(ents, n), rng.integers(lo, hi, n), rng.choice(ents, n)], 1).astype(np.int32)
        return np.unique(tri, axis=0)
    t1, t2 = mk(ents1, 2600, 0, 12), mk(ents2, 2200, 12, 24)
    kg1, kg2 = eng.DeviceKG(t1, ents1, n_ent), eng.DeviceKG(t2, ents2, n_ent)
    tset = eng.DeviceTripleSet([kg1.triples, kg2.triples], n_ent, n_rel)
    te, tr = eng.EmbeddingTable(ent, True, "Adagrad", "cuda"), eng.EmbeddingTable(rel, True, "Adagrad", "cuda")
    trn = eng.TripleTrainer(te, tr, eng.loss_cfg("limited", "L2", 0.01, 2.0, 0.2), lr=0.01)
    return trn, kg1, kg2, tset


def test_batch_shards_union_is_the_whole_batch(cuda_device):
    """One GPU: the gradients of the G shards of a step's batch (shard = (g, G)) add up to the whole batch's gradients,
    same touched rows, same loss — the property the exact-parity multi-GPU mode rests on."""
    B, k = 512, 10
    for G in (2, 3, 8):
        whole, kg1, kg2, tset = _exact_setup()
        parts, *_ = _exact_setup()
        for step in range(2):
            whole.score_sampled(kg1, kg2, tset, B, k, step, 4242)
            for g in range(G):
                parts.score_sampled(kg1, kg2, tset, B, k, step, 4242, shard=(g, G))
            torch.cuda.synchronize()
            for a, b in ((whole.ent, parts.ent), (whole.rel, parts.rel)):
                torch.testing.assert_close(b.grad, a.grad, rtol=1e-4, atol=1e-6)
                assert torch.equal(a.touched != 0, b.touched != 0)
            lw, lp = whole.read_loss(), parts.read_loss()
            assert abs(lw - lp) <= 1e-6 * abs(lw), (lw, lp)
            whole.apply(); parts.apply()


def _exact_worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from openea_b200 import parallel as par
        B, k, steps = 512, 10, 12
        single, kg1, kg2, tset = _exact_setup()
        sharded, kg1b, kg2b, tsetb = _exact_setup()
        ex = par.ExactReplicaStep(sharded)
        for step in range(steps):
            single.step_sampled(kg1, kg2, tset, B, k, step % 9, 99 + step // 9)
            ex.step(kg1b, kg2b, tsetb, B, k, step % 9, 99 + step // 9)
        torch.cuda.synchronize()
        lw, lp = single.read_loss(), sharded.read_loss()
        assert abs(lw - lp) <= 1e-4 * abs(lw), (lw, lp)
        for a, b in ((single.ent, sharded.ent), (single.rel, sharded.rel)):
            torch.testing.assert_close(b.weight, a.weight, rtol=1e-4, atol=1e-6)
            torch.testing.assert_close(b.state1, a.state1, rtol=1e-4, atol=1e-6)
            # replicas are bit-identical to each other
            mine = b.weight.clone()
            other = [torch.empty_like(mine) for _ in range(world)]
            dist.all_gather(other, mine)
            assert all(torch.equal(o, mine) for o in other)
        out.put((rank, "ok"))
    except Exception as e:
        import traceback
        out.put((rank, "FAIL: %r\n%s" % (e, traceback.format_exc())))
    finally:
        dist.destroy_process_group()


def test_exact_parity_mode_equals_single_gpu():
    """SURVEY §8e exact-parity mode over NCCL: 12 sharded-batch steps on 2 GPUs leave the tables and Adagrad slots within
    1e-4 of the single-GPU run on the same seeds, and the replicas bit-identical to each other."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_exact_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    res = [out.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res


def _gcn_worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        import scipy.sparse as sp
        from openea_b200 import gnn, parallel_gnn as pg
        from openea_b200.approaches.gcn_align import GCNAlignUnit
        from openea_b200.engine import EmbeddingTable
        rng = np.random.default_rng(4)
        n, d, t, k = 2003, 100, 150, 5
        a = sp.random(n, n, density=0.004, random_state=7, format="csr", dtype=np.float32)
        support = gnn.preprocess_adj(a + a.T)
        W0 = (rng.standard_normal((n, d)) / np.sqrt(n)).astype(np.float32)
        ill = np.stack([rng.permutation(n)[:t], rng.permutation(n)[:t]], 1)
        negs = [np.repeat(ill[:, 0], k), rng.integers(0, n, t * k), rng.integers(0, n, t * k), np.repeat(ill[:, 1], k)]
        tn = [torch.as_tensor(x, dtype=torch.int32, device="cuda") for x in negs]
        single = GCNAlignUnit(gnn.DeviceCsr(support, "cuda"), EmbeddingTable(W0, True, "SGD", "cuda"), None, ill, 3.0, k, 8.0)
        shard = pg.RowShard(n)
        unit = pg.ShardedGCNAlignUnit(support, EmbeddingTable(shard.local_rows(W0), True, "SGD", "cuda"), None, ill,
                                      3.0, k, 8.0, shard=shard)
        for _ in range(3):
            want = float(single.train_step(*tn))
            got = float(unit.train_step(*tn))
            assert abs(got - want) <= 1e-4 * max(1.0, abs(want)), (got, want)
            torch.testing.assert_close(unit.outputs, single.outputs, rtol=1e-4, atol=1e-6)
        W = shard.to_global(pg.all_gather_rows(unit.table.weight, shard))
        torch.testing.assert_close(W, single.table.weight, rtol=1e-4, atol=1e-6)
        out.put((rank, "ok"))
    except Exception as e:
        import traceback
        out.put((rank, "FAIL: %r\n%s" % (e, traceback.format_exc())))
    finally:
        dist.destroy_process_group()


def test_row_sharded_gcn_unit_equals_single_gpu():
    """SURVEY §8e-ii over NCCL: the row-sharded GCN-Align unit (liboea kernels + 3 all-gathers / 3 reduce-scatters per
    step) reproduces the single-GPU unit's loss, outputs and updated entity table."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gcn_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    res = [out.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res


def _alinet_worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        import scipy.sparse as sp
        from openea_b200 import gnn, parallel_gnn as pg
        from openea_b200.approaches.alinet import AliNetModel
        rng = np.random.default_rng(11)
        n, dims = 3001, [64, 48, 32]
        a1 = sp.csr_matrix(sp.random(n, n, density=0.003, random_state=1, format="csr", dtype=np.float32) + sp.eye(n, dtype=np.float32))
        a2 = sp.csr_matrix(sp.random(n, n, density=0.006, random_state=2, format="csr", dtype=np.float32) + sp.eye(n, dtype=np.float32))
        a2.data[:] = 1.0
        dev = torch.device("cuda", rank)
        pos = torch.as_tensor(np.stack([rng.permutation(n)[:200], rng.permutation(n)[:200]], 1), device=dev)
        neg = torch.as_tensor(np.stack([rng.integers(0, n, 2000), rng.integers(0, n, 2000)], 1), device=dev)
        ref = AliNetModel(n, dims, gnn.DeviceCsr(a1, dev), gnn.DeviceCsr(a2, dev), dev, seed=3)
        ref_outs = ref.forward()
        ref_loss = ref.loss(ref_outs, pos, neg, 1.5, 0.1)
        ref_loss.backward()
        shard = pg.RowShard(n)
        model = pg.ShardedAliNetModel(n, dims, a1, a2, dev, seed=3, shard=shard)
        outs = model.forward()
        for o, r in zip(outs, ref_outs):
            torch.testing.assert_close(o, r, rtol=1e-4, atol=1e-5)
        loss = model.loss(outs, pos, neg, 1.5, 0.1)
        torch.testing.assert_close(loss, ref_loss, rtol=1e-4, atol=1e-4)
        loss.backward()
        model.sync_grads()
        for name, p in model.params.items():
            want = ref.params[name].grad
            if name == "init_embedding":
                want = torch.as_tensor(shard.local_rows(want.cpu().numpy()), device=dev)
            torch.testing.assert_close(p.grad, want, rtol=1e-3, atol=1e-5, msg=lambda m, name=name: "%s: %s" % (name, m))
        out.put((rank, "ok"))
    except Exception as e:
        import traceback
        out.put((rank, "FAIL: %r\n%s" % (e, traceback.format_exc())))
    finally:
        dist.destroy_process_group()


def test_row_sharded_alinet_model_equals_single_gpu():
    """The row-sharded AliNet model (liboea aggregation kernels on rectangular row blocks + autograd all-gathers) gives
    the single-GPU model's layer outputs, loss and gradients."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_alinet_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    res = [out.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res


def _rdgcn_worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from types import SimpleNamespace
        from openea_b200 import parallel_gnn as pg
        from openea_b200.approaches.rdgcn import RDGCNLayer
        rng = np.random.default_rng(21)
        n, r, d, t, k = 2501, 23, 64, 120, 5
        tri = np.unique(np.stack([rng.integers(0, n, 9000), rng.integers(0, r, 9000), rng.integers(0, n, 9000)], 1), axis=0)
        half = len(tri) // 2
        kgs = SimpleNamespace(kg1=SimpleNamespace(relation_triples_list=[tuple(x) for x in tri[:half].tolist()]),
                              kg2=SimpleNamespace(relation_triples_list=[tuple(x) for x in tri[half:].tolist()]),
                              entities_num=n, relations_num=r,
                              train_links=[(int(a), int(b)) for a, b in zip(rng.permutation(n)[:t], rng.permutation(n)[:t])])
        args = SimpleNamespace(dim=d, alpha=0.1, beta=0.3, gamma=1.0, neg_triple_num=k)
        emb = rng.standard_normal((n, d)).astype(np.float32)
        dev = torch.device("cuda", rank)
        ill = np.array(kgs.train_links)
        negs = tuple(torch.as_tensor(x, dtype=torch.int32, device=dev) for x in
                     (np.repeat(ill[:, 0], k), rng.integers(0, n, t * k), rng.integers(0, n, t * k), np.repeat(ill[:, 1], k)))
        ref = RDGCNLayer(args, kgs, emb, dev, seed=5)
        ref_out = ref.forward()
        ref_loss = ref.loss(ref_out, negs)
        ref_loss.backward()
        shard = pg.RowShard(n)
        layer = pg.ShardedRDGCNLayer(args, kgs, emb, dev, seed=5, shard=shard)
        out_full = layer.forward()
        torch.testing.assert_close(out_full, ref_out, rtol=1e-4, atol=1e-5)
        loss = layer.loss(out_full, negs)
        torch.testing.assert_close(loss, ref_loss, rtol=1e-4, atol=1e-5)
        loss.backward()
        layer.sync_grads()
        for name, p in layer.params.items():
            want = ref.params[name].grad
            if name == "X0":
                want = torch.as_tensor(shard.local_rows(want.cpu().numpy()), device=dev)
            atol = max(1e-4 * float(want.abs().max()), 1e-7)
            torch.testing.assert_close(p.grad, want, rtol=1e-3, atol=atol, msg=lambda m, name=name: "%s: %s" % (name, m))
        out.put((rank, "ok"))
    except Exception as e:
        import traceback
        out.put((rank, "FAIL: %r\n%s" % (e, traceback.format_exc())))
    finally:
        dist.destroy_process_group()


def test_row_sharded_rdgcn_layer_equals_single_gpu():
    """The row-sharded RDGCN layer (entity rows sharded, relation-side tensors replicated, 2 all-reduces + 5 all-gathers
    per forward) gives the single-GPU layer's output, loss and gradients with the real kernels."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rdgcn_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    res = [out.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res


def _bootea_worker(rank, world, port, folder, out, mode):
    import contextlib
    import io
    import re
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from openea_b200 import presets
        from openea_b200.approaches import BootEA
        from openea_b200.modules.load.kgs import read_kgs_from_folder
        args = presets.bootea("15K")
        args.training_data, args.output = folder, folder + "out%d/" % rank
        args.batch_size, args.max_epoch, args.start_valid, args.sub_epoch = 1000, 200, 100, 10
        args.truncated_epsilon, args.dim, args.sim_th = 0.9, 32, 0.5
        args.multi_gpu_mode = mode
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            kgs = read_kgs_from_folder(folder, args.dataset_division, "swapping", True)
            m = BootEA(); m.set_args(args); m.set_kgs(kgs); m.init(); m.run(); m.test(save=False)
        text = buf.getvalue()
        h1 = float(re.findall(r"accurate results: hits@\[1, 5, 10, 50\] = \[\s*([0-9.]+)", text)[-1])
        local = int(m._dkg1.triples.shape[0] + m._dkg2.triples.shape[0])
        total = torch.tensor([local], device="cuda"); dist.all_reduce(total)
        n_all = kgs.kg1.relation_triples_num + kgs.kg2.relation_triples_num
        # 'seed': the ranks' shards are a partition of the triples; 'exact': every rank holds all of them (the batch is sharded)
        assert int(total) == (n_all if mode == "seed" else world * n_all)
        agree = torch.tensor([h1, -h1], device="cuda", dtype=torch.float64); dist.all_reduce(agree, op=dist.ReduceOp.MAX)
        assert float(agree[0]) == h1 and float(-agree[1]) == h1, "every rank must print the same (sharded) evaluation"
        # chance is 0.24 %.  ONE device with this configuration (200 epochs, validation / early stop from epoch 100; the CPU
        # warp emulator) reaches 5.00 %, early stop at epoch 120; the exact mode equals one device up to fp32 summation order,
        # so its threshold sits below that with room for seed noise.  The stale seed-row mode trains, but visibly worse
        # (DESIGN.md §6: it discards the gradients non-owners produce), hence its lower bar.  That exact ≡ one GPU numerically (1e-4) is pinned by
        # test_exact_parity_mode_equals_single_gpu; this test checks the lifecycle plumbing and that the model learns.
        assert h1 > (3.0 if mode == "exact" else 0.8), h1
        out.put((rank, "ok"))
    except Exception as e:
        import traceback
        out.put((rank, "FAIL: %r\n%s" % (e, traceback.format_exc())))
    finally:
        dist.destroy_process_group()


@pytest.mark.first_hw_run
@pytest.mark.parametrize("mode", ["exact", "seed"])
def test_bootea_lifecycle_on_two_gpus(tmp_path, mode):
    """SURVEY §8e-i through the reference lifecycle under both multi-GPU modes: 'exact' (default: batch sharded, gradients
    all-reduced, one-GPU accuracy) and 'seed' (head-owner triple shards, per-epoch seed-row exchange over peer memory,
    replicas assembled before validation / bootstrapping / test) — sharded evaluation, every rank reports the same result."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    from openea_b200.synth import write_dataset
    folder = write_dataset(str(tmp_path) + "/tiny/", "tiny")
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_bootea_worker, args=(r, 2, port, folder, out, mode)) for r in range(2)]
    for p in procs:
        p.start()
    res = [out.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res
