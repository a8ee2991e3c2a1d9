"""CPU: the N>1 host logic under torch.distributed/gloo with world_size 2 — triple sharding by head owner,
the per-epoch seed-row all-gather (SeedRowSync), owner assembly, and the k-way merge of partial column top-k
lists used by the sharded CSLS evaluation (values checked against the NumPy oracle)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from openea_b200 import parallel as par
    from oracle import finding as orf
    try:
        # ---- triple sharding: a partition by head owner
        rng = np.random.default_rng(0)
        tri = np.stack([rng.integers(0, 101, 500), rng.integers(0, 7, 500), rng.integers(0, 101, 500)], 1)
        mine = par.shard_triples(tri, rank, world)
        assert (mine[:, 0] % world == rank).all()
        cnt = torch.tensor([len(mine)])
        dist.all_reduce(cnt)
        assert int(cnt) == 500
        # ---- seed-row sync: after the sync every replica holds the OWNER's copy of every seed row
        rows, pitch = 101, 8
        w = torch.full((rows, pitch), float(rank + 1))          # replica r holds value r+1 everywhere
        seeds = np.array([3, 4, 10, 11, 11, 50, 99, 100])
        before = w.clone()
        sync = par.SeedRowSync(w, seeds, rank, world)
        sync.sync()
        for i in range(rows):
            if i in set(seeds.tolist()):
                assert (w[i] == float(i % world + 1)).all(), (rank, i, w[i])
            else:
                assert (w[i] == before[i]).all()
        assert sync.bytes_per_sync == world * sync.max_cnt * pitch * 4
        # ---- owner assembly: every row from its owner
        w2 = torch.full((rows, pitch), float(rank + 1))
        par.assemble_owned_rows(w2, rank, world)
        want = torch.tensor([(i % world) + 1.0 for i in range(rows)])
        assert (w2[:, 0] == want).all()
        # ---- sharded CSLS column means: partial top-k per row block, all-gather, merge == oracle
        rng = np.random.default_rng(5)
        s = rng.standard_normal((37, 23)).astype(np.float32)     # [n1, n2]
        k = 5
        lo, hi = par.block_range(37, rank, world)
        part_v, _ = orf.topk_rows(np.ascontiguousarray(s[lo:hi].T), k)       # columns over my rows → [n2, k]
        merged = par.merge_partial_topk(par.allgather_partial(torch.from_numpy(part_v)), k).numpy()
        np.testing.assert_allclose(merged, orf.nearest_k_mean(np.ascontiguousarray(s.T), k), rtol=1e-6)
        # ---- ragged row blocks re-assembled on every rank (the arg-max columns of the sharded evaluation)
        full = torch.arange(37 * 3, dtype=torch.int32).reshape(37, 3)
        assert torch.equal(par.allgather_blocks(full[lo:hi].clone(), 37), full)
        assert torch.equal(par.allgather_blocks(full[lo:hi, 0].clone(), 37), full[:, 0])
        ranges = [par.block_range(37, r, world) for r in range(world)]
        assert ranges[0][0] == 0 and ranges[-1][1] == 37 and all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
        out.put((rank, "ok"))
    except Exception as e:  # surface the failure in the parent
        out.put((rank, "FAIL: %r" % (e,)))
    finally:
        dist.destroy_process_group()


def test_world_size_2_gloo():
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    res = [out.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res


def _modes_worker(rank, world, port, out):
    """Round-2 additions under gloo: the push / pull split of the seed-row exchange, the delta-sum replica combination,
    and the exact-parity sharded-batch step with the product's kernel SOURCES doing the rank-local work on the CPU warp
    emulator (tests/emu) — against the same steps in one process."""
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from openea_b200 import engine as eng, parallel as par
        # ---- push() publishes, pull() applies: what happens to the table between the two does not leak into the peers' copies
        w = torch.full((41, 4), float(rank + 1))
        x = par.SeedRowSync(w, np.arange(0, 41, 3), rank, world)
        x.push()
        w += 100.0                                          # a training step between push and pull
        x.pull()
        for i in range(41):
            owner = i % world
            if i % 3 == 0 and owner != rank:
                assert (w[i] == owner + 1.0).all(), (rank, i, w[i])      # the owner's PUBLISHED value, not its later one
            else:
                assert (w[i] == rank + 1.0 + 100.0).all()
        assert x.status() == 0
        # ---- delta-sum: x ← x_ref + Σ_g (x_g − x_ref); replicas identical afterwards, optimiser slots included
        class T:                                             # the attribute surface ReplicaDeltaSum reads
            def __init__(self):
                self.weight = torch.arange(12, dtype=torch.float32).reshape(3, 4).clone()
                self.state1 = torch.full((3, 4), 0.1)
                self.state2 = None
        t = T()
        ref_w, ref_s = t.weight.clone(), t.state1.clone()
        comb = par.ReplicaDeltaSum([t])
        t.weight += (rank + 1) * 0.5                          # rank-dependent local training
        t.state1 += (rank + 1) * 0.25
        comb.sync()
        tot = sum(g + 1 for g in range(world))
        assert torch.allclose(t.weight, ref_w + 0.5 * tot) and torch.allclose(t.state1, ref_s + 0.25 * tot)
        t.weight += 1.0; comb.sync()                          # a second combination starts from the new common point
        assert torch.allclose(t.weight, ref_w + 0.5 * tot + world * 1.0)
        # ---- exact-parity step on the emulator: sharded batch + all-reduced gradients == the whole batch in one process
        from tests.emu import build_emu
        so = build_emu.build()
        if so is not None:
            build_emu.patch_engine(pytest.MonkeyPatch(), build_emu.load(so))
            rng = np.random.default_rng(3)
            n, n_rel, d = 60, 5, 12

            def kg(lo):
                tri = np.stack([rng.integers(lo, lo + n, 150), rng.integers(0, n_rel, 150), rng.integers(lo, lo + n, 150)], 1)
                return np.unique(tri.astype(np.int32), axis=0)
            t1, t2 = kg(0), kg(n)
            ent = (rng.standard_normal((2 * n, d)) / np.sqrt(d)).astype(np.float32)
            rel = (rng.standard_normal((n_rel, d)) / np.sqrt(d)).astype(np.float32)

            def make():
                kg1 = eng.DeviceKG(t1, np.arange(0, n), 2 * n, device="cpu"); kg2 = eng.DeviceKG(t2, np.arange(n, 2 * n), 2 * n, device="cpu")
                tset = eng.DeviceTripleSet([kg1.triples, kg2.triples], 2 * n, n_rel, device="cpu")
                tr = eng.TripleTrainer(eng.EmbeddingTable(ent, True, "Adagrad", device="cpu"), eng.EmbeddingTable(rel, True, "Adagrad", device="cpu"),
                                       eng.loss_cfg("limited", "L2", 0.1, 2.0, 0.2), 0.01)
                return tr, kg1, kg2, tset
            single, a1, a2, ats = make()
            sharded, b1, b2, bts = make()
            ex = par.ExactReplicaStep(sharded)
            for step in range(4):
                single.score_sampled(a1, a2, ats, 48, 5, step % 3, 77 + step // 3); single.apply()
                ex.step(b1, b2, bts, 48, 5, step % 3, 77 + step // 3)
            for a, b in ((single.ent, sharded.ent), (single.rel, sharded.rel)):
                assert torch.allclose(b.weight, a.weight, rtol=1e-4, atol=1e-6) and torch.allclose(b.state1, a.state1, rtol=1e-4, atol=1e-6)
                mine = b.weight.clone(); other = [torch.empty_like(mine) for _ in range(world)]
                dist.all_gather(other, mine)
                assert all(torch.equal(o, mine) for o in other)          # replicas bit-identical to each other
            assert abs(single.read_loss() - sharded.read_loss()) <= 1e-4 * abs(single.loss_dev.item() + 1.0) + 1e-3
        out.put((rank, "ok"))
    except Exception as e:
        import traceback
        out.put((rank, "FAIL: %r\n%s" % (e, traceback.format_exc())))
    finally:
        dist.destroy_process_group()


def test_round2_modes_world_size_2_gloo():
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_modes_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    res = [out.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res
