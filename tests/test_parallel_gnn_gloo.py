"""CPU: the row-sharded GCN-Align unit (openea_b200/parallel_gnn.py, SURVEY §8e-ii) under torch.distributed/gloo with
world sizes 2 and 3: partition + padding, the three all-gathers and three reduce-scatters per step, pair sharding and
loss weighting.  The rank-local numerics come from a torch stand-in (the kernels need a GPU); the result must equal the
single-process oracle step (oracle/gnn.py) — i.e. the collective algebra is exact."""
import os
import socket

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


class _Csr:
    def __init__(self, mat):
        self.m = sp.csr_matrix(mat, dtype=np.float32)          # duplicate entries are kept as they are
        self.shape, self.nnz = self.m.shape, self.m.nnz
        self.val = torch.tensor(self.m.data, dtype=torch.float32)
        c = self.m.tocoo(copy=True)
        self.t = torch.sparse_coo_tensor(np.vstack([c.row, c.col]), c.data, c.shape).coalesce()

    def transpose(self):
        return _Csr(self.m.T)


class _Table:
    def __init__(self, values):
        self.weight = torch.tensor(values, dtype=torch.float32)
        self.dim = self.weight.shape[1]
        self.device = torch.device("cpu")


class TorchOps:
    """Rank-local numerics of the unit in plain torch (test stand-in for KernelOps)."""

    def csr(self, mat, device, keep_duplicates=False):
        return _Csr(mat)

    def spmm(self, A, X, relu=False, mask_src=None):
        y = torch.sparse.mm(A.t, X)
        if relu:
            y = torch.relu(y)
        if mask_src is not None:
            y = y * (mask_src > 0)
        return y

    def lookup(self, table):
        from oracle.gnn import l2n
        return l2n(table.weight)

    def update(self, table, grad_rows, lr):
        from oracle.gnn import l2n
        w = table.weight.clone().requires_grad_(True)
        (l2n(w) * grad_rows).sum().backward()
        table.weight -= lr * w.grad

    def align_loss(self, x, dim, left, right, k, negs, gamma, grad, loss_out):
        from oracle.gnn import align_loss
        xg = x.clone().requires_grad_(True)
        ill = np.stack([left.numpy(), right.numpy()], 1)
        loss = align_loss(xg, ill, gamma, k, *[n.numpy() for n in negs])
        loss.backward()
        grad += xg.grad
        loss_out += loss.detach().double()


class EmuOps(TorchOps):
    """The unit's sparse products and its loss through the REAL kernel sources (oea_spmm.cu on the CPU warp emulator):
    the sharded row blocks, padded rows, position-mapped indices and the relu-mask epilogue reach the same code a GPU
    runs.  Table lookups / updates stay the torch stand-ins (their kernels live in a file the emulator does not cover)."""

    def __init__(self):
        import ctypes as C
        from tests.emu import build_emu
        from tests.test_emu_spmm import HostCsr
        self.C, self.HostCsr = C, HostCsr
        self.lib = build_emu.load()

    def csr(self, mat, device, keep_duplicates=False):
        ops = self

        class Wrapped(ops.HostCsr):
            def transpose(self):
                return Wrapped(ops.lib, self.m.T)
        return Wrapped(self.lib, mat)

    @staticmethod
    def _padded(x):
        """[n, d] → contiguous float32 [n, ceil4(d)] NumPy buffer (the kernels want 16-byte rows)."""
        a = x.detach().numpy().astype(np.float32)
        p = (a.shape[1] + 3) // 4 * 4
        out = np.zeros((a.shape[0], p), dtype=np.float32)
        out[:, :a.shape[1]] = a
        return out

    def spmm(self, A, X, relu=False, mask_src=None):
        C = self.C
        x = self._padded(X)
        d = x.shape[1]
        y = np.zeros((A.m.shape[0], d), dtype=np.float32)
        m = None if mask_src is None else self._padded(mask_src)
        nbytes = self.lib.oea_spmm_workspace_bytes(A.n_seg, d)
        ws = np.zeros(max(4, nbytes // 4), dtype=np.float32)
        cs, hb = A.csr(), A.hubs()
        rc = self.lib.oea_spmm_csr(C.byref(cs), C.byref(hb), x.ctypes.data, d, y.ctypes.data, d, d, int(relu),
                                   None if m is None else m.ctypes.data, 0.0, ws.ctypes.data, nbytes, None)
        assert rc == 0, rc
        return torch.from_numpy(y[:, :X.shape[1]].copy())

    def align_loss(self, x, dim, left, right, k, negs, gamma, grad, loss_out):
        xp = self._padded(x)
        g = np.zeros_like(xp)
        loss = np.zeros(1, dtype=np.float64)
        i32 = lambda t: np.ascontiguousarray(t.numpy(), dtype=np.int32)
        arrs = [i32(left), i32(right)] + [i32(n) for n in negs]
        rc = self.lib.oea_align_loss_l1(xp.ctypes.data, xp.shape[1], dim, arrs[0].ctypes.data, arrs[1].ctypes.data, len(arrs[0]),
                                        k, arrs[2].ctypes.data, arrs[3].ctypes.data, arrs[4].ctypes.data, arrs[5].ctypes.data,
                                        gamma, loss.ctypes.data, g.ctypes.data, None)
        assert rc == 0, rc
        grad += torch.from_numpy(g[:, :x.shape[1]])
        loss_out += float(loss[0])


def _problem(with_features):
    rng = np.random.default_rng(4)
    n, d, t, k = 53, 8, 11, 3                      # 53 rows: ragged last block for world 2 and 3
    a = sp.random(n, n, density=0.08, random_state=7, format="csr", dtype=np.float32)
    a = a + a.T + sp.eye(n, dtype=np.float32)
    deg = np.asarray(a.sum(1)).ravel()
    support = sp.diags(deg ** -0.5) @ a @ sp.diags(deg ** -0.5)
    feats = sp.random(n, 9, density=0.3, random_state=3, format="csr", dtype=np.float32) if with_features else None
    if feats is not None:
        feats.data[:] = 1.0
    W0 = rng.standard_normal((9 if with_features else n, d)).astype(np.float32)
    ill = np.stack([rng.permutation(n)[:t], rng.permutation(n)[:t]], 1)
    negs = [np.repeat(ill[:, 0], k), rng.integers(0, n, t * k), rng.integers(0, n, t * k), np.repeat(ill[:, 1], k)]
    return support, feats, W0, ill, negs, k


def _worker(rank, world, port, with_features, out, ops_kind="torch"):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from openea_b200 import parallel_gnn as pg
        from oracle import gnn as orc
        support, feats, W0, ill, negs, k = _problem(with_features)
        gamma, lr = 1.0, 0.5
        shard = pg.RowShard(support.shape[0])
        assert (shard.rank, shard.world) == (rank, world) and shard.n_pad == shard.block * world >= shard.n
        table = _Table(W0 if with_features else shard.local_rows(W0))
        ops = EmuOps() if ops_kind == "kernels" else TorchOps()
        unit = pg.ShardedGCNAlignUnit(support, table, feats, ill, gamma, k, lr, shard=shard, ops=ops)
        tn = [torch.as_tensor(x, dtype=torch.int32) for x in negs]
        want_W = W0
        for _ in range(2):
            got = float(unit.train_step(*tn))
            want_loss, want_W, want_out = orc.unit_train_step(support, want_W, feats, ill, gamma, k, negs, lr)
            assert abs(got - want_loss) <= 1e-5 * max(1.0, abs(want_loss)), (got, want_loss)
            np.testing.assert_allclose(unit.outputs.numpy(), want_out, rtol=1e-4, atol=1e-6)
        if with_features:
            W = table.weight.numpy()                                     # replicated: identical on every rank
        else:
            W = shard.to_global(pg.all_gather_rows(table.weight, shard)).numpy()   # assemble the owners' rows in id order
            assert not table.weight[shard.n_local:].any(), "padding rows of the shard must stay zero"
        np.testing.assert_allclose(W, want_W, rtol=1e-4, atol=1e-6)
        out.put((rank, "ok"))
    except Exception as e:  # surface the failure in the parent
        import traceback
        out.put((rank, "FAIL: %r\n%s" % (e, traceback.format_exc())))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,ops_kind", [(2, "torch"), (3, "torch"), (2, "kernels")])
@pytest.mark.parametrize("with_features", [False, True])
def test_sharded_gcn_unit_equals_single_process_oracle(world, with_features, ops_kind):
    """ops_kind 'kernels': the SpMMs and the alignment loss run the product's kernel sources on the CPU warp emulator."""
    if ops_kind == "kernels":
        from tests.emu import build_emu
        if build_emu.build() is None:
            pytest.skip("no CUDA headers for the emulator build")
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, with_features, out, ops_kind)) for r in range(world)]
    for p in procs:
        p.start()
    res = [out.get(timeout=400) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(r, "ok") for r in range(world)], res


def test_row_shard_partition_is_exact():
    """Cyclic ownership: the row blocks (columns renumbered to positions) reassemble the matrix, padding is empty,
    duplicates are merged or kept on request, and ownership balances a frequency-ordered degree profile."""
    from openea_b200 import parallel_gnn as pg
    m = sp.random(10, 10, density=0.5, random_state=1, format="csr")
    back = sp.lil_matrix((10, 10))
    for r in range(4):
        sh = pg.RowShard(10, rank=r, world_size=4)
        assert (sh.block, sh.n_pad) == (3, 12) and sh.my_ids.tolist() == list(range(r, 10, 4))
        blk = sh.square_rows_of(m)
        assert blk.shape == (3, 12) and blk[sh.n_local:].nnz == 0
        id_of_pos = np.full(12, -1)
        id_of_pos[sh.pos_of_id] = np.arange(10)
        coo = blk.tocoo()
        for i, j, v in zip(coo.row, coo.col, coo.data):
            back[sh.my_ids[i], id_of_pos[j]] = v
        assert (sh.cols_of(m)[:, :sh.n_local] != m[:, sh.my_ids]).nnz == 0
        x = np.arange(20.0).reshape(10, 2)
        assert np.array_equal(sh.local_rows(x)[:sh.n_local], x[sh.my_ids])
    assert abs(back.tocsr() - m).max() < 1e-12
    sh = pg.RowShard(4, rank=0, world_size=2)
    dup = sp.csr_matrix((np.array([1.0, 2.0, 5.0]), np.array([1, 1, 3]), np.array([0, 2, 2, 3, 3])), shape=(4, 4))
    assert sh.square_rows_of(dup, keep_duplicates=True).nnz == 3 and sh.square_rows_of(dup).nnz == 2
    gathered = torch.arange(4.0)[:, None]                       # position order of ids 0, 2, 1, 3
    assert sh.to_global(gathered[[0, 1, 2, 3]]).flatten().tolist() == [0.0, 2.0, 1.0, 3.0]
    deg = 1000.0 / (1 + np.arange(1000))                        # Zipf degrees in id (= frequency) order
    load = [deg[pg.RowShard(1000, r, 4).my_ids].sum() for r in range(4)]
    assert max(load) / min(load) < 1.7                          # contiguous blocks would give rank 0 over 5x rank 3


# ---- AliNet: row-sharded model vs the single-process model (same forward code, torch stand-ins for the kernels) ----------
def _alinet_standins(model):
    from oracle.gnn import edge_softmax_aggregate
    model.spmm_fn = lambda X, A: torch.sparse.mm(A.t, X)
    model.gat_fn = lambda s1, s2, M, A, slope: edge_softmax_aggregate(A.m, s1, s2, M, slope)


def _alinet_problem():
    rng = np.random.default_rng(11)
    n = 47
    a1 = sp.random(n, n, density=0.1, random_state=1, format="csr", dtype=np.float32) + sp.eye(n, dtype=np.float32)
    a2 = sp.random(n, n, density=0.15, random_state=2, format="csr", dtype=np.float32) + sp.eye(n, dtype=np.float32)
    a2.data[:] = 1.0
    pos = np.stack([rng.permutation(n)[:9], rng.permutation(n)[:9]], 1)
    neg = np.stack([rng.integers(0, n, 40), rng.integers(0, n, 40)], 1)
    return n, [8, 8, 4], sp.csr_matrix(a1), sp.csr_matrix(a2), torch.as_tensor(pos), torch.as_tensor(neg)


def _alinet_worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from openea_b200 import parallel_gnn as pg
        from openea_b200.approaches.alinet import AliNetModel
        n, dims, a1, a2, pos, neg = _alinet_problem()
        ops = TorchOps()
        ref = AliNetModel(n, dims, ops.csr(a1, "cpu"), ops.csr(a2, "cpu"), torch.device("cpu"), seed=3)
        _alinet_standins(ref)
        ref_outs = ref.forward()
        ref_loss = ref.loss(ref_outs, pos, neg, 1.5, 0.1)
        ref_loss.backward()

        shard = pg.RowShard(n)
        model = pg.ShardedAliNetModel(n, dims, a1, a2, torch.device("cpu"), seed=3, shard=shard, ops=ops)
        _alinet_standins(model)
        assert model.params["init_embedding"].shape[0] == shard.block
        outs = model.forward()
        for o, r in zip(outs, ref_outs):
            assert o.shape == r.shape
            torch.testing.assert_close(o, r, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(model.input_embedding(), ref.params["init_embedding"])
        loss = model.loss(outs, pos, neg, 1.5, 0.1)          # replicated consumer: the same value on every rank
        torch.testing.assert_close(loss, ref_loss, rtol=1e-5, atol=1e-6)
        loss.backward()
        model.sync_grads()
        for name, p in model.params.items():
            want = ref.params[name].grad
            if name == "init_embedding":
                want = torch.as_tensor(shard.local_rows(want.numpy()))
            assert p.grad is not None, name
            torch.testing.assert_close(p.grad, want, rtol=1e-4, atol=1e-6, msg=lambda m, name=name: "%s: %s" % (name, m))
        out.put((rank, "ok"))
    except Exception as e:  # surface the failure in the parent
        import traceback
        out.put((rank, "FAIL: %r\n%s" % (e, traceback.format_exc())))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_alinet_model_equals_single_process_model(world):
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_alinet_worker, args=(r, world, port, out)) for r in range(world)]
    for p in procs:
        p.start()
    res = [out.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(r, "ok") for r in range(world)], res


# ---- RDGCN: row-sharded layer vs the same layer on one process (torch stand-ins for the kernels) ---------------------------
def _edge_logit_aggregate(edge_logits, X, A, slope):
    """EdgeLogitAggregateFn in plain torch: softmax over every row's edges of leaky_relu(logit_e), times X[col e]."""
    m = A.m
    row = torch.as_tensor(np.repeat(np.arange(m.shape[0]), np.diff(m.indptr)), dtype=torch.long)
    col = torch.as_tensor(m.indices, dtype=torch.long)
    logit = torch.nn.functional.leaky_relu(edge_logits, slope)
    mx = torch.full((m.shape[0],), -1e30).scatter_reduce(0, row, logit, "amax")
    ex = torch.exp(logit - mx[row])
    den = torch.zeros(m.shape[0]).index_add(0, row, ex)
    return torch.zeros(m.shape[0], X.shape[1]).index_add(0, row, (ex / den[row])[:, None] * X[col])


def _rdgcn_problem():
    from types import SimpleNamespace
    rng = np.random.default_rng(21)
    n, r, d, t, k = 41, 5, 8, 7, 3
    tri = np.unique(np.stack([rng.integers(0, n, 150), rng.integers(0, r, 150), rng.integers(0, n, 150)], 1), axis=0)
    half = len(tri) // 2
    kgs = SimpleNamespace(kg1=SimpleNamespace(relation_triples_list=[tuple(x) for x in tri[:half].tolist()]),
                          kg2=SimpleNamespace(relation_triples_list=[tuple(x) for x in tri[half:].tolist()]),
                          entities_num=n, relations_num=r,
                          train_links=[(int(a), int(b)) for a, b in zip(rng.permutation(n)[:t], rng.permutation(n)[:t])])
    args = SimpleNamespace(dim=d, alpha=0.1, beta=0.3, gamma=1.0, neg_triple_num=k)
    emb = rng.standard_normal((n, d)).astype(np.float32)
    ill = np.array(kgs.train_links)
    negs = [np.repeat(ill[:, 0], k), rng.integers(0, n, t * k), rng.integers(0, n, t * k), np.repeat(ill[:, 1], k)]
    return args, kgs, emb, ill, negs, k


def _rdgcn_worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from openea_b200 import parallel_gnn as pg
        from oracle.gnn import align_loss
        args, kgs, emb, ill, negs, k = _rdgcn_problem()
        ops = TorchOps()

        def build(shard):
            layer = pg.ShardedRDGCNLayer(args, kgs, emb, torch.device("cpu"), seed=5, shard=shard, ops=ops)
            layer.spmm_fn = lambda X, A: torch.sparse.mm(A.t, X)
            layer.edge_fn = _edge_logit_aggregate
            for name, p in layer.params.items():              # the reference initialises the gates / biases at zero:
                if name.endswith(".b"):                       # perturb them so that their gradients are exercised too
                    with torch.no_grad():
                        p += 0.1 * torch.randn(p.shape, generator=torch.Generator().manual_seed(len(name)))
            return layer
        ref = build(pg.RowShard(kgs.entities_num, rank=0, world_size=1))
        ref_out = ref.forward()
        ref_loss = align_loss(ref_out, ill, args.gamma, k, *negs)
        ref_loss.backward()

        shard = pg.RowShard(kgs.entities_num)
        layer = build(shard)
        assert layer.params["X0"].shape[0] == shard.block and tuple(layer.r_mat.shape) == (shard.block, shard.n_pad)
        n_edges = torch.tensor([layer.r_mat.nnz])
        dist.all_reduce(n_edges)
        assert int(n_edges) == ref.r_mat.nnz                  # every triple's r_mat entry lives on exactly one rank
        out_full = layer.forward()
        torch.testing.assert_close(out_full, ref_out, rtol=1e-4, atol=1e-5)
        loss = align_loss(out_full, ill, args.gamma, k, *negs)
        torch.testing.assert_close(loss, ref_loss, rtol=1e-5, atol=1e-6)
        loss.backward()
        layer.sync_grads()
        for name, p in layer.params.items():
            want = ref.params[name].grad
            assert p.grad is not None and want is not None, name
            if name == "X0":
                want = torch.as_tensor(shard.local_rows(want.numpy()))
            # (the bias of a 1-filter conv in front of a row softmax has a mathematically zero gradient: only noise)
            atol = max(1e-5 * float(want.abs().max()), 1e-7)
            torch.testing.assert_close(p.grad, want, rtol=1e-3, atol=atol, msg=lambda m, name=name: "%s: %s" % (name, m))
        out.put((rank, "ok"))
    except Exception as e:  # surface the failure in the parent
        import traceback
        out.put((rank, "FAIL: %r\n%s" % (e, traceback.format_exc())))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_rdgcn_layer_equals_single_process_layer(world):
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rdgcn_worker, args=(r, world, port, out)) for r in range(world)]
    for p in procs:
        p.start()
    res = [out.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(r, "ok") for r in range(world)], res


def test_single_gpu_rdgcn_layer_hooks_are_identities():
    """The unsharded RDGCNLayer (identity hooks, gnn.DeviceCsr containers) and the sharded layer on a one-rank partition
    build the same graph data and give the same forward output with the torch stand-ins."""
    from openea_b200 import lib as L
    from openea_b200 import parallel_gnn as pg
    from openea_b200.approaches.rdgcn import RDGCNLayer
    if not os.path.exists(L.LIB_PATH):
        pytest.skip("liboea.so not built (DeviceCsr asks it for the hub-row threshold)")
    args, kgs, emb, ill, negs, k = _rdgcn_problem()

    class _HostCsr(_Csr):                       # DeviceCsr → the stand-in container, from the same scipy matrix
        def __init__(self, dc):
            super().__init__(dc._host)
    base = RDGCNLayer(args, kgs, emb, torch.device("cpu"), seed=5)
    one = pg.ShardedRDGCNLayer(args, kgs, emb, torch.device("cpu"), seed=5, shard=pg.RowShard(kgs.entities_num, 0, 1),
                               ops=TorchOps())
    assert base.r_mat.nnz == one.r_mat.nnz and torch.equal(base.edge_rel, one.edge_rel)
    for name in ("M", "head_avg", "tail_avg", "r_mat"):
        a, b = getattr(base, name)._host, getattr(one, name).m
        assert a.shape == b.shape and abs(a - b).max() < 1e-7, name
        setattr(base, name, _HostCsr(getattr(base, name)))
    for layer in (base, one):
        layer.spmm_fn = lambda X, A: torch.sparse.mm(A.t, X)
        layer.edge_fn = _edge_logit_aggregate
    with torch.no_grad():
        torch.testing.assert_close(base.forward(), one.forward(), rtol=1e-5, atol=1e-6)
