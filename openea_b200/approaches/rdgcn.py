"""RDGCN on the CUDA engine (approaches/rdgcn.py of the reference): relation-aware dual-graph convolution.

Graph (Layer.build, rdgcn.py:317-338), X₀ = trainable entity name embeddings [E, d]:
    dual X₁ = [head_rᵀ·X₀/cnt ‖ tail_rᵀ·X₀/cnt]  (compute_r :258-266; the dense [R×E]·[E×d] products of the reference
              are incidence-matrix SpMMs here — same result, ~100× less work)
    dual H₁ = self-attention over relations with the Jaccard adjacency dual_A (add_self_att_layer :233-248)
    primal H₁ = relu(Σ_e softmax_row(leaky_relu(w·dual_H₁[rel e] + b))·X₀[col e])  (add_sparse_att_layer :202-215)
    X₁ = X₀ + α·H₁ ;  dual X₂ from X₁ ; dual H₂ = dual attention (add_dual_att_layer :217-231) ; X₂ = X₀ + β·H₂
    two diag-GCN layers M·(X∘w) with relu + highway gates (:184-191, :250-256) ; L1 margin loss (:293-315) ; Adam.
The normalised adjacency M mirrors the reference's degree computation, including its indexing of the entity-degree
array with the RELATION id (`degree[triple[1]] += 1`, rdgcn.py:49-51).

Sparse work (M·X, incidence aggregation, the per-edge softmax and its backward, the L1 loss, hard-negative search)
runs in liboea.so kernels via autograd wrappers (openea_b200/gnn.py); the R×R relation attention (R ≈ 450) and the
d×d gates are small dense torch ops (cuBLAS); Adam is the engine's dense row optimiser.

The reference initialises X₀ from fastText vectors (`wiki-news-300d-1M.vec`) of entity names, which are not
available offline: pass `args.name_embeds` (path to an [E, d] .npy) or `args.synthetic_names = True` (seeded N(0,1)
vectors, aligned entities share a vector up to noise — the benchmark generator of SURVEY §8d).
"""
import math
import os
import time

import numpy as np
import scipy.sparse as sp
import torch

import openea_b200.modules.load.read as rd
from openea_b200 import finding as F
from openea_b200 import gnn
from openea_b200.approaches.alinet import DenseAdam
from openea_b200.approaches.rdgcn_ops import get_neg as get_neg_device
from openea_b200.models.basic_model import BasicModel
from openea_b200.modules.finding.evaluation import valid, test, early_stop
from openea_b200.modules.utils.util import load_session

LEAKY_SLOPE = 0.2


# ---- graph construction (host; values as the reference computes them) -------------------------------------
def get_mat(triple_list, ent_num):
    """Symmetric position set + the reference's degree vector (rdgcn.py:45-60), relation-id quirk included."""
    degree = np.ones(ent_num, dtype=np.int64)
    tri = np.asarray(triple_list, dtype=np.int64).reshape(-1, 3)
    neq = tri[:, 0] != tri[:, 1]                       # compares head with RELATION id, as the reference does
    np.add.at(degree, tri[neq, 0], 1)
    np.add.at(degree, tri[neq, 1], 1)                  # … and increments degree[relation id]
    keep = tri[:, 0] != tri[:, 2]
    h, t = tri[keep, 0], tri[keep, 2]
    rows = np.concatenate([h, t, np.arange(ent_num)])
    cols = np.concatenate([t, h, np.arange(ent_num)])
    pos = sp.coo_matrix((np.ones(rows.size), (rows, cols)), shape=(ent_num, ent_num)).tocsr()
    pos.data[:] = 1.0
    return pos, degree


def get_sparse_matrix(triple_list, ent_num):
    """M[sec, fir] = 1/√deg[fir]/√deg[sec] over the positions (rdgcn.py:63-72)."""
    pos, degree = get_mat(triple_list, ent_num)
    coo = pos.tocoo()
    fir, sec = coo.row, coo.col
    val = 1.0 / np.sqrt(degree[fir]) / np.sqrt(degree[sec])
    return sp.coo_matrix((val, (sec, fir)), shape=(ent_num, ent_num)).tocsr()


def rfunc(triple_list, ent_num, rel_num):
    """Relation incidence (rdgcn.py:17-42): head/tail entity sets per relation as 0/1 matrices [R, E] and the per-triple
    (h, t) → relation-id matrix r_mat (one entry per triple, duplicates of (h, t) kept)."""
    tri = np.asarray(triple_list, dtype=np.int64).reshape(-1, 3)
    head_r = sp.coo_matrix((np.ones(len(tri)), (tri[:, 1], tri[:, 0])), shape=(rel_num, ent_num)).tocsr()
    tail_r = sp.coo_matrix((np.ones(len(tri)), (tri[:, 1], tri[:, 2])), shape=(rel_num, ent_num)).tocsr()
    head_r.data[:] = 1.0
    tail_r.data[:] = 1.0
    return head_r, tail_r, tri


def dual_adjacency(head_r, tail_r):
    """dual_A[i, j] = Jaccard(heads_i, heads_j) + Jaccard(tails_i, tails_j) (rdgcn.py:268-277), vectorised."""
    out = 0.0
    for m in (head_r, tail_r):
        inter = (m @ m.T).toarray()
        size = np.asarray(m.sum(1)).reshape(-1)
        union = size[:, None] + size[None, :] - inter
        out = out + inter / np.maximum(union, 1e-30)
    return out.astype(np.float32)


def _glorot(shape, gen):
    lim = math.sqrt(6.0 / (shape[0] + shape[1]))
    return (torch.rand(*shape, generator=gen) * 2 - 1) * lim


class RDGCNLayer:
    """Parameters + forward of Layer.build (rdgcn.py:317-338)."""

    def __init__(self, args, kgs, embedding, device, seed=0):
        self.dim = args.dim
        self.alpha, self.beta, self.gamma, self.k = args.alpha, args.beta, args.gamma, args.neg_triple_num
        triples = kgs.kg1.relation_triples_list + kgs.kg2.relation_triples_list
        E, R = kgs.entities_num, kgs.relations_num
        # the sparse aggregations (liboea kernels with autograd wrappers); the row-sharded layer and the gloo test of
        # its collective algebra replace them per instance
        self.spmm_fn, self.edge_fn = gnn.SpmmFn.apply, gnn.EdgeLogitAggregateFn.apply
        self.M = self._entity_rows(get_sparse_matrix(triples, E), device)
        head_r, tail_r, tri = rfunc(triples, E, R)
        norm = lambda m: sp.diags(1.0 / np.maximum(np.asarray(m.sum(1)).reshape(-1), 1e-30)) @ m
        self.head_avg, self.tail_avg = self._entity_cols(norm(head_r), device), self._entity_cols(norm(tail_r), device)
        self.dual_A = torch.from_numpy(dual_adjacency(head_r, tail_r)).to(device)
        self.bias_mat = -1e9 * (1.0 - (self.dual_A > 0).to(torch.float32))
        # r_mat: one entry per triple at (h, t) whose value is the relation id; CSR order gives the edge → relation map
        order = np.lexsort((tri[:, 2], tri[:, 0]))          # CSR built by hand: the COO→CSR conversion would SUM duplicates
        indptr = np.concatenate([[0], np.cumsum(np.bincount(tri[:, 0], minlength=E))])
        rm = sp.csr_matrix((tri[order, 1].astype(np.float64) + 1.0, tri[order, 2], indptr), shape=(E, E))
        self.r_mat = self._entity_rows(rm, device, keep_duplicates=True)
        assert self.r_mat.nnz == len(tri) or self.r_mat.shape[0] != E       # a row block holds its rows' triples only
        self.edge_rel = (self.r_mat.val - 1.0).round().to(torch.long)
        gen = torch.Generator().manual_seed(seed)
        d = self.dim
        p = {"X0": torch.as_tensor(np.asarray(embedding), dtype=torch.float32).clone()}
        p["self.W"] = _glorot((2 * d, d), gen)                       # conv1d(filters=dim, k=1, no bias)
        for name in ("self.f1", "self.f2", "dual.f1", "dual.f2"):
            p[name + ".w"], p[name + ".b"] = _glorot((d, 4), gen)[:, :1].repeat(1, 4), torch.zeros(1, 4)
        p["dual.W"], p["dual.b"] = _glorot((2 * d, d), gen), torch.zeros(1, d)
        for name in ("sp1", "sp2"):                                   # conv1d(1 filter) on dual_H [R, 2d]
            p[name + ".w"], p[name + ".b"] = _glorot((2 * d, 4), gen)[:, :1].repeat(1, 4), torch.zeros(1, 4)
        p["diag1.w"], p["diag2.w"] = torch.ones(1, d), torch.ones(1, d)
        for name in ("hw1", "hw2"):
            p[name + ".W"], p[name + ".b"] = _glorot((d, d), gen), torch.zeros(1, d)
        p["X0"] = self._own_rows(p["X0"])
        self.params = {k_: v.to(device).requires_grad_(True) for k_, v in p.items()}
        ill = np.array(kgs.train_links)
        self.left = torch.as_tensor(ill[:, 0], dtype=torch.int32, device=device).contiguous()
        self.right = torch.as_tensor(ill[:, 1], dtype=torch.int32, device=device).contiguous()

    # ---- hooks of the row-sharded variant (openea_b200/parallel_gnn.ShardedRDGCNLayer): identities on one GPU -------
    def _entity_rows(self, mat, device, keep_duplicates=False):
        """An [E, E] matrix that aggregates INTO entity rows: the rows this process owns."""
        return gnn.DeviceCsr(mat, device, keep_duplicates=keep_duplicates)

    def _entity_cols(self, mat, device):
        """An [R, E] matrix that reduces OVER entity rows: the columns this process owns."""
        return gnn.DeviceCsr(mat, device)

    def _own_rows(self, x):
        return x

    def _all_rows(self, x):
        """What an aggregation into entity rows reads: every entity row of x."""
        return x

    def _sum_over_owners(self, x):
        """Completes a reduction over entity rows of which every process holds a part."""
        return x

    def _full_output(self, x):
        return x

    # column 0 of the [·, 4] vectors is the real 1-filter conv weight (kept 4 wide for the 16-B row optimiser)
    def _vec(self, name):
        return self.params[name + ".w"][:, :1], self.params[name + ".b"][:, :1]

    def _dual_input(self, x):
        return self._sum_over_owners(torch.cat([self.spmm_fn(x, self.head_avg), self.spmm_fn(x, self.tail_avg)], dim=1))

    def _att(self, fts, values, f1, f2):
        w1, b1 = self._vec(f1)
        w2, b2 = self._vec(f2)
        logits = (fts @ w1 + b1) + (fts @ w2 + b2).t()
        coefs = torch.softmax(torch.nn.functional.leaky_relu(self.dual_A * logits, LEAKY_SLOPE) + self.bias_mat, dim=1)
        return torch.relu(coefs @ values)

    def _sparse_att(self, x, dual_h, name):
        w, b = self._vec(name)
        edge_logits = (dual_h @ w + b).reshape(-1)[self.edge_rel]
        return torch.relu(self.edge_fn(edge_logits, self._all_rows(x), self.r_mat, LEAKY_SLOPE))

    def _highway(self, l1, l2, name):
        gate = torch.sigmoid(gnn.dense_matmul(l1, self.params[name + ".W"]) + self.params[name + ".b"])
        return gate * l2 + (1.0 - gate) * l1

    def forward(self):
        P = self.params
        x0 = P["X0"]
        dual_x1 = self._dual_input(x0)
        dual_h1 = self._att(dual_x1 @ P["self.W"], dual_x1, "self.f1", "self.f2")
        x1 = x0 + self.alpha * self._sparse_att(x0, dual_h1, "sp1")
        dual_x2 = self._dual_input(x1)
        dual_h2 = self._att(dual_x2 @ P["dual.W"] + P["dual.b"], dual_h1, "dual.f1", "dual.f2")
        x2 = x0 + self.beta * self._sparse_att(x1, dual_h2, "sp2")
        g1 = self._highway(x2, torch.relu(self.spmm_fn(self._all_rows(x2 * P["diag1.w"]), self.M)), "hw1")
        g2 = torch.relu(self.spmm_fn(self._all_rows(g1 * P["diag2.w"]), self.M))
        return self._full_output(self._highway(g1, g2, "hw2"))

    def loss(self, out, negs):
        return gnn.AlignLossL1Fn.apply(out, self.left, self.right, self.k, negs, self.gamma)


class RDGCN(BasicModel):

    def __init__(self):
        super().__init__()
        self.loss = 0
        self.output = None
        self.optimizer = None
        self.gcn_model = None
        self.local_name_vectors = None
        self.word_embed = '../../datasets/wiki-news-300d-1M.vec'

    def _name_vectors(self):
        path = getattr(self.args, "name_embeds", None)
        if path and os.path.exists(path):
            return np.load(path).astype(np.float32)
        if getattr(self.args, "synthetic_names", False):
            rng = np.random.default_rng(getattr(self.args, "seed", 0) or 0)
            vec = rng.standard_normal((self.kgs.entities_num, self.args.dim)).astype(np.float32)
            noise = getattr(self.args, "synthetic_name_noise", 0.7)
            for a, b in self.kgs.train_links + self.kgs.valid_links + self.kgs.test_links:
                vec[b] = vec[a] + noise * rng.standard_normal(self.args.dim).astype(np.float32)
            return vec
        raise FileNotFoundError(
            "RDGCN needs entity name vectors: the reference reads %s (fastText), which is not shipped; set "
            "args.name_embeds to an [entities, dim] .npy or args.synthetic_names = True" % self.word_embed)

    def init(self):
        assert getattr(self.args, "dropout", 0) == 0, "every shipped config trains without dropout"
        self.session = load_session()
        self.local_name_vectors = self._name_vectors()
        from openea_b200 import parallel as par
        layer_cls = RDGCNLayer
        if par.world()[1] > 1:      # one process per GPU (torchrun): entity rows sharded (openea_b200/parallel_gnn.py)
            from openea_b200 import parallel_gnn as pg
            layer_cls = pg.ShardedRDGCNLayer
            par.mark_replicas_in_sync()        # every rank holds the same outputs: the evaluation may be sharded
        self.gcn_model = layer_cls(self.args, self.kgs, self.local_name_vectors, self.session.device,
                                   seed=getattr(self.args, "seed", 0) or 0)
        self.optimizer = DenseAdam(list(self.gcn_model.params.values()), self.args.learning_rate)

    def _output(self):
        with torch.no_grad():
            return self.gcn_model.forward()

    def _get_neg(self, ids, output, k):
        if k <= 32:
            return get_neg_device(ids, output, k)
        # large k (125 at the 15K scale): distance block + radix select of the k nearest (set semantics)
        emb, d = F.to_device_rows(output, False)
        sub = emb.index_select(0, torch.as_tensor(ids, dtype=torch.long, device=emb.device)).contiguous()
        s = F.sim_matrix(sub, emb, d, "manhattan")
        from openea_b200.modules.bootstrapping.alignment_finder import _topk_of_matrix
        return _topk_of_matrix(s, k).reshape(-1)

    def training(self):
        k = self.args.neg_triple_num
        links = np.array(self.kgs.train_links)
        dev = self.session.device
        neg_left = torch.as_tensor(np.repeat(links[:, 0], k), dtype=torch.int32, device=dev)
        neg2_right = torch.as_tensor(np.repeat(links[:, 1], k), dtype=torch.int32, device=dev)
        negs = None
        for i in range(1, self.args.max_epoch + 1):
            start = time.time()
            if i % 10 == 1:   # hard negatives: the k L1-nearest entities of every seed (rdgcn.py:484-491)
                out = self._output()
                neg2_left = self._get_neg(links[:, 1], out, k).to(torch.int32).contiguous()
                neg_right = self._get_neg(links[:, 0], out, k).to(torch.int32).contiguous()
                negs = (neg_left, neg_right, neg2_left, neg2_right)
            out = self.gcn_model.forward()
            loss = self.gcn_model.loss(out, negs)
            loss.backward()
            if hasattr(self.gcn_model, "sync_grads"):      # row-sharded layer: partial gradients of the replicated weights
                self.gcn_model.sync_grads()
            self.optimizer.step()
            print('epoch {}, avg. relation triple loss: {:.4f}, cost time: {:.4f}s'.format(i, float(loss.detach().item()),
                                                                                           time.time() - start))
            if i >= self.args.start_valid and i % self.args.eval_freq == 0:
                flag = self.valid_(self.args.stop_metric)
                self.flag1, self.flag2, self.early_stop = early_stop(self.flag1, self.flag2, flag)
                if self.early_stop or i == self.args.max_epoch:
                    break

    def _rows(self, emb, ids):
        return emb[torch.as_tensor(ids, dtype=torch.long, device=emb.device)].contiguous()

    def test(self, save=True):
        emb = self._output()
        e1, e2 = self._rows(emb, self.kgs.test_entities1), self._rows(emb, self.kgs.test_entities2)
        rest_12, _, _ = test(e1, e2, None, self.args.top_k, self.args.test_threads_num,
                             metric=self.args.eval_metric, normalize=self.args.eval_norm, csls_k=0, accurate=True)
        test(e1, e2, None, self.args.top_k, self.args.test_threads_num,
             metric=self.args.eval_metric, normalize=self.args.eval_norm, csls_k=self.args.csls, accurate=True)
        if save:
            rd.save_results(self.out_folder, [(self.kgs.test_entities1[i], self.kgs.test_entities2[j]) for i, j in rest_12])

    def save(self):
        rd.save_embeddings(self.out_folder, self.kgs, self._output().cpu().numpy(), None, None, mapping_mat=None)

    def valid_(self, stop_metric):
        emb = self._output()
        e1 = self._rows(emb, self.kgs.valid_entities1)
        e2 = self._rows(emb, self.kgs.valid_entities2 + self.kgs.test_entities2)
        hits1_12, mrr_12 = valid(e1, e2, None, self.args.top_k, self.args.test_threads_num, metric=self.args.eval_metric)
        return hits1_12 if stop_metric == 'hits1' else mrr_12

    def run(self):
        t = time.time()
        self.training()
        print("training finish")
        print("Training ends. Total time = {:.3f} s.".format(time.time() - t))
