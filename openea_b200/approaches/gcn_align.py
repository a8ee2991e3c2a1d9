"""GCN-Align on the CUDA engine (approaches/gcn_align.py of the reference).

Two independent 2-layer GCNs trained full-batch with SGD (lr = args.learning_rate, 8 in the shipped config):
  SE (structure): layer 1 is featureless, its "weights" are the entity table W0 [N, se_dim], created by
      trunc_normal → ROW-NORMALISED inside the graph every step (gcn_align.py:52-56,530): H1 = relu(A·Ŵ0);
      layer 2 has no weights (transform=False): OUT = A·H1.
  AE (attributes): P = X_attr·Ŵ with X_attr the sparse 0/1 entity×attribute matrix and Ŵ the row-normalised
      [n_attr, ae_dim] matrix; H1 = relu(A·P); OUT = A·H1.
  A = D^-½ (A_w + I)ᵀ D^-½, A_w the functionality-weighted adjacency (gcn_align.py:566-578,642-664).
  loss = L1 margin alignment loss over the seed pairs with k negatives per side (gcn_align.py:298-320).
Every A·X / Aᵀ·dY is oea_spmm_csr; the loss is oea_align_loss_l1; normalisation forward/backward and the
SGD update go through the table kernels of path (i).
"""
import math
import os
import time

import numpy as np
import torch

import openea_b200.modules.load.read as rd
from openea_b200 import gnn
from openea_b200.engine import EmbeddingTable
from openea_b200.models.basic_model import BasicModel
from openea_b200.modules.finding.evaluation import valid, test, early_stop
from openea_b200.modules.utils.util import load_session, merge_dic


class GCNAlignUnit:
    """One GCN_Align_Unit (gcn_align.py:498-539) with explicit forward / backward over liboea kernels."""

    def __init__(self, support, table, features, ill, gamma, k, lr):
        self.A = support                       # DeviceCsr [N, N]
        self.At = support.transpose()
        self.table = table                     # EmbeddingTable (row-normalised lookup, SGD)
        self.X = features                      # DeviceCsr [N, F] or None (featureless)
        self.Xt = features.transpose() if features is not None else None
        dev = table.device
        self.left = torch.as_tensor(ill[:, 0], dtype=torch.int32, device=dev).contiguous()
        self.right = torch.as_tensor(ill[:, 1], dtype=torch.int32, device=dev).contiguous()
        self.gamma, self.k, self.lr = float(gamma), int(k), float(lr)
        self.loss_dev = torch.zeros(1, dtype=torch.float64, device=dev)
        self.outputs = None
        self._h1 = None

    def forward(self):
        wn = self.table.lookup(padded=True)                      # l2_normalize(W, 1), [rows, pitch]
        pre = wn if self.X is None else gnn.spmm(self.X, wn)     # dot(x, W, sparse=True)
        self._h1 = gnn.spmm(self.A, pre, relu=True)              # relu(A · pre)
        self.outputs = gnn.spmm(self.A, self._h1)                # second layer: no weights, identity act
        return self.outputs

    def train_step(self, neg_left, neg_right, neg2_left, neg2_right):
        out = self.forward()
        g_out = torch.zeros_like(out)
        self.loss_dev.zero_()
        gnn.align_loss_l1(out, self.table.dim, self.left, self.right, self.k, neg_left, neg_right, neg2_left,
                          neg2_right, self.gamma, g_out, self.loss_dev)
        g_h1 = gnn.spmm(self.At, g_out, mask_src=self._h1)       # Aᵀ·dOUT, then relu'
        g_pre = gnn.spmm(self.At, g_h1)
        g_w = g_pre if self.X is None else gnn.spmm(self.Xt, g_pre)
        self.table.scatter_grad(g_w)                             # through the row normalisation
        self.table.apply(self.lr)                                # GradientDescentOptimizer
        return self.loss_dev


class GraphedTrainStep:
    """One unit's full-batch train_step (9 kernels + a few memsets, tens of microseconds of device work at the 15K shape) captured
    once as a CUDA graph: an epoch is one graph launch instead of a launch-latency-bound chain.  The four negative-index
    vectors live in static buffers (refreshed in place every 10 epochs); the loss stays on the device."""

    def __init__(self, unit, negs):
        self.unit = unit
        self.static = [n.clone() for n in negs]
        self.graph = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        with torch.cuda.graph(self.graph):
            self.loss = unit.train_step(*self.static)

    def refresh(self, negs):
        for dst, src in zip(self.static, negs):
            dst.copy_(src)

    def step(self):
        self.graph.replay()
        return self.loss


class GCN_Align(BasicModel):

    def __init__(self):
        super().__init__()
        self.attr = None
        self.opt = 'SGD'
        self.dropout = 0.0
        self.vec_ae = self.vec_se = None
        self.model_ae = self.model_se = None
        self.adj = self.support = self.ae_input = self.train = None
        self.e = None

    def init(self):
        assert self.args.alignment_module == 'mapping'
        assert self.args.neg_triple_num > 1
        assert self.args.learning_rate >= 0.01
        assert getattr(self.args, "dropout", 0) == 0, "every shipped config trains without dropout"
        self.session = load_session()
        dev = self.session.device
        n = self.kgs.entities_num
        self.e = n
        ent_attrs = merge_dic(self.kgs.kg1.entity_attributes_dict, self.kgs.kg2.entity_attributes_dict)
        self.attr = gnn.attribute_features(n, ent_attrs)
        triples = self.kgs.kg1.relation_triples_list + self.kgs.kg2.relation_triples_list
        self.adj = gnn.weighted_adjacency(n, triples)
        self.support = gnn.DeviceCsr(gnn.preprocess_adj(self.adj), dev)
        self.ae_input = gnn.DeviceCsr(self.attr, dev)
        self.train = np.array(self.kgs.train_links)
        g = torch.Generator().manual_seed(getattr(self.args, "seed", 0) or 0)

        def trunc_normal(shape):  # stddev = 1/√shape[0] (gcn_align.py:52-56)
            std = 1.0 / math.sqrt(shape[0])
            return torch.nn.init.trunc_normal_(torch.empty(*shape), std=std, a=-2 * std, b=2 * std, generator=g)
        ae_init, se_init = trunc_normal([self.attr.shape[1], self.args.ae_dim]), trunc_normal([n, self.args.se_dim])
        unit_args = (self.train, self.args.gamma, self.args.neg_triple_num, self.args.learning_rate)
        from openea_b200 import parallel as par
        if par.world()[1] > 1:
            # one process per GPU (torchrun): adjacency, layer outputs and the SE entity table are row-sharded, one
            # exchange per layer (openea_b200/parallel_gnn.py); every rank seeds the same generator, so the shards are
            # slices of the single-GPU initialisation
            from openea_b200 import parallel_gnn as pg
            shard = pg.RowShard(n)
            par.mark_replicas_in_sync()        # every rank holds the same outputs: the evaluation may be sharded
            norm_adj = gnn.preprocess_adj(self.adj)
            self.model_ae = pg.ShardedGCNAlignUnit(norm_adj, EmbeddingTable(ae_init, True, "SGD", dev), self.attr,
                                                   *unit_args, shard=shard)
            self.model_se = pg.ShardedGCNAlignUnit(norm_adj, EmbeddingTable(shard.local_rows(se_init.numpy()), True,
                                                                            "SGD", dev), None, *unit_args, shard=shard)
            return
        self.model_ae = GCNAlignUnit(self.support, EmbeddingTable(ae_init, True, "SGD", dev), self.ae_input, *unit_args)
        self.model_se = GCNAlignUnit(self.support, EmbeddingTable(se_init, True, "SGD", dev), None, *unit_args)

    def _embeddings(self):
        se = self.model_se.outputs[:, :self.args.se_dim]
        if self.args.test_method == "sa":
            ae = self.model_ae.outputs[:, :self.args.ae_dim]
            beta = self.args.beta
            return torch.cat([se * beta, ae * (1.0 - beta)], dim=1)
        return se

    def train_embeddings(self, loss=None, optimizer=None, output=None):
        neg_num = self.args.neg_triple_num
        train_num = len(self.kgs.train_links)
        dev = self.session.device
        links = torch.as_tensor(self.train, dtype=torch.int32, device=dev)
        neg_left = links[:, 0].repeat_interleave(neg_num).contiguous()       # fixed left, random right
        neg2_right = links[:, 1].repeat_interleave(neg_num).contiguous()     # random left, fixed right
        neg2_left = neg_right = None
        single = not (torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1)
        use_graphs = single and dev.type == "cuda" and os.environ.get("OEA_GNN_GRAPH", "1") != "0" and \
            isinstance(self.model_se, GCNAlignUnit) and isinstance(self.model_ae, GCNAlignUnit)
        graphs = None
        for i in range(1, self.args.max_epoch + 1):
            start = time.time()
            if i % 10 == 1:   # uniform negatives over all entities, refreshed every 10 epochs (gcn_align.py:753-755)
                neg2_left = torch.as_tensor(np.random.choice(self.e, train_num * neg_num), dtype=torch.int32, device=dev)
                neg_right = torch.as_tensor(np.random.choice(self.e, train_num * neg_num), dtype=torch.int32, device=dev)
                if torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1:
                    for neg in (neg2_left, neg_right):     # the sharded units need the same negatives on every rank
                        torch.distributed.broadcast(neg, src=0)
            negs = (neg_left, neg_right, neg2_left, neg2_right)
            if graphs is not None:
                if i % 10 == 1:
                    for gr in graphs:
                        gr.refresh(negs)
                l1, l2 = graphs[0].step(), graphs[1].step()
            else:
                l1 = self.model_ae.train_step(*negs)
                l2 = self.model_se.train_step(*negs)
                if use_graphs and i == 1:      # epoch 1 ran eagerly (it is also the warm-up); the rest replay two graphs
                    graphs = (GraphedTrainStep(self.model_ae, negs), GraphedTrainStep(self.model_se, negs))
            batch_loss = float((l1 + l2).item())
            print('epoch {}, avg. relation triple loss: {:.4f}, cost time: {:.4f}s'.format(i, batch_loss,
                                                                                           time.time() - start))
            if i >= self.args.start_valid and i % self.args.eval_freq == 0:
                flag = self.valid_(self.args.stop_metric)
                self.flag1, self.flag2, self.early_stop = early_stop(self.flag1, self.flag2, flag)
                if self.early_stop or i == self.args.max_epoch:
                    break
        self.model_se.forward()
        self.model_ae.forward()
        self.vec_se = self.model_se.outputs[:, :self.args.se_dim].cpu().numpy()
        self.vec_ae = self.model_ae.outputs[:, :self.args.ae_dim].cpu().numpy()
        return self.vec_se, self.vec_ae

    def _rows(self, emb, ids):
        return emb[torch.as_tensor(ids, dtype=torch.long, device=emb.device)].contiguous()

    def test(self, save=True):
        emb = self._embeddings()
        embeds1, embeds2 = self._rows(emb, self.kgs.test_entities1), self._rows(emb, self.kgs.test_entities2)
        rest_12, _, _ = test(embeds1, embeds2, None, self.args.top_k, self.args.test_threads_num,
                             metric=self.args.eval_metric, normalize=self.args.eval_norm, csls_k=0, accurate=True)
        test(embeds1, embeds2, None, self.args.top_k, self.args.test_threads_num,
             metric=self.args.eval_metric, normalize=self.args.eval_norm, csls_k=self.args.csls, accurate=True)
        if save:
            ent_ids_rest_12 = [(self.kgs.test_entities1[i], self.kgs.test_entities2[j]) for i, j in rest_12]
            rd.save_results(self.out_folder, ent_ids_rest_12)

    def save(self):
        rd.save_embeddings(self.out_folder, self.kgs, self.vec_se, None, self.vec_ae, mapping_mat=None)

    def valid_(self, stop_metric):
        self.model_se.forward()
        if self.args.test_method == "sa":
            self.model_ae.forward()
        emb = self._embeddings()
        embeds1 = self._rows(emb, self.kgs.valid_entities1)
        embeds2 = self._rows(emb, self.kgs.valid_entities2 + self.kgs.test_entities2)
        hits1_12, mrr_12 = valid(embeds1, embeds2, None, self.args.top_k, self.args.test_threads_num,
                                 metric=self.args.eval_metric)
        return hits1_12 if stop_metric == 'hits1' else mrr_12

    def run(self):
        t = time.time()
        self.train_embeddings()
        print("Training ends. Total time = {:.3f} s.".format(time.time() - t))
