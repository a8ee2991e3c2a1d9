"""AliNet on the CUDA engine (approaches/alinet.py of the reference): gated multi-hop neighbourhood aggregation.

Per layer i (dims layer_dims[i] → layer_dims[i+1]):
    one-hop   BN → X·W → A₁·(XW) + b → tanh                        (GraphConvolution.call, alinet.py:574-590)
    two-hop   BN → M = X·K ; s1 = tanh(rowsum((X·K₁)∘X)), s2 likewise ; edge softmax over the 2-hop adjacency of
              leaky_relu(a_ij(s1_i + s2_j)) ; tanh(Σ_j α_ij M_j)     (AliNetGraphAttentionLayer.call, :656-677)
    gate      g = relu(tanh(BN(two)·W_g)) ; tanh(BN(one)·(1 − g) + BN(two)·g)   (HighwayLayer.call, :613-622)
    (the last layer is one-hop only).  BatchNormalization runs in inference mode in the reference's TF1 graph
    (no `training=` argument): y = γ·x/√(1+1e-3) + β with trainable γ, β.
Loss = Σ‖e1−e2‖² + 0.1·Σ relu(1.5 − ‖n1−n2‖²) on the l2-normalised concatenation [layers…, input] (compute_loss,
:828-850) + rel_param · relation loss (compute_rel_loss, :852-866); Adam (TF form), full graph per step.

What runs where: every sparse aggregation (A·X, its transpose in the backward, the edge softmax, the SDDMM) is a
liboea.so kernel wrapped in torch.autograd.Function (openea_b200/gnn.py); the dense X·W products are cuBLAS GEMMs
through torch.matmul and the surrounding element-wise glue is ordinary torch autograd; validation / test / the
ε-truncated cross-KG neighbour search use the K3 kernels; Adam is the engine's dense row optimiser.
"""
import math
import os
import pickle
import random
import time

import numpy as np
import scipy.sparse as sp
import scipy.special
import torch

import openea_b200.modules.load.read as rd
from openea_b200 import finding as F
from openea_b200 import gnn
from openea_b200.models.basic_model import BasicModel
from openea_b200.modules.bootstrapping.alignment_finder import check_new_alignment
from openea_b200.modules.finding.evaluation import early_stop
from openea_b200.modules.utils.util import generate_out_folder, load_session

BN_EPS = 1e-3          # tf.keras.layers.BatchNormalization default epsilon
LEAKY_SLOPE = 0.2      # tf.nn.leaky_relu default alpha


# ---- graph construction (host, one-off) ------------------------------------------------------------------
class AKG:
    """Triple container with the lookups AliNet's builders use (alinet.py:456-536)."""

    def __init__(self, triples, ori_triples=None):
        self.triples = set(triples)
        self.triple_list = list(self.triples)
        self.triples_num = len(self.triples)
        self.heads = {h for h, _, _ in self.triple_list}
        self.props = {r for _, r, _ in self.triple_list}
        self.tails = {t for _, _, t in self.triple_list}
        self.ents = self.heads | self.tails
        print("triples num", self.triples_num)
        print("head ent num", len(self.heads))
        print("total ent num", len(self.ents))
        self.prop_list = sorted(self.props)
        self.ent_list = sorted(self.ents)
        self.ori_triples = None if ori_triples is None else set(ori_triples)
        self.out_related_ents_dict, self.in_related_ents_dict = {}, {}
        self.rt_dict, self.hr_dict = {}, {}
        for h, r, t in self.triple_list:
            self.out_related_ents_dict.setdefault(h, set()).add(t)
            self.in_related_ents_dict.setdefault(t, set()).add(h)
            self.rt_dict.setdefault(h, set()).add((r, t))
            self.hr_dict.setdefault(t, set()).add((h, r))
        self.ht = {(h, t) for h, _, t in self.triples}


def remove_unlinked_triples(triples, linked_ents):
    print("before removing unlinked triples:", len(triples))
    kept = {(h, r, t) for h, r, t in triples if h in linked_ents and t in linked_ents}
    print("after removing unlinked triples:", len(kept))
    return list(kept)


def generate_rel_ht(triples):
    rel_ht = {}
    for h, r, t in triples:
        rel_ht.setdefault(r, []).append((h, t))
    return rel_ht


def enhance_triples(kg1, kg2, ents1, ents2):
    """Project every triple between two seed-linked entities into the other KG unless the edge already exists there."""
    assert len(ents1) == len(ents2)
    print("before enhanced:", len(kg1.triples), len(kg2.triples))
    to2, to1 = dict(zip(ents1, ents2)), dict(zip(ents2, ents1))
    new2 = {(to2[h], r, to2[t]) for h, r, t in kg1.triples
            if h in to2 and t in to2 and to2[t] not in kg2.out_related_ents_dict.get(to2[h], set())}
    new1 = {(to1[h], r, to1[t]) for h, r, t in kg2.triples
            if h in to1 and t in to1 and to1[t] not in kg1.out_related_ents_dict.get(to1[h], set())}
    print("after enhanced:", len(new1), len(new2))
    return new1, new2


def normalize_adj(adj):
    return gnn.normalize_adj(adj)


def no_weighted_adj(total_ent_num, triple_list, is_two_adj=False):
    """Symmetric 0/1 neighbour matrix of the triples (both directions, de-duplicated), then D^-½(A+I)ᵀD^-½
    (alinet.py:155-178).  Returns (scipy COO, None)."""
    start = time.time()
    tri = np.asarray([(h, t) for h, _, t in triple_list], dtype=np.int64).reshape(-1, 2)
    rows = np.concatenate([tri[:, 0], tri[:, 1]])
    cols = np.concatenate([tri[:, 1], tri[:, 0]])
    m = sp.coo_matrix((np.ones(rows.size), (rows, cols)), shape=(total_ent_num, total_ent_num)).tocsr()
    m.data[:] = 1.0                      # a set of neighbours per node: multi-edges count once
    one_adj = gnn.normalize_adj(m + sp.eye(total_ent_num))
    print('generating one-adj costs time: {:.4f}s'.format(time.time() - start))
    return one_adj, None


def generate_2hop_triples(kg, linked_ents=None):
    """(h, r_x, r_y, t) paths h→m→t with t not already a 1-hop out-neighbour of h nor h an in-neighbour of t; the 5
    most frequent relation-pair patterns are skipped; kept paths contribute (h, r_x+r_y, t) and a self loop (h, 0, h)
    (alinet.py:250-287)."""
    triples = kg.triples
    if linked_ents is not None:
        triples = remove_unlinked_triples(triples, linked_ents)
    by_head = {}
    for h, r, t in triples:
        by_head.setdefault(h, []).append((r, t))
    quads, patterns = set(), {}
    for h, rx, m in triples:
        for ry, t in by_head.get(m, ()):
            if t not in kg.out_related_ents_dict.get(h, set()) and h not in kg.in_related_ents_dict.get(t, set()):
                patterns[(rx, ry)] = patterns.get((rx, ry), 0) + 1     # counted per joined row, as iterrows() does
                quads.add((h, rx, ry, t))
    print("total 2-hop neighbors:", len(quads))
    print("total 2-hop relation patterns:", len(patterns))
    ranked = sorted(patterns.items(), key=lambda kv: kv[1], reverse=True)
    selected = {p for p, _ in ranked[5:]}
    print("selected relation patterns:", len(selected))
    out = set()
    for h, rx, ry, t in quads:
        if (rx, ry) in selected:
            out.add((h, 0, h))
            out.add((h, rx + ry, t))
    print("selected 2-hop neighbors:", len(out))
    return out


def update_labeled_alignment_x(pre_labeled_alignment, curr_labeled_alignment, sim_mat):
    labeled = dict(pre_labeled_alignment)
    n1 = n2 = 0
    for i, j in curr_labeled_alignment:
        if labeled.get(i, -1) == i and j != i:
            n2 += 1
        if i in labeled:
            pre_j = labeled[i]
            if sim_mat[i, j] >= sim_mat[i, pre_j]:
                if pre_j == i and j != i:
                    n1 += 1
                labeled[i] = j
        else:
            labeled[i] = j
    print("update wrongly: ", n1, "greedy update wrongly: ", n2)
    out = set(labeled.items())
    check_new_alignment(out, context="after editing (<-)")
    return out


def update_labeled_alignment_y(labeled_alignment, sim_mat):
    by_j = {}
    for i, j in labeled_alignment:
        by_j.setdefault(j, set()).add(i)
    out = set()
    for j, claim in by_j.items():
        best_i, best = -1, -10
        for i in claim:
            if len(claim) == 1 or sim_mat[i, j] > best:
                best, best_i = sim_mat[i, j], i
        out.add((best_i, j))
    check_new_alignment(out, context="after editing (->)")
    return out


# ---- the model -----------------------------------------------------------------------------------------------
def _glorot(shape, gen):
    lim = math.sqrt(6.0 / (shape[0] + shape[1]))
    return (torch.rand(*shape, generator=gen) * 2 - 1) * lim


def _bn(x, gamma, beta):
    return x * (gamma / math.sqrt(1.0 + BN_EPS)) + beta


def _l2n(x):
    return x * torch.rsqrt(torch.clamp((x * x).sum(1, keepdim=True), min=1e-12))


class AliNetModel:
    """Parameters + forward of the AliNet graph (alinet.py:784-826).  `adj1` / `adj2` are gnn.DeviceCsr."""

    def __init__(self, n_ent, layer_dims, adj1, adj2, device, seed=0):
        gen = torch.Generator().manual_seed(seed)
        self.adj1, self.adj2 = adj1, adj2
        self.dims = list(layer_dims)
        p = {}
        p["init_embedding"] = _glorot((n_ent, self.dims[0]), gen)
        n_layers = len(self.dims) - 1
        for i in range(n_layers):
            di, do = self.dims[i], self.dims[i + 1]
            p["gcn%d.kernel" % i] = _glorot((di, do), gen)
            p["gcn%d.bias" % i] = torch.zeros(1, do)
            p["gcn%d.bn_gamma" % i], p["gcn%d.bn_beta" % i] = torch.ones(1, di), torch.zeros(1, di)
            if i < n_layers - 1:
                p["gat%d.kernel" % i] = _glorot((di, do), gen)
                p["gat%d.kernel1" % i], p["gat%d.kernel2" % i] = _glorot((di, di), gen), _glorot((di, di), gen)
                p["gat%d.bn_gamma" % i], p["gat%d.bn_beta" % i] = torch.ones(1, di), torch.zeros(1, di)
                p["hw%d.kernel" % i] = _glorot((do, do), gen)
                p["hw%d.bn_gamma" % i], p["hw%d.bn_beta" % i] = torch.ones(1, do), torch.zeros(1, do)
        self.params = {k: v.to(device).requires_grad_(True) for k, v in p.items()}
        self.n_layers = n_layers
        # the two sparse aggregations (liboea kernels with autograd wrappers); the row-sharded model and the gloo test of
        # its collective algebra replace them per instance
        self.spmm_fn, self.gat_fn = gnn.SpmmFn.apply, gnn.GatAggregateFn.apply

    # hooks of the row-sharded variant (openea_b200/parallel_gnn.ShardedAliNetModel): identity on one GPU
    def _layer_input(self, x):
        """What an aggregation reads: all rows of x."""
        return x

    def _layer_outputs(self, outs):
        return outs

    def input_embedding(self):
        """All rows of the input embedding table."""
        return self.params["init_embedding"]

    def set_adj1(self, mat, device):
        self.adj1 = gnn.DeviceCsr(mat, device)

    def forward(self):
        """Returns [layer outputs…] (alinet.py:784-826)."""
        P = self.params
        x = P["init_embedding"]
        outs = []
        for i in range(self.n_layers):
            xb = _bn(x, P["gcn%d.bn_gamma" % i], P["gcn%d.bn_beta" % i])
            one = torch.tanh(self.spmm_fn(self._layer_input(gnn.dense_matmul(xb, P["gcn%d.kernel" % i])), self.adj1) + P["gcn%d.bias" % i])
            if i < self.n_layers - 1:
                xg = _bn(x, P["gat%d.bn_gamma" % i], P["gat%d.bn_beta" % i])
                mapped = gnn.dense_matmul(xg, P["gat%d.kernel" % i])
                s1 = torch.tanh((gnn.dense_matmul(xg, P["gat%d.kernel1" % i]) * xg).sum(1))
                s2 = torch.tanh((gnn.dense_matmul(xg, P["gat%d.kernel2" % i]) * xg).sum(1))
                two = torch.tanh(self.gat_fn(s1, self._layer_input(s2[:, None])[:, 0], self._layer_input(mapped),
                                             self.adj2, LEAKY_SLOPE))
                g_in1 = _bn(two, P["hw%d.bn_gamma" % i], P["hw%d.bn_beta" % i])   # one BN object serves both inputs
                g_in2 = _bn(one, P["hw%d.bn_gamma" % i], P["hw%d.bn_beta" % i])
                gate = torch.relu(torch.tanh(gnn.dense_matmul(g_in1, P["hw%d.kernel" % i])))
                x = torch.tanh(g_in2 * (1 - gate) + g_in1 * gate)
            else:
                x = one
            outs.append(x)
        return self._layer_outputs(outs)

    def concat_embeds(self, outs):
        """l2-normalised concatenation of every layer's l2-normalised output + the input embedding (:832-837)."""
        return _l2n(torch.cat([_l2n(o) for o in outs + [self.input_embedding()]], dim=1))

    def loss(self, outs, pos_links, neg_links, neg_margin, balance, hs=None, ts=None, rel_win=None, rel_param=0.0):
        emb = self.concat_embeds(outs)
        pos = ((emb[pos_links[:, 0]] - emb[pos_links[:, 1]]) ** 2).sum()
        nd = ((emb[neg_links[:, 0]] - emb[neg_links[:, 1]]) ** 2).sum(1)
        total = pos + balance * torch.relu(neg_margin - nd).sum()
        if rel_param > 0 and hs is not None and len(hs) > 0:
            diff = emb[hs] - emb[ts]                                            # compute_rel_loss, :852-866
            r = _l2n(diff.reshape(-1, rel_win, emb.shape[1]).mean(1, keepdim=True).expand(-1, rel_win, -1)
                     .reshape(-1, emb.shape[1]))
            total = total + rel_param * ((diff - r) ** 2).sum()
        return total


class DenseAdam:
    """tf.train.AdamOptimizer over dense parameters through the engine's row optimiser (TF form: ε outside the
    bias correction).  Parameters are [rows, cols] tensors with cols % 4 == 0."""

    def __init__(self, params, lr):
        import ctypes as C
        from openea_b200 import lib as L
        self.C, self.L = C, L
        self.lib = L.load()
        self.lr, self.t = float(lr), 0
        self.items = []
        for p in params:
            assert p.dim() == 2 and p.shape[1] % 4 == 0 and p.is_contiguous(), "dense Adam needs [rows, 4k] parameters"
            m, v = torch.zeros_like(p), torch.zeros_like(p)
            touched = torch.zeros(p.shape[0], dtype=torch.int32, device=p.device)
            self.items.append((p, m, v, touched))

    def step(self):
        from openea_b200.engine import _stream_ptr
        C, L = self.C, self.L
        self.t += 1
        cfg = L.OptCfg(L.OPT_ADAM, self.lr, 0.9, 0.999, 1e-8, self.t)
        for p, m, v, touched in self.items:
            g = p.grad if p.grad is not None else torch.zeros_like(p)
            tab = L.Table(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), touched.data_ptr(), p.shape[0],
                          p.shape[1], p.shape[1], 0)
            L.check(self.lib.oea_rowopt_apply(C.byref(tab), C.byref(cfg), _stream_ptr()), "oea_rowopt_apply")
            p.grad = None          # the kernel zeroed the buffer; drop it so autograd allocates a fresh one


class NeighborTable:
    """ε-truncated candidate lists as one device matrix: row_of[entity] → row of `ids` [n_keys, num] (−1: no list).
    `table[entity]` still gives the Python list the reference's dict gave (alinet.py:1019-1039)."""

    def __init__(self, keys, ids, n_ent):
        self.ids = ids                                               # [n_keys, num] entity ids, on the device
        self.row_of = torch.full((n_ent,), -1, dtype=torch.long, device=ids.device)
        self.row_of[torch.as_tensor(keys, dtype=torch.long, device=ids.device)] = torch.arange(len(keys), device=ids.device)

    def __getitem__(self, entity):
        return self.ids[self.row_of[entity]].tolist()

    def rows(self, entities):
        return self.ids[self.row_of[entities]]


def sample_negative_links(pos_links, neighbors1, neighbors2, pools, k, excluded_keys, n_ent, gen):
    """generate_input_batch's negative links (alinet.py:983-1006) as tensor ops on the links' device.
    truncated (neighbour tables given): for every positive (e1, e2), k DISTINCT candidates c of e1 give (e1, c) and k
    of e2 give (c, e2) (random.sample without replacement = the k largest of `num` random keys per row);
    uniform: k rounds of batch_size distinct entities from each pool, zipped.
    The result is a set: distinct pairs minus the known links (`excluded_keys`, sorted packed keys i·n_ent + j),
    returned sorted like np.array(sorted(neg))."""
    dev = pos_links.device
    b = pos_links.shape[0]
    if neighbors1 is not None:
        def side(table, anchors):
            cand = table.rows(anchors)                                                   # [b, num]
            pick = torch.rand(cand.shape, device=dev, generator=gen).topk(k, dim=1).indices
            return cand.gather(1, pick)                                                  # [b, k] distinct per row
        c1, c2 = side(neighbors1, pos_links[:, 0]), side(neighbors2, pos_links[:, 1])
        left = torch.cat([pos_links[:, :1].expand(b, k).reshape(-1), c2.reshape(-1)])
        right = torch.cat([c1.reshape(-1), pos_links[:, 1:].expand(b, k).reshape(-1)])
    else:
        pool1, pool2 = pools
        draw = lambda pool: torch.cat([pool[torch.randperm(pool.numel(), device=dev, generator=gen)[:b]] for _ in range(k)])
        left, right = draw(pool1), draw(pool2)
    keys = torch.unique(left.long() * n_ent + right.long())                              # sorted, distinct
    if excluded_keys.numel():
        pos = torch.searchsorted(excluded_keys, keys).clamp(max=excluded_keys.numel() - 1)
        keys = keys[excluded_keys[pos] != keys]
    return torch.stack([keys // n_ent, keys % n_ent], 1)


class AliNet(BasicModel):

    def __init__(self):
        super().__init__()
        self.adj = None
        self.new_edges1, self.new_edges2 = set(), set()
        self.new_links = set()
        self.sup_links_set = set()
        self.new_sup_links_set = set()
        self.rel_ht_dict = None
        self.rel_win_size = None
        self.is_two = True
        self.model = None
        self.optimizer = None
        self._outs = None

    def set_kgs(self, kgs):
        self.kgs = kgs
        self._tri1 = getattr(kgs.kg1, "relation_triples_array", None)      # array-backed loader: build graphs on arrays
        self._tri2 = getattr(kgs.kg2, "relation_triples_array", None)
        if self._tri1 is None or self._tri2 is None:
            self.kg1 = AKG(self.kgs.kg1.relation_triples_set)
            self.kg2 = AKG(self.kgs.kg2.relation_triples_set)

    def _akgs(self):
        """The set / dict containers of alinet.py:456-536, built only when the neighbourhood augmentation needs them."""
        if getattr(self, "kg1", None) is None:
            self.kg1 = AKG(self.kgs.kg1.relation_triples_set)
            self.kg2 = AKG(self.kgs.kg2.relation_triples_set)
        return self.kg1, self.kg2

    def set_args(self, args):
        self.args = args
        self.out_folder = generate_out_folder(self.args.output, self.args.training_data, self.args.dataset_division,
                                              self.__class__.__name__)

    def init(self):
        assert getattr(self.args, "dropout", 0.0) == 0.0, "every shipped config trains without dropout"
        self.session = load_session()
        dev = self.session.device
        self.ref_ent1 = self.kgs.test_entities1 + self.kgs.valid_entities1
        self.ref_ent2 = self.kgs.test_entities2 + self.kgs.valid_entities2
        self.sup_ent1, self.sup_ent2 = self.kgs.train_entities1, self.kgs.train_entities2
        self.linked_ents = set(self.kgs.train_entities1 + self.kgs.train_entities2 + self.kgs.valid_entities1 +
                               self.kgs.test_entities1 + self.kgs.test_entities2 + self.kgs.valid_entities2)
        saved = self.args.training_data + self.args.dataset_division + 'alinet_saved_data.pkl'
        if self._tri1 is not None:
            # sorted-key joins on the loader's arrays (approaches/alinet_graph.py) instead of the row-by-row walk
            from openea_b200.approaches import alinet_graph as ag
            t0 = time.time()
            one_adj, two_adj, triples = ag.build(self._tri1, self._tri2, self.sup_ent1, self.sup_ent2, self.linked_ents,
                                                 self.kgs.entities_num)
            self.rel_index = ag.relation_index(triples)             # (relations, row pointer, (h, t) pairs by relation)
            self.rel_ht_dict = dict.fromkeys(self.rel_index[0].tolist())   # the keys are what the window size needs
            adj = [one_adj, two_adj]
            print('generating the one- and two-hop adjacencies on arrays costs time: {:.4f}s'.format(time.time() - t0))
        else:
            self.rel_index = None
            enh1, enh2 = enhance_triples(self.kg1, self.kg2, self.sup_ent1, self.sup_ent2)
            triples = remove_unlinked_triples(self.kg1.triple_list + self.kg2.triple_list + list(enh1) + list(enh2),
                                              self.linked_ents)
            self.rel_ht_dict = generate_rel_ht(triples)
            if os.path.exists(saved):
                print('load saved adj data from', saved)
                adj = pickle.load(open(saved, 'rb'))
            else:
                one_adj, _ = no_weighted_adj(self.kgs.entities_num, triples)
                two = generate_2hop_triples(self.kg1, self.linked_ents) | generate_2hop_triples(self.kg2, self.linked_ents)
                two_adj, _ = no_weighted_adj(self.kgs.entities_num, list(two))
                adj = [one_adj, two_adj]
                try:
                    pickle.dump(adj, open(saved, 'wb'))
                    print('save adj data to', saved)
                except OSError:
                    pass
        self.adj = adj
        self.rel_win_size = self.args.batch_size // max(1, len(self.rel_ht_dict))
        if self.rel_win_size <= 1:
            self.rel_win_size = self.args.min_rel_win
        self.sim_th = self.args.sim_th
        self.sup_links = np.stack([np.array(self.sup_ent1), np.array(self.sup_ent2)], 1)
        self.sup_links_set = set(zip(self.sup_ent1, self.sup_ent2))
        seed = getattr(self.args, "seed", 0) or 0
        from openea_b200 import parallel as par
        if par.world()[1] > 1:
            # one process per GPU (torchrun): rows of both adjacencies, of every layer and of the input embedding table
            # are sharded (openea_b200/parallel_gnn.py); batches must be identical on every rank
            from openea_b200 import parallel_gnn as pg
            random.seed(seed)
            par.mark_replicas_in_sync()        # every rank holds the same outputs: the evaluation may be sharded
            np.random.seed(seed)
            self.model = pg.ShardedAliNetModel(self.kgs.entities_num, self.args.layer_dims, adj[0], adj[1], dev, seed=seed)
        else:
            self.model = AliNetModel(self.kgs.entities_num, self.args.layer_dims, gnn.DeviceCsr(adj[0], dev),
                                     gnn.DeviceCsr(adj[1], dev), dev, seed=seed)
        self.optimizer = DenseAdam(list(self.model.params.values()), self.args.learning_rate)

    # ---- batches (alinet.py:983-1017) ----
    def _batch_state(self):
        """Device-side constants of the batch generator: the seed links, the two uniform pools, the RNG stream, and the
        sorted keys of the links a negative must not hit (seed links + links found by the augmentation)."""
        dev = self.session.device
        if getattr(self, "_bs", None) is None:
            n = self.kgs.entities_num
            gen = torch.Generator(device=dev)
            gen.manual_seed(getattr(self.args, "seed", 0) or 0)
            self._bs = dict(links=torch.as_tensor(self.sup_links, dtype=torch.long, device=dev), n=n, gen=gen,
                            pools=(torch.as_tensor(self.sup_ent1 + self.ref_ent1, dtype=torch.long, device=dev),
                                   torch.as_tensor(self.sup_ent2 + self.ref_ent2, dtype=torch.long, device=dev)),
                            known=None, known_src=None)
        bs = self._bs
        if bs["known_src"] is not self.new_sup_links_set:          # augment_neighborhood replaces the set object
            known = np.array(sorted(self.sup_links_set | self.new_sup_links_set), dtype=np.int64).reshape(-1, 2)
            bs["known"] = torch.as_tensor(np.sort(known[:, 0] * bs["n"] + known[:, 1]), device=dev)
            bs["known_src"] = self.new_sup_links_set
        return bs

    def generate_input_batch(self, batch_size, neighbors1=None, neighbors2=None):
        batch_size = min(batch_size, len(self.sup_ent1))
        index = np.random.choice(len(self.sup_ent1), batch_size)
        k = self.args.neg_triple_num
        if neighbors1 is None or isinstance(neighbors1, NeighborTable):
            # the whole batch on the device: no Python loop over the positives (alinet.py:983-1006 as tensor ops)
            bs = self._batch_state()
            pos = bs["links"][torch.as_tensor(index, device=bs["links"].device)]
            neg = sample_negative_links(pos, neighbors1, neighbors2, bs["pools"], k, bs["known"], bs["n"], bs["gen"])
            return pos, neg
        pos_links = self.sup_links[index, ]
        if neighbors1 is None:
            pool1, pool2 = self.sup_ent1 + self.ref_ent1, self.sup_ent2 + self.ref_ent2
            neg1, neg2 = [], []
            for _ in range(k):
                neg1.extend(random.sample(pool1, batch_size))
                neg2.extend(random.sample(pool2, batch_size))
            neg = set(zip(neg1, neg2))
        else:
            neg = set()
            for e1, e2 in pos_links.tolist():
                neg.update((e1, c) for c in random.sample(neighbors1[e1], k))
                neg.update((c, e2) for c in random.sample(neighbors2[e2], k))
        neg = neg - self.sup_links_set - self.new_sup_links_set
        return pos_links, np.array(sorted(neg), dtype=np.int64).reshape(-1, 2)

    def generate_rel_batch(self):
        if self.rel_index is not None:     # rel_win_size random (h, t) pairs per relation, with replacement, in one shot
            rels, ptr, pairs = self.rel_index
            size = np.diff(ptr)
            pick = ptr[:-1, None] + (np.random.random((len(rels), self.rel_win_size)) * size[:, None]).astype(np.int64)
            chosen = pairs[pick.reshape(-1)]
            return chosen[:, 0], np.repeat(rels, self.rel_win_size), chosen[:, 1]
        hs, rs, ts = [], [], []
        for r, hts in self.rel_ht_dict.items():
            for h, t in (random.choice(hts) for _ in range(self.rel_win_size)):
                hs.append(h); ts.append(t); rs.append(r)
        return hs, rs, ts

    def find_neighbors(self):
        """Cross-KG ε-truncated candidates from the last layer's output (alinet.py:1019-1039), on the GPU."""
        if self.args.truncated_epsilon <= 0.0:
            return None, None
        start = time.time()
        with torch.no_grad():
            last = self.model.forward()[-1]
        ents1, ents2 = self.sup_ent1 + self.ref_ent1, self.sup_ent2 + self.ref_ent2
        num = int((1 - self.args.truncated_epsilon) * len(ents1))
        print("neighbors num", num)
        e1, _ = F.to_device_rows(last[torch.as_tensor(ents1, device=last.device)], True)
        e2, _ = F.to_device_rows(last[torch.as_tensor(ents2, device=last.device)], True)

        def cross(a, b, ids_b, keys):
            res = F.topk(a, b, last.shape[1], "inner", num, want=("idx",))["idx"] if num <= 32 else None
            if res is None:
                s = F.sim_matrix(a, b, last.shape[1], "inner")
                from openea_b200.modules.bootstrapping.alignment_finder import _topk_of_matrix
                res = _topk_of_matrix(s, num)
            ids = torch.as_tensor(ids_b, dtype=torch.long, device=res.device)[res.long()]
            return NeighborTable(keys, ids, self.kgs.entities_num)
        n1, n2 = cross(e1, e2, ents2, ents1), cross(e2, e1, ents1, ents2)
        print('finding neighbors for sampling costs time: {:.4f}s'.format(time.time() - start))
        return n1, n2

    # ---- evaluation / saving: l2-normalised concatenation [input, layers…] (alinet.py:922-981) ----
    def _concat_rows(self, ids):
        with torch.no_grad():
            outs = self.model.forward()
            parts = [_l2n(_l2n(o)[torch.as_tensor(ids, device=o.device)]) for o in [self.model.input_embedding()] + outs]
        return torch.cat(parts, dim=1)

    def _eval_valid_embeddings(self):
        if len(self.kgs.valid_links) > 0:
            return (self._concat_rows(self.kgs.valid_entities1),
                    self._concat_rows(self.kgs.valid_entities2 + self.kgs.test_entities2), None)
        return self._concat_rows(self.kgs.test_entities1), self._concat_rows(self.kgs.test_entities2), None

    def _eval_test_embeddings(self):
        return self._concat_rows(self.kgs.test_entities1), self._concat_rows(self.kgs.test_entities2), None

    def save(self):
        with torch.no_grad():
            outs = self.model.forward()
            ent = torch.cat([_l2n(o) for o in [self.model.input_embedding()] + outs], dim=1).cpu().numpy()
        rd.save_embeddings(self.out_folder, self.kgs, ent, None, None, mapping_mat=None)

    # ---- neighbourhood augmentation (alinet.py:885-920; disabled by sim_th = 0 in the shipped configs) ----
    def augment_neighborhood(self):
        with torch.no_grad():
            last = self.model.forward()[-1]
        e1 = last[torch.as_tensor(self.ref_ent1, device=last.device)]
        e2 = last[torch.as_tensor(self.ref_ent2, device=last.device)]
        sim_mat = scipy.special.expit(F.sim(e1, e2, "inner", True, self.args.csls).cpu().numpy())
        from openea_b200.modules.bootstrapping.alignment_finder import find_alignment
        pair_index = find_alignment(sim_mat, self.sim_th, 1)
        if not pair_index:
            return
        self.new_links = update_labeled_alignment_x(self.new_links, pair_index, sim_mat)
        self.new_links = update_labeled_alignment_y(self.new_links, sim_mat)
        new1 = [self.ref_ent1[i] for i, _ in self.new_links]
        new2 = [self.ref_ent2[j] for _, j in self.new_links]
        self.new_sup_links_set = set(zip(new1, new2))
        if not new1:
            return
        kg1, kg2 = self._akgs()
        self.new_edges1, self.new_edges2 = enhance_triples(kg1, kg2, self.sup_ent1 + new1, self.sup_ent2 + new2)
        triples = remove_unlinked_triples(kg1.triple_list + kg2.triple_list + list(self.new_edges1) +
                                          list(self.new_edges2), self.linked_ents)
        one_adj, _ = no_weighted_adj(self.kgs.entities_num, triples)
        print("gcn update adj...")
        self.model.set_adj1(one_adj, self.session.device)

    def train_step(self, pos_links, neg_links, hs=None, ts=None):
        dev = self.session.device
        tl = lambda a: a.to(device=dev, dtype=torch.long) if isinstance(a, torch.Tensor) else \
            torch.as_tensor(np.asarray(a), dtype=torch.long, device=dev)
        outs = self.model.forward()
        loss = self.model.loss(outs, tl(pos_links), tl(neg_links), self.args.neg_margin, self.args.neg_margin_balance,
                               None if hs is None else tl(hs), None if ts is None else tl(ts), self.rel_win_size,
                               self.args.rel_param)
        loss.backward()
        if hasattr(self.model, "sync_grads"):        # row-sharded model: partial gradients of the replicated weights
            self.model.sync_grads()
        self.optimizer.step()
        return float(loss.detach().item())

    def run(self):
        flag1 = flag2 = 0
        steps = max(1, len(self.sup_ent2) // self.args.batch_size)
        neighbors1 = neighbors2 = None
        for epoch in range(1, self.args.max_epoch + 1):
            start = time.time()
            epoch_loss = 0.0
            for _ in range(steps):
                pos, neg = self.generate_input_batch(self.args.batch_size, neighbors1, neighbors2)
                hs = ts = None
                if self.args.rel_param > 0:
                    hs, _, ts = self.generate_rel_batch()
                epoch_loss += self.train_step(pos, neg, hs, ts)
            print('epoch {}, loss: {:.4f}, cost time: {:.4f}s'.format(epoch, epoch_loss, time.time() - start))
            if epoch % self.args.eval_freq == 0 and epoch >= self.args.start_valid:
                flag = self.valid(self.args.stop_metric)
                flag1, flag2, is_stop = early_stop(flag1, flag2, flag)
                if is_stop:
                    print("\n == training stop == \n")
                    break
                neighbors1, neighbors2 = self.find_neighbors()
                if epoch >= self.args.start_augment * self.args.eval_freq and self.args.sim_th > 0.0:
                    self.augment_neighborhood()
