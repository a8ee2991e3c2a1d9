"""Attr2Vec on the CUDA engine (approaches/attr2vec.py of the reference): attribute embeddings trained by
tf.nn.nce_loss on the attribute pairs that co-occur on an entity or on its seed-aligned counterpart.

The step is engine.NceTrainer: pairs drawn on the device, TF's unique log-uniform sampler, the sampled-NCE head over
l2-normalised input and class tables (oea_nce_score_fed, reduce_mean) and Adagrad.  Entity vectors are the mean of an
entity's own selected attributes' normalised vectors: a CSR of 1/count weights built once on the host, Y = A·Ê with
oea_spmm_csr, then sklearn's row normalisation (oea_rows_normalize).  Attr2Vec is not a BasicModel; its public surface
is the reference's.
"""
import random
import time

import numpy as np
import scipy.sparse as sp
import torch

from openea_b200 import engine as eng
from openea_b200 import gnn
from openea_b200 import lib as L
from openea_b200 import parallel as par
from openea_b200.approaches.jape import popular_attributes
from openea_b200.modules.base.initializers import xavier_init
from openea_b200.modules.finding import evaluation
from openea_b200.modules.load import read
from openea_b200.modules.utils.util import generate_out_folder, merge_dic

PAIR_THRESHOLD = 0.9      # run() builds its training pairs at 0.9, not at top_attr_threshold (attr2vec.py:185)
MAX_DIM = 128             # the NCE head's widest row


def get_kg_popular_attributes(kg, threshold):
    """attr2vec.py:19-28 with its printed lines; the selection is jape.popular_attributes."""
    print("total attributes:", len({attr for _, attr, _ in kg.attribute_triples_list}))
    selected = popular_attributes(kg, threshold)
    print("selected attributes", len(selected))
    return selected


def get_kgs_popular_attributes(kgs, threshold):
    """attr2vec.py:31-36: (kg1's, kg2's, their union) popular attribute sets."""
    a1, a2 = get_kg_popular_attributes(kgs.kg1, threshold), get_kg_popular_attributes(kgs.kg2, threshold)
    print("total selected attributes", len(a1 | a2))
    return a1, a2, a1 | a2


def entity_attribute_matrix(kgs, attributes=None, with_links=False):
    """The rows of merge_dic(kg1.entity_attributes_dict, kg2.entity_attributes_dict) as a boolean CSR
    [entities_num, attributes_num], restricted to `attributes` (a set; None = all).  with_links: a row of an entity in
    a training link also holds its counterpart's attributes (attr2vec.py:44-49); only entities of the merged dict
    have rows at all, as there."""
    merged = merge_dic(kgs.kg1.entity_attributes_dict, kgs.kg2.entity_attributes_dict)
    ents = np.fromiter(merged.keys(), dtype=np.int64, count=len(merged))
    counts = np.fromiter((len(v) for v in merged.values()), dtype=np.int64, count=len(merged))
    attrs = np.fromiter((a for v in merged.values() for a in v), dtype=np.int64, count=int(counts.sum()))
    shape = (kgs.entities_num, kgs.attributes_num)
    m = sp.csr_matrix((np.ones(len(attrs), dtype=np.float32), (np.repeat(ents, counts), attrs)), shape=shape)
    if with_links:
        link = merge_dic(dict(zip(kgs.train_entities1, kgs.train_entities2)),
                         dict(zip(kgs.train_entities2, kgs.train_entities1)))
        src = np.fromiter(link.keys(), dtype=np.int64, count=len(link))
        dst = np.fromiter(link.values(), dtype=np.int64, count=len(link))
        keep = np.isin(src, ents)
        move = sp.csr_matrix((np.ones(int(keep.sum()), dtype=np.float32), (src[keep], dst[keep])),
                             shape=(kgs.entities_num, kgs.entities_num))
        m = m + move @ m
    if attributes is not None:
        mask = np.zeros(kgs.attributes_num, dtype=np.float32)
        mask[np.fromiter(attributes, dtype=np.int64, count=len(attributes))] = 1.0
        m = m @ sp.diags(mask)
    m = (m > 0).astype(np.float32).tocsr()
    m.eliminate_zeros()
    m.sort_indices()
    return m


def generate_training_data(kgs, threshold=1.0):
    """attr2vec.py:39-55 vectorised: every unordered pair of each entity's attributes (with its counterpart's when it
    is in a training link) among the `threshold`-popular ones → int32 [n, 2].  Each pair is oriented smaller id first
    (input, label): the reference orients it, and orders the pairs, by CPython's set iteration, which is mostly but not
    always ascending for small ids, so only the multiset of unordered pairs is its contract and the orientation here is
    normalised."""
    _, _, selected = get_kgs_popular_attributes(kgs, threshold)
    print("entity attribute dict", len(kgs.kg1.entity_attributes_dict.keys() | kgs.kg2.entity_attributes_dict.keys()))
    m = entity_attribute_matrix(kgs, selected, with_links=True)
    ptr, idx = m.indptr.astype(np.int64), m.indices.astype(np.int64)
    row_end = np.repeat(ptr[1:], np.diff(ptr))
    later = row_end - np.arange(len(idx)) - 1          # the attributes after position p in its row
    first_pos = np.repeat(np.arange(len(idx)), later)
    start = np.repeat(np.cumsum(later) - later, later)
    second_pos = first_pos + 1 + (np.arange(len(first_pos)) - start)
    pairs = np.stack([idx[first_pos], idx[second_pos]], axis=1).astype(np.int32)
    print("training data of attribute correlations", len(pairs))
    return pairs


def mean_attribute_matrix(kgs, selected):
    """The CSR A with A[e, a] = 1/|attrs(e) ∩ selected| for an entity's own selected attributes (attr2vec.py:64-70)."""
    m = entity_attribute_matrix(kgs, selected)
    counts = np.diff(m.indptr)
    m.data = (1.0 / np.repeat(counts, counts)).astype(np.float32)
    return m


def entity_vectors(attr_table, mean_csr):
    """get_ent_embeds_from_attributes (attr2vec.py:58-76): normalize(A·Ê) → device [entities_num, dim]."""
    lib = L.load()
    Y = gnn.spmm(mean_csr, attr_table.lookup(padded=True))
    out = torch.zeros_like(Y)
    n, pitch = Y.shape
    L.check(lib.oea_rows_normalize(eng._ptr(Y), pitch, n, attr_table.dim, eng._ptr(out), pitch, eng._stream_ptr()),
            "oea_rows_normalize")
    return out[:, :attr_table.dim]


class Attr2Vec:

    def __init__(self):
        self.num_sampled_negs = -1
        self.kgs = None
        self.args = None
        self.out_folder = None
        self.flag1, self.flag2 = -1, -1
        self.early_stop = False
        self.session = None
        self.selected_attributes = None
        self.opt = 'Adagrad'
        self.seed = random.getrandbits(48)       # keys the pair draws and the sampler, as BasicModel's epoch seed
        self._mean_csr = None

    def set_args(self, args):
        self.args = args
        self.out_folder = generate_out_folder(self.args.output, self.args.training_data, self.args.dataset_division,
                                              self.__class__.__name__)

    def set_kgs(self, kgs):
        self.kgs = kgs
        _, _, self.selected_attributes = get_kgs_popular_attributes(kgs, self.args.top_attr_threshold)
        self.num_sampled_negs = len(self.selected_attributes) // 5

    def init(self):
        if par.world()[1] > 1:
            raise NotImplementedError("Attr2Vec runs on one GPU")
        if self.num_sampled_negs < 1:
            raise ValueError("Attr2Vec samples len(selected attributes) // 5 = %d classes: %d attributes are selected at "
                             "top_attr_threshold %s, fewer than 5" % (self.num_sampled_negs, len(self.selected_attributes),
                                                                      self.args.top_attr_threshold))
        if self.args.dim > MAX_DIM:
            raise ValueError("Attr2Vec's NCE head takes dim <= %d, got dim = %d" % (MAX_DIM, self.args.dim))
        self._define_variables()
        self._define_embed_graph()

    def _define_variables(self):
        shape = [self.kgs.attributes_num, self.args.dim]
        self.embeds = xavier_init(shape, 'attr_embed', True, optimizer=self.opt)
        self.nce_weights = xavier_init(shape, 'nce_weights', True, optimizer=self.opt)
        zeros = torch.zeros(self.kgs.attributes_num, 1)
        self.nce_biases = eng.EmbeddingTable(zeros, False, self.opt, self.embeds.device)

    def _define_embed_graph(self):
        self.trainer = eng.NceTrainer((self.embeds, self.nce_weights, self.nce_biases), self.num_sampled_negs,
                                      self.args.learning_rate)
        self.loss = self.optimizer = self.trainer

    def _entity_matrix(self):
        print("get entity embeddings from attributes")
        start = time.time()
        if self._mean_csr is None:
            self._mean_csr = gnn.DeviceCsr(mean_attribute_matrix(self.kgs, self.selected_attributes),
                                           self.embeds.device)
        mat = entity_vectors(self.embeds, self._mean_csr)
        print('cost time: {:.4f}s'.format(time.time() - start))
        return mat

    def eval_attribute_embeddings(self):
        return self.embeds.lookup().cpu().numpy()

    def eval_kg1_ent_embeddings(self):
        return self._entity_matrix()[torch.as_tensor(self.kgs.kg1.entities_list, device=self.embeds.device)].cpu().numpy()

    def eval_kg2_ent_embeddings(self):
        return self._entity_matrix()[torch.as_tensor(self.kgs.kg2.entities_list, device=self.embeds.device)].cpu().numpy()

    def eval_sim_mat(self):
        mat = self._entity_matrix()
        dev = self.embeds.device
        e1 = mat[torch.as_tensor(self.kgs.valid_entities1 + self.kgs.test_entities1, device=dev)]
        e2 = mat[torch.as_tensor(self.kgs.valid_entities2 + self.kgs.test_entities2, device=dev)]
        return (e1 @ e2.t()).cpu().numpy()

    def launch_training_1epo(self, epoch, steps, training_data_list=None):
        start = time.time()
        if training_data_list is not None:
            self.trainer.set_pairs(training_data_list)
        for i in range(steps):
            self.trainer.step(self.args.batch_size, self.seed, epoch, i)
        epoch_loss = self.trainer.read_loss()
        print('epoch {}, attribute loss: {:.4f}, cost time: {:.4f}s'.format(epoch, epoch_loss, time.time() - start))
        return epoch_loss

    def valid(self):
        mat = self._entity_matrix()
        dev = self.embeds.device
        embeds1 = mat[torch.as_tensor(self.kgs.valid_entities1, device=dev)]
        embeds2 = mat[torch.as_tensor(self.kgs.valid_entities2, device=dev)]
        hits1_12, mrr_12 = evaluation.valid(embeds1, embeds2, None, self.args.top_k, self.args.test_threads_num,
                                            metric=self.args.eval_metric)
        if self.args.stop_metric == 'hits1':
            return hits1_12
        return mrr_12

    def test(self, save=True):
        mat = self._entity_matrix()
        dev = self.embeds.device
        embeds1 = mat[torch.as_tensor(self.kgs.test_entities1, device=dev)]
        embeds2 = mat[torch.as_tensor(self.kgs.test_entities2, device=dev)]
        rest_12, _, _ = evaluation.test(embeds1, embeds2, None, self.args.top_k, self.args.test_threads_num,
                                        metric=self.args.eval_metric, csls_k=self.args.csls)
        if save:
            ent_ids_rest_12 = [(self.kgs.test_entities1[i], self.kgs.test_entities2[j]) for i, j in rest_12]
            read.save_results(self.out_folder, ent_ids_rest_12)

    def run(self):
        pairs = generate_training_data(self.kgs, threshold=PAIR_THRESHOLD)
        steps = len(pairs) // self.args.batch_size
        self.trainer.set_pairs(pairs)
        for i in range(1, self.args.attr_max_epoch + 1):
            self.launch_training_1epo(i, steps)

    def save(self):
        read.save_embeddings(self.out_folder, self.kgs, None, None, self.eval_attribute_embeddings())
