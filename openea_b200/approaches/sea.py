"""SEA on the CUDA engine (approaches/sea.py of the reference; SURVEY §8f-2): TransE with the margin loss (one uniform
negative, Adam) on the K1 kernels + a cycle-consistent pair of mapping matrices trained on labelled and unlabelled
entity pairs.

Mapping step (sea.py:78-100), per batch of labelled pairs (a, b) and unlabelled pairs (x, y):

    mapped_12 = N(Ê[a]·M₁)   mapped_21 = N(Ê[b]·M₂)   cyc_1 = N(Ê[x]·M₁·M₂)   cyc_2 = N(Ê[y]·M₂·M₁)
    loss = α₁·(‖Ê[b] − mapped_12‖² + ‖Ê[a] − mapped_21‖²) + α₂·(‖Ê[x] − cyc_1‖² + ‖Ê[y] − cyc_2‖²)

with Ê the l2-normalised lookup and N = tf.nn.l2_normalize WITHOUT an axis: the whole [batch, d] matrix is divided by
its Frobenius norm (sea.py:84-85,90-93 — kept as written).  The rows are gathered and their gradients pushed back
through the normalisation by the K1 lookup / scatter kernels and all three variables are stepped by the row optimiser
with the mapping optimiser's own Adam slots; the four [batch, d]·[d, d] products in between (a few hundred rows) are
library GEMMs issued through torch, like the dense X·W products of path (ii).
"""
import math
import time

import numpy as np
import torch

from openea_b200 import parallel as par
from openea_b200.models.basic_model import BasicModel
from openea_b200.modules.base.initializers import orthogonal_init
from openea_b200.modules.finding.evaluation import early_stop
from openea_b200.modules.load import read as rd
from openea_b200.modules.utils.util import load_session, task_divide


def frobenius_normalize(x):
    """tf.nn.l2_normalize(x) with axis=None: x · rsqrt(max(Σ x², 1e-12)) over ALL elements."""
    return x * torch.rsqrt(torch.clamp((x * x).sum(), min=1e-12))


def sea_mapping_loss(l1, l2, u1, u2, m1, m2, alpha_1, alpha_2):
    """The mapping loss of sea.py:83-98 on looked-up rows (any float dtype; autograd-friendly)."""
    sq = lambda a, b: ((a - b) ** 2).sum()
    sup = sq(l2, frobenius_normalize(l1 @ m1)) + sq(l1, frobenius_normalize(l2 @ m2))
    semi = sq(u1, frobenius_normalize(u1 @ m1 @ m2)) + sq(u2, frobenius_normalize(u2 @ m2 @ m1))
    return alpha_1 * sup + alpha_2 * semi


class SEAMappingTrainer:
    """session.run([mapping_loss, mapping_optimizer]) of sea.py:99-100,130-136."""

    def __init__(self, ent, m1, m2, alpha_1, alpha_2, lr):
        self.ent = ent.new_slots()          # the mapping optimiser's own slots on the entity variable (SURVEY A.3)
        self.rel = None
        self.m1, self.m2 = m1, m2
        self.alpha_1, self.alpha_2, self.lr = float(alpha_1), float(alpha_2), float(lr)
        self.loss_dev = torch.zeros(1, dtype=torch.float64, device=ent.device)

    def step(self, labeled1, labeled2, unlabeled1, unlabeled2):
        dev = self.ent.device
        parts = [torch.as_tensor(x, dtype=torch.int32, device=dev).reshape(-1) for x in
                 (labeled1, labeled2, unlabeled1, unlabeled2)]
        ids = torch.cat(parts).contiguous()
        rows = self.ent.lookup(ids).requires_grad_(True)
        l1, l2, u1, u2 = torch.split(rows, [p.numel() for p in parts])
        d = self.ent.dim
        m1 = self.m1.weight[:, :d].detach().clone().requires_grad_(True)
        m2 = self.m2.weight[:, :d].detach().clone().requires_grad_(True)
        loss = sea_mapping_loss(l1, l2, u1, u2, m1, m2, self.alpha_1, self.alpha_2)
        loss.backward()
        self.loss_dev += loss.detach().double()
        self.ent.scatter_grad(rows.grad.contiguous(), ids)
        for tab, g in ((self.m1, m1.grad), (self.m2, m2.grad)):
            tab.grad[:, :d] += g
            tab.touched.fill_(1)
        for tab in (self.ent, self.m1, self.m2):
            tab.apply(self.lr)

    def read_loss(self, reset=True):
        v = float(self.loss_dev.item())
        if reset:
            self.loss_dev.zero_()
        return v


class SEA(BasicModel):

    def __init__(self):
        super().__init__()
        self.mapping_mat_1 = self.mapping_mat_2 = None

    def init(self):
        if par.world()[1] > 1:
            raise NotImplementedError("%s runs on one GPU: its extra training passes have no cross-rank exchange yet" %
                                      self.__class__.__name__)
        self.session = load_session()
        self._define_variables()
        self._define_embed_graph()
        # hyper-parameter guards of the reference (sea.py:30-39)
        required = dict(loss='margin-based', alignment_module='mapping', neg_sampling='uniform', optimizer='Adam',
                        eval_metric='inner', loss_norm='L2', ent_l2_norm=True, rel_l2_norm=True, neg_triple_num=1)
        for key, want in required.items():
            assert getattr(self.args, key) == want, "SEA needs %s=%r" % (key, want)

    def _define_variables(self):
        super()._define_variables()
        dim, opt = self.args.dim, self.args.optimizer
        self.mapping_mat_1 = orthogonal_init([dim, dim], 'mapping_matrix_1', optimizer=opt)
        self.mapping_mat_2 = orthogonal_init([dim, dim], 'mapping_matrix_2', optimizer=opt)
        self.mapping_mat = self.mapping_mat_1          # what valid() / test() map KG1's embeddings with (sea.py:110,116)
        self.eye_mat_1 = self.eye_mat_2 = None         # defined but unused by the reference's losses

    def _define_embed_graph(self):
        super()._define_embed_graph()
        self.mapping_trainer = SEAMappingTrainer(self.ent_embeds, self.mapping_mat_1, self.mapping_mat_2,
                                                 self.args.alpha_1, self.args.alpha_2, self.args.learning_rate)
        self.mapping_loss = self.mapping_optimizer = self.mapping_trainer

    def save(self):
        ent_embeds = self.ent_embeds.lookup().cpu().numpy()
        rel_embeds = self.rel_embeds.lookup().cpu().numpy()
        rd.save_embeddings(self.out_folder, self.kgs, ent_embeds, rel_embeds, None,
                           mapping_mat=self.mapping_mat_1.raw().cpu().numpy(),
                           rev_mapping_mat=self.mapping_mat_2.raw().cpu().numpy())

    def launch_training_1epo(self, epoch, triple_steps, steps_tasks, training_batch_queue, neighbors1, neighbors2):
        self.launch_triple_training_1epo(epoch, triple_steps, steps_tasks, training_batch_queue, neighbors1, neighbors2)
        self.launch_mapping_training_1epo(epoch, triple_steps)

    def launch_mapping_training_1epo(self, epoch, triple_steps):
        start = time.time()
        dev = self.ent_embeds.device
        if getattr(self, "_links_dev", None) is None:
            as_dev = lambda links: torch.as_tensor(np.asarray(links, dtype=np.int32).reshape(-1, 2), device=dev)
            self._links_dev = as_dev(self.kgs.train_links)
            self._unlabeled_dev = as_dev(self.kgs.test_links + self.kgs.valid_links)
        # every step draws its two samples without replacement, independently of the other steps (random.sample per
        # step, sea.py:126-129): all steps' index sets in one device draw each
        n_l, n_u = self._links_dev.shape[0], self._unlabeled_dev.shape[0]
        m_l, m_u = n_l // triple_steps, n_u // triple_steps
        pick = lambda n, m: torch.rand(triple_steps, n, device=dev).topk(m, dim=1).indices if m > 0 else None
        pl, pu = pick(n_l, m_l), pick(n_u, m_u)
        empty = torch.zeros(0, 2, dtype=torch.int32, device=dev)
        for step in range(triple_steps):
            lab = self._links_dev[pl[step]] if pl is not None else empty
            unl = self._unlabeled_dev[pu[step]] if pu is not None else empty
            self.mapping_trainer.step(lab[:, 0], lab[:, 1], unl[:, 0], unl[:, 1])
        epoch_loss = self.mapping_trainer.read_loss() / max(1, triple_steps * m_l)
        print('epoch {}, avg. mapping loss: {:.4f}, cost time: {:.4f}s'.format(epoch, epoch_loss, time.time() - start))
        return epoch_loss

    def run(self):
        t = time.time()
        a = self.args
        triples_num = self._local_triples_num()
        triple_steps = int(math.ceil(triples_num / a.batch_size))
        steps_tasks = task_divide(list(range(triple_steps)), a.batch_threads_num)
        every = getattr(a, "checkpoint_every", 0)
        for i in range(getattr(self, "_start_epoch", 1), a.max_epoch + 1):
            self.launch_training_1epo(i, triple_steps, steps_tasks, None, None, None)
            if every and i % every == 0:
                self.save_checkpoint(self.out_folder + "checkpoint.pt", i)
            if i >= a.start_valid and i % a.eval_freq == 0:
                flag = self.valid(a.stop_metric)
                self.flag1, self.flag2, self.early_stop = early_stop(self.flag1, self.flag2, flag)
                if self.early_stop or i == a.max_epoch:
                    break
        print("Training ends. Total time = {:.3f} s.".format(time.time() - t))
