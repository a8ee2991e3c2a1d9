"""JAPE on the CUDA engine (approaches/jape.py of the reference; SURVEY §8f-2).

Structure embedding: the triple loss Σ s⁺ − neg_alpha·Σ s⁻ with s = ‖ĥ + r̂ − t̂‖² (jape.py:72-82), Adagrad — two
passes of the fed scorer with the positive loss (scale 1 on the positives, −neg_alpha on the negatives) and one row
optimiser step; batches from the device producer.

Attribute branch: the reference trains Attr2Vec (an NCE skip-gram over attribute ids, approaches/attr2vec.py) first and
then, every epoch, only EVALUATES the attribute-similarity loss — `launch_sim_1epo` fetches `sim_loss` without its
optimiser (jape.py:125-135) — so the attribute branch never changes an entity embedding; its only output is the
printed "sim loss".  `attribute_similarity` below restates that branch as a host-side auxiliary in torch (not part of
any hot path): NCE with TF's log-uniform unique candidate sampler and expected-count correction (from the TF 1.x
documentation), entity vectors as the mean of their attribute vectors, similarities above the threshold.
"""
import math
import time

import numpy as np
import torch

from openea_b200 import engine as eng
from openea_b200 import parallel as par
from openea_b200.models.basic_model import BasicModel
from openea_b200.modules.finding.evaluation import early_stop
from openea_b200.modules.utils.util import load_session, merge_dic, task_divide


class JapeTripleTrainer(eng.ModelTrainer):
    """Σ s⁺ − α·Σ s⁻ on the TransE instance of oea_model_score_fed (positive loss, signed scales)."""

    def __init__(self, ent, rel, neg_alpha, lr):
        super().__init__("TransE", (ent, rel), eng.loss_cfg("positive", "L2"), lr)
        self.neg_alpha = float(neg_alpha)

    def score_fed(self, pos, neg=None, loss_out=None, scale=None):
        super().score_fed(pos, None, loss_out, scale=1.0)
        if neg is not None and neg.shape[1]:
            super().score_fed(neg, None, loss_out, scale=-self.neg_alpha)


def popular_attributes(kg, threshold):
    """get_kg_popular_attributes (attr2vec.py:19-29): the `threshold` share of attributes with the most triples."""
    count = {}
    for _, attr, _ in kg.attribute_triples_list:
        count[attr] = count.get(attr, 0) + 1
    ranked = sorted(count, key=count.get, reverse=True)
    return set(ranked[:int(len(count) * threshold)])


def log_uniform_unique(range_max, num_sampled, rng):
    """tf.nn.log_uniform_candidate_sampler(unique=True): classes drawn with P(c) = log((c + 2) / (c + 1)) / log(range_max + 1)
    until `num_sampled` distinct ones are held.  → (ids, number of draws it took: the sampler's `num_tries`)."""
    ids, seen, tries = [], set(), 0
    while len(ids) < num_sampled:
        for c in (np.exp(rng.random(2 * num_sampled) * math.log(range_max + 1.0)).astype(np.int64) - 1) % range_max:
            tries += 1
            if int(c) not in seen:
                seen.add(int(c))
                ids.append(int(c))
                if len(ids) == num_sampled:
                    break
    return np.asarray(ids, dtype=np.int64), tries


def nce_loss(weights, biases, labels, inputs, sampled, num_tries, range_max):
    """tf.nn.nce_loss with its defaults (one true class, shared sampled classes, subtract_log_q, accidental hits kept):
    sigmoid cross-entropy of the true logit against 1 and of every sampled logit against 0, logits corrected by
    −log(expected count) with expected count = 1 − (1 − p)^num_tries for the unique sampler.  → [batch]."""
    prob = lambda c: torch.log((c.double() + 2.0) / (c.double() + 1.0)) / math.log(range_max + 1.0)
    expected = lambda c: -torch.expm1(num_tries * torch.log1p(-prob(c)))
    true_logits = (inputs * weights[labels]).sum(1) + biases[labels] - torch.log(expected(labels)).to(inputs.dtype)
    sampled_logits = inputs @ weights[sampled].t() + biases[sampled] - torch.log(expected(sampled)).to(inputs.dtype)
    bce = torch.nn.functional.binary_cross_entropy_with_logits
    return bce(true_logits, torch.ones_like(true_logits), reduction="none") + \
        bce(sampled_logits, torch.zeros_like(sampled_logits), reduction="none").sum(1)


def attribute_similarity(kgs, args, device, epochs=None, seed=0):
    """Attr2Vec (approaches/attr2vec.py) as a host-side auxiliary in torch: attribute vectors trained by NCE on the
    attribute pairs that co-occur on an entity (or on its seed-aligned counterpart), entity vectors as the mean of
    their popular attributes' vectors, and the reference-entity similarity matrix thresholded as jape.py:147."""
    selected = popular_attributes(kgs.kg1, args.top_attr_threshold) | popular_attributes(kgs.kg2, args.top_attr_threshold)
    ent_attrs = merge_dic(kgs.kg1.entity_attributes_dict, kgs.kg2.entity_attributes_dict)
    link = merge_dic(dict(zip(kgs.train_entities1, kgs.train_entities2)), dict(zip(kgs.train_entities2, kgs.train_entities1)))
    popular = popular_attributes(kgs.kg1, 0.9) | popular_attributes(kgs.kg2, 0.9)            # generate_training_data(threshold=0.9)
    pairs = []
    for ent, attrs in ent_attrs.items():
        if ent in link:
            attrs = attrs | ent_attrs.get(link[ent], set())
        attrs = sorted(attrs & popular)
        pairs.extend((a, b) for i, a in enumerate(attrs) for b in attrs[i + 1:])            # itertools.combinations(…, 2)
    print("training data of attribute correlations", len(pairs))
    n_attr, dim, batch = kgs.attributes_num, args.dim, args.batch_size
    num_sampled = len(selected) // 5
    gen = torch.Generator().manual_seed(seed)
    rng = np.random.default_rng(seed)
    std = math.sqrt(2.0 / (n_attr + dim))
    make = lambda: (torch.randn(n_attr, dim, generator=gen) * std).to(device).requires_grad_(True)
    embeds, nce_w = make(), make()
    bias = torch.zeros(n_attr, device=device, requires_grad=True)
    steps = len(pairs) // batch
    if steps > 0 and num_sampled > 0:
        data = torch.as_tensor(np.asarray(pairs, dtype=np.int64), device=device)
        opt = torch.optim.Adagrad([embeds, nce_w, bias], lr=args.learning_rate, initial_accumulator_value=0.1)
        l2n = lambda x: torch.nn.functional.normalize(x, dim=1, eps=1e-6)
        for epoch in range(1, (args.attr_max_epoch if epochs is None else epochs) + 1):
            start, total = time.time(), 0.0
            for _ in range(steps):
                pick = data[torch.as_tensor(rng.choice(len(pairs), batch, replace=False), device=device)]
                sampled, tries = log_uniform_unique(n_attr, num_sampled, rng)
                loss = nce_loss(l2n(nce_w), bias, pick[:, 1], l2n(embeds)[pick[:, 0]], torch.as_tensor(sampled, device=device),
                                tries, n_attr).mean()
                opt.zero_grad()
                loss.backward()
                opt.step()
                total += float(loss.detach())
            print('epoch {}, attribute loss: {:.4f}, cost time: {:.4f}s'.format(epoch, total, time.time() - start))
    vec = torch.nn.functional.normalize(embeds.detach(), dim=1)
    ent_mat = torch.zeros(kgs.entities_num, dim, device=device)
    for ent, attrs in ent_attrs.items():
        ids = sorted(attrs & selected)
        if ids:
            ent_mat[ent] = vec[torch.as_tensor(ids, device=device)].mean(0)
    ent_mat = torch.nn.functional.normalize(ent_mat, dim=1)
    ref1 = torch.as_tensor(kgs.valid_entities1 + kgs.test_entities1, device=device)
    ref2 = torch.as_tensor(kgs.valid_entities2 + kgs.test_entities2, device=device)
    sim = ent_mat[ref1] @ ent_mat[ref2].t()
    return torch.where(sim < args.attr_sim_mat_threshold, torch.zeros_like(sim), sim)


class JAPE(BasicModel):

    def __init__(self):
        super().__init__()
        self.attr_sim_mat = None
        self.ref_entities1, self.ref_entities2 = None, None

    def init(self):
        if par.world()[1] > 1:
            raise NotImplementedError("JAPE runs on one GPU")
        self.ref_entities1 = self.kgs.valid_entities1 + self.kgs.test_entities1
        self.ref_entities2 = self.kgs.valid_entities2 + self.kgs.test_entities2
        self.session = load_session()
        self._define_variables()
        self._define_embed_graph()
        # hyper-parameter guards of the reference (jape.py:35-50)
        required = dict(alignment_module='sharing', init='normal', neg_sampling='uniform', optimizer='Adagrad',
                        eval_metric='inner', loss_norm='L2', ent_l2_norm=True, rel_l2_norm=True)
        for key, want in required.items():
            assert getattr(self.args, key) == want, "JAPE needs %s=%r" % (key, want)
        assert self.args.neg_triple_num >= 1 and self.args.neg_alpha >= 0.0
        assert self.args.top_attr_threshold > 0.0 and self.args.attr_sim_mat_threshold > 0.0 and self.args.attr_sim_mat_beta > 0.0

    def _define_embed_graph(self):
        self.triple_trainer = JapeTripleTrainer(self.ent_embeds, self.rel_embeds, self.args.neg_alpha, self.args.learning_rate)
        self.neg_per_pos = self.args.neg_triple_num
        self.triple_loss = self.triple_optimizer = self.triple_trainer

    def sim_loss(self, rows):
        """jape.py:84-93 for the reference entities at `rows` (a sub-matrix of attr_sim_mat): evaluation only."""
        ref1 = self.ent_embeds.lookup([self.ref_entities1[i] for i in rows])
        ref2 = self.ent_embeds.lookup(self.ref_entities2)
        trans = torch.nn.functional.normalize(self.attr_sim_mat[torch.as_tensor(rows, device=ref2.device)] @ ref2, dim=1, eps=1e-6)
        return float(self.args.attr_sim_mat_beta * ((ref1 - trans) ** 2).sum())

    def launch_sim_1epo(self, epoch):
        t = time.time()
        steps = len(self.ref_entities1) // self.args.sub_mat_size
        loss = 0.0
        for _ in range(steps):
            rows = np.random.choice(len(self.ref_entities1), self.args.sub_mat_size, replace=False).tolist()
            loss += self.sim_loss(rows)
        print('epoch {}, sim loss: {:.4f}, cost time: {:.4f}s'.format(epoch, loss, time.time() - t))

    def run_attr2vec(self):
        t = time.time()
        print("Training attribute embeddings:")
        self.attr_sim_mat = attribute_similarity(self.kgs, self.args, self.ent_embeds.device)
        print("Training attributes ends. Total time = {:.3f} s.".format(time.time() - t))

    def run(self):
        self.run_attr2vec()
        print("Joint training:")
        t = time.time()
        a = self.args
        triple_steps = int(math.ceil(self._local_triples_num() / a.batch_size))
        steps_tasks = task_divide(list(range(triple_steps)), a.batch_threads_num)
        for i in range(getattr(self, "_start_epoch", 1), a.max_epoch + 1):
            self.launch_triple_training_1epo(i, triple_steps, steps_tasks, None, None, None)
            self.launch_sim_1epo(i)
            if i >= a.start_valid and i % a.eval_freq == 0:
                flag = self.valid(a.stop_metric)
                self.flag1, self.flag2, self.early_stop = early_stop(self.flag1, self.flag2, flag)
                if self.early_stop or i == a.max_epoch:
                    break
        print("Training ends. Total time = {:.3f} s.".format(time.time() - t))
