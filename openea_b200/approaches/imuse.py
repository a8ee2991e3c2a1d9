"""IMUSE on the CUDA engine (approaches/imuse.py of the reference; SURVEY §8f-2).

Training is TransE with the margin loss (one uniform negative, SGD) on the K1 kernels plus an align loss
Σ ‖ê₁ − ê₂‖² over the entity pairs a string matcher found before training (imuse.py:303-306,309-322), which is
`oea_pair_distance_loss` followed by the row optimiser with the align optimiser's own instance.

The string matcher ("interactive model", imuse.py:17-42) is host-side preprocessing outside the hot path: attributes of
the two KGs are paired by the similarity of their names, entities by the mean similarity of their values on paired
attributes.  It is restated here on plain dicts with two differences that do not change what is computed:
  * Levenshtein.ratio (python-Levenshtein is not installable offline) is computed from the longest common subsequence,
    ratio = 2·LCS(a, b) / (|a| + |b|) — the same number, since that package's ratio counts a substitution as 2 edits —
    with Hyyrö's bit-parallel LCS on Python integers;
  * an entity pair can only score above the (positive) threshold if the two entities share at least one paired
    attribute, so only those pairs are scored instead of all |E₁|·|E₂|.
The cost stays what the reference's is — every entity with a paired attribute against every such entity of the other
KG, one string comparison each — so, like there, the matcher is only practical on small KGs or selective attributes.
Where the reference's result depends on the iteration order of a Python set of tuples holding strings (which changes
from process to process), ids are visited in ascending order here; and its 8 worker processes each keep their own
"already taken" set (imuse.py:83-92), so a right-hand entity can be handed out once per worker — here once overall.
"""
import math
import time
from collections import defaultdict

import numpy as np
import torch

from openea_b200 import engine as eng
from openea_b200 import parallel as par
from openea_b200.models.basic_model import BasicModel
from openea_b200.modules.finding.evaluation import early_stop
from openea_b200.modules.utils.util import load_session, task_divide


def lcs_length(a, b):
    """Length of the longest common subsequence (bit-parallel: one big-integer update per character of b)."""
    if not a or not b:
        return 0
    masks = {}
    for i, ch in enumerate(a):
        masks[ch] = masks.get(ch, 0) | (1 << i)
    full = (1 << len(a)) - 1
    s = full
    for ch in b:
        u = s & masks.get(ch, 0)
        s = ((s + u) | (s - u)) & full
    return len(a) - bin(s).count("1")


def levenshtein_ratio(a, b):
    """Levenshtein.ratio(a, b) of python-Levenshtein: (|a| + |b| − d) / (|a| + |b|) with substitutions costing 2."""
    total = len(a) + len(b)
    return 1.0 if total == 0 else 2.0 * lcs_length(a, b) / total


compute_two_values_similarity = levenshtein_ratio        # imuse.py:198-199


def greedy_partner_scan(candidates, threshold):
    """The scan both matching passes of the reference share (imuse.py:42-66,100-122).  `candidates`: for every left item
    (ascending), its (right item, similarity) list in ascending right-item order.  Walking the right items, every time
    the running best (starting at `threshold`, strict >) improves, the new best is paired with the left item unless an
    earlier left item already took it; a left item that collected several partners keeps the last one.  → {left: right}."""
    taken, out = set(), {}
    for left in sorted(candidates):
        best, best_sim = None, threshold
        for right, sim in candidates[left]:
            if sim > best_sim:
                best, best_sim = right, sim
                if best not in taken:
                    out[left] = best
                    taken.add(best)
    return out


def get_aligned_attr_pair_by_name_similarity(kgs, sim_thresholds_attr, top_k=10):
    """imuse.py:202-246: pair attributes by the similarity of the last path segment of their names, keep the top_k
    pairs by the number of attribute triples they cover."""
    name = lambda d: {i: a.split('/')[-1] for a, i in d.items()}
    names1, names2 = name(kgs.kg1.attributes_id_dict), name(kgs.kg2.attributes_id_dict)
    attrs2 = sorted(kgs.kg2.attributes_set)
    cand = {a1: [(a2, levenshtein_ratio(names1[a1], names2[a2])) for a2 in attrs2] for a1 in kgs.kg1.attributes_set}
    # the reference pairs only the FINAL best of each attribute (the check follows its inner loop, :222-224)
    pairs, used = [], set()
    for a1 in sorted(cand):
        best, best_sim = None, sim_thresholds_attr
        for a2, sim in cand[a1]:
            if sim > best_sim:
                best, best_sim = a2, sim
        if best is not None and best not in used:
            pairs.append((a1, best))
            used.add(best)
    count1, count2 = defaultdict(int), defaultdict(int)
    for _, a, _ in kgs.kg1.attribute_triples_set:
        count1[a] += 1
    for _, a, _ in kgs.kg2.attribute_triples_set:
        count2[a] += 1
    pairs.sort(key=lambda p: count1[p[0]] + count2[p[1]], reverse=True)        # stable, like sorted(..., reverse=True)
    return set(pairs[:top_k])


def _values_by_attribute(attr_triples, wanted):
    """attribute → {entity: value} over the wanted attributes; of several values of one (entity, attribute) the
    reference keeps whichever its set iteration meets first (imuse.py:153-156) — here the smallest string."""
    out = defaultdict(dict)
    for e, a, v in attr_triples:
        if a in wanted and (e not in out[a] or v < out[a][e]):
            out[a][e] = v
    return out


def align_entity_by_attributes(kgs, aligned_attr_pair_set, sim_thresholds_ent):
    """imuse.py:69-97 (+ run_one_ea :42-66): entity pairs whose values on the paired attributes are similar on average."""
    print('align_entity_by_attributes...')
    if len(aligned_attr_pair_set) == 0:
        return set()
    vals1 = _values_by_attribute(kgs.kg1.attribute_triples_set, {a for a, _ in aligned_attr_pair_set})
    vals2 = _values_by_attribute(kgs.kg2.attribute_triples_set, {a for _, a in aligned_attr_pair_set})
    acc = defaultdict(lambda: [0.0, 0])                      # (e1, e2) → [Σ similarity, #paired attributes both have]
    cache = {}
    for a1, a2 in sorted(aligned_attr_pair_set):
        for e1, v1 in vals1.get(a1, {}).items():
            for e2, v2 in vals2.get(a2, {}).items():
                key = (v1, v2)
                if key not in cache:
                    cache[key] = levenshtein_ratio(v1, v2)
                slot = acc[(e1, e2)]
                slot[0] += cache[key]
                slot[1] += 1
    cand = defaultdict(list)
    for (e1, e2), (total, cnt) in sorted(acc.items()):
        cand[e1].append((e2, total / cnt))
    return set(greedy_partner_scan(cand, sim_thresholds_ent).items())


def align_attribute_by_entities(kgs, aligned_ent_pair_set, sim_thresholds_attr):
    """The intent of imuse.py:125-148: attribute pairs whose values agree on the already aligned entities.  (As written,
    the reference filters attribute ids against a set of ENTITY ids there (:131-134) and only reaches this pass when
    interactive_model_iter_num > 1; the shipped configurations use 1.)"""
    print('align_attribute_by_entities...')
    if not aligned_ent_pair_set:
        return set()
    by_ent1, by_ent2 = defaultdict(dict), defaultdict(dict)
    for store, triples in ((by_ent1, kgs.kg1.attribute_triples_set), (by_ent2, kgs.kg2.attribute_triples_set)):
        for e, a, v in triples:
            if a not in store[e] or v < store[e][a]:
                store[e][a] = v
    acc = defaultdict(lambda: [0.0, 0])
    for e1, e2 in sorted(aligned_ent_pair_set):
        for a1, v1 in by_ent1.get(e1, {}).items():
            for a2, v2 in by_ent2.get(e2, {}).items():
                slot = acc[(a1, a2)]
                slot[0] += levenshtein_ratio(v1, v2)
                slot[1] += 1
    cand = defaultdict(list)
    for (a1, a2), (total, cnt) in sorted(acc.items()):
        cand[a1].append((a2, total / cnt))
    return set(greedy_partner_scan(cand, sim_thresholds_attr).items())


def interactive_model(kgs, args):
    """imuse.py:17-39."""
    start = time.time()
    ent_pairs = set()
    attr_pairs = get_aligned_attr_pair_by_name_similarity(kgs, 0.6)
    print('aligned_attr_pair_set:', len(attr_pairs))
    i = 0
    while True:
        i += 1
        found = align_entity_by_attributes(kgs, attr_pairs, args.sim_thresholds_ent)
        ent_pairs |= found
        print(i, 'len(aligned_ent_pair_set_all):', len(ent_pairs), 'len(aligned_ent_pair_set_iter):', len(found))
        if i >= args.interactive_model_iter_num:
            break
        more = align_attribute_by_entities(kgs, ent_pairs, args.sim_thresholds_attr)
        if len(attr_pairs | more) == len(attr_pairs):
            break
        attr_pairs |= more
        print(i, 'len(aligned_attr_pair_set_all):', len(attr_pairs), 'len(aligned_attr_pair_set_iter):', len(more))
    print(time.time() - start)
    return ent_pairs


class IMUSE(BasicModel):

    def __init__(self):
        super().__init__()
        self.aligned_ent_pair_set = None
        self.alignment_trainer = None

    def init(self):
        if par.world()[1] > 1:
            raise NotImplementedError("%s runs on one GPU: its extra training passes have no cross-rank exchange yet" %
                                      self.__class__.__name__)
        self.aligned_ent_pair_set = interactive_model(self.kgs, self.args)
        self.session = load_session()
        self._define_variables()
        self._define_embed_graph()
        # hyper-parameter guards of the reference (imuse.py:262-273)
        required = dict(init='normal', loss='margin-based', neg_sampling='uniform', optimizer='SGD', eval_metric='inner',
                        loss_norm='L2', ent_l2_norm=True, rel_l2_norm=True, neg_triple_num=1)
        for key, want in required.items():
            assert getattr(self.args, key) == want, "IMUSE needs %s=%r" % (key, want)
        assert self.args.learning_rate >= 0.01

    def _define_embed_graph(self):
        super()._define_embed_graph()
        self.alignment_trainer = eng.TripleTrainer(self.ent_embeds.new_slots(), self.rel_embeds.new_slots(),
                                                   self.triple_trainer.loss, self.args.learning_rate)
        self.align_loss = self.align_optimizer = self.alignment_trainer

    def launch_align_training_1epo(self, epoch):
        start = time.time()
        dev = self.ent_embeds.device
        if getattr(self, "_pairs_dev", None) is None:
            pairs = np.asarray(sorted(self.aligned_ent_pair_set), dtype=np.int32).reshape(-1, 2)
            self._pairs_dev = torch.as_tensor(pairs, device=dev)
        n = self._pairs_dev.shape[0]
        steps = int(math.ceil(n / self.args.batch_size))
        tr = self.alignment_trainer
        for _ in range(steps):                       # every step feeds ALL pairs (imuse.py:314-317)
            tr.score_pairs(self._pairs_dev[:, 0], self._pairs_dev[:, 1])
            tr.apply()
        epoch_loss = tr.read_loss() / max(1, steps * n)
        print('epoch {}, align learning loss: {:.4f}, time: {:.4f}s'.format(epoch, epoch_loss, time.time() - start))
        return epoch_loss

    def run(self):
        t = time.time()
        a = self.args
        triples_num = self._local_triples_num()
        triple_steps = int(math.ceil(triples_num / a.batch_size))
        steps_tasks = task_divide(list(range(triple_steps)), a.batch_threads_num)
        every = getattr(a, "checkpoint_every", 0)
        for i in range(getattr(self, "_start_epoch", 1), a.max_epoch + 1):
            self.launch_triple_training_1epo(i, triple_steps, steps_tasks, None, None, None)
            self.launch_align_training_1epo(i)
            if every and i % every == 0:
                self.save_checkpoint(self.out_folder + "checkpoint.pt", i)
            if i >= a.start_valid and i % a.eval_freq == 0:
                flag = self.valid(a.stop_metric)
                self.flag1, self.flag2, self.early_stop = early_stop(self.flag1, self.flag2, flag)
                if self.early_stop or i == a.max_epoch:
                    break
        print("Training ends. Total time = {:.3f} s.".format(time.time() - t))
