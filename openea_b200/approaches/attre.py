"""AttrE on the CUDA engine (approaches/attre.py of the reference; SURVEY §8f-2): three losses per epoch, each with its
own SGD instance —

  structure     margin TransE on relation triples                                  K1 sampled step (BasicModel)
  characters    margin TransE-form loss on attribute triples (e, a, v):  ê_ce[e] + â[a] − v̄,  where the value vector
                v̄ = Σ_p w_p · ĉ[char_p(v)] composes the (normalised) embeddings of the literal's first `literal_len`
                characters with the n-gram weights w_p = Σ_{s=0}^{L−1−p} 1/(L − s)  (attre.py:83-107: the sum over all
                suffix means of the reversed sequence, written out)
  joint         Σ (1 − ⟨ê_se[e], ê_ce[e]⟩) over all entities                        (attre.py:186-188)

Rows are gathered and normalised by the K1 lookup kernel, the margin loss and its gradient are one kernel
(oea_loss_rows), gradients return through the normalisation by the K1 scatter kernel and the tables are stepped by the
row optimiser; in between sit a [batch, L, d] weighted sum (the character composition) and a row-wise dot product,
issued through torch.  Batches (fixed-size positive slices with wrap-around, one corrupted entity per positive) are
index arithmetic on the device.
"""
import math
import time

import numpy as np
import torch

from openea_b200 import parallel as par
from openea_b200.models.basic_model import BasicModel
from openea_b200.modules.base.initializers import init_embeddings
from openea_b200.modules.base.losses import get_loss_func
from openea_b200.modules.finding.evaluation import early_stop
from openea_b200.modules.utils.util import load_session, task_divide


def clean_literal(v):
    """clean_attribute_triples (attre.py:25-32): cut at the first '(', strip punctuation, cut at the first '\"'."""
    v = v.split('(')[0].rstrip(' ')
    for ch in '.(),':
        v = v.replace(ch, '')
    return v.replace('_', ' ').replace('-', ' ').split('"')[0]


def formatting_attr_triples(kgs, literal_len):
    """attre.py:17-80 on arrays: → (triples1 [n1, 3], triples2 [n2, 3] as (entity, attribute, value id), the character
    ids of every value [n1 + n2, literal_len] (0 = padding / rare character), number of character rows).
    Every attribute triple gets its own value id, KG1's first.  Characters rarer than 10⁻⁴ of all characters of the
    distinct literals are dropped; the reference numbers the kept ones in the iteration order of a Python set — here by
    descending frequency (the numbering is arbitrary: each id only names a row of a randomly initialised table)."""
    lists = [[(e, a, clean_literal(v)) for e, a, v in kg.local_attribute_triples_list] for kg in (kgs.kg1, kgs.kg2)]
    values = sorted({v for triples in lists for _, _, v in triples})
    count = {}
    for literal in values:
        for ch in literal:
            count[ch] = count.get(ch, 0) + 1
    total = sum(count.values())
    ranked = sorted(count.items(), key=lambda kv: (-kv[1], kv[0]))
    char_id = {ch: i + 1 for i, (ch, n) in enumerate(c for c in ranked if c[1] / total >= 0.0001)}
    out, char_rows = [], []
    vid = 0
    for triples in lists:
        arr = np.zeros((len(triples), 3), dtype=np.int32)
        for i, (e, a, v) in enumerate(triples):
            arr[i] = (e, a, vid)
            char_rows.append([char_id.get(ch, 0) for ch in v[:literal_len]] + [0] * max(0, literal_len - len(v)))
            vid += 1
        out.append(arr)
    chars = np.asarray(char_rows, dtype=np.int32).reshape(-1, literal_len)
    return out[0], out[1], chars, len(char_id) + 1


def ngram_weights(length):
    """Position weights of n_gram_compositional_func (attre.py:83-107)."""
    return np.array([sum(1.0 / (length - s) for s in range(length - p)) for p in range(length)], dtype=np.float32)


class AttrE(BasicModel):

    def __init__(self):
        super().__init__()
        self.ent_embeds_ce = self.attr_embeds = self.char_embeds = None

    def init(self):
        if par.world()[1] > 1:
            raise NotImplementedError("AttrE runs on one GPU: its extra training passes have no cross-rank exchange yet")
        self.attribute_triples_list1, self.attribute_triples_list2, self.value_id_char_ids, self.char_list_size = \
            formatting_attr_triples(self.kgs, self.args.literal_len)
        self.session = load_session()
        self._define_variables()
        self._define_embed_graph()

    def _define_variables(self):
        super()._define_variables()
        a, opt = self.args, self.args.optimizer
        self.ent_embeds_ce = init_embeddings([self.kgs.entities_num, a.dim], 'ent_embeds_ce', a.init, a.ent_l2_norm, optimizer=opt)
        self.attr_embeds = init_embeddings([self.kgs.attributes_num, a.dim], 'attr_embeds', a.init, a.attr_l2_norm, optimizer=opt)
        self.char_embeds = init_embeddings([self.char_list_size, a.dim], 'char_embeds', a.init, a.char_l2_norm, optimizer=opt)

    def _define_embed_graph(self):
        super()._define_embed_graph()
        dev = self.ent_embeds.device
        self._chars = torch.as_tensor(np.asarray(self.value_id_char_ids, dtype=np.int64).reshape(-1, self.args.literal_len),
                                      device=dev)
        self._weights = torch.as_tensor(ngram_weights(self.args.literal_len), device=dev)
        # each generate_optimizer call of the reference owns its slots; SGD has none, new_slots keeps the structure
        self._ce_tables = (self.ent_embeds_ce, self.attr_embeds, self.char_embeds)
        self._joint_tables = (self.ent_embeds.new_slots(), self.ent_embeds_ce.new_slots())
        self.loss_ce_dev = torch.zeros(1, dtype=torch.float64, device=dev)

    # ---- character-level triple step (attre.py:176-182,190-218) ---------------------------------------------------
    def value_vectors(self, value_ids):
        """(looked-up character rows as a leaf [n·L, d], the composed value vectors [n, d])."""
        ids = self._chars[value_ids.long()].reshape(-1)
        rows = self.char_embeds.lookup(ids.to(torch.int32)).requires_grad_(True)
        vec = (rows.reshape(-1, self.args.literal_len, self.args.dim) * self._weights[None, :, None]).sum(1)
        return ids, rows, vec

    def ce_step(self, pos, neg):
        """One session.run([triple_loss_ce, triple_optimizer_ce]); pos / neg: [3, n] int32 (entity | attribute | value id)."""
        n_pos = pos.shape[1]
        ents = torch.cat([pos[0], neg[0]]).contiguous()
        attrs = torch.cat([pos[1], neg[1]]).contiguous()
        e_rows = self.ent_embeds_ce.lookup(ents).requires_grad_(True)
        a_rows = self.attr_embeds.lookup(attrs).requires_grad_(True)
        char_ids, c_rows, v = self.value_vectors(torch.cat([pos[2], neg[2]]))
        loss = get_loss_func(e_rows[:n_pos], a_rows[:n_pos], v[:n_pos], e_rows[n_pos:], a_rows[n_pos:], v[n_pos:], self.args)
        loss.backward()
        self.ent_embeds_ce.scatter_grad(e_rows.grad.contiguous(), ents)
        self.attr_embeds.scatter_grad(a_rows.grad.contiguous(), attrs)
        self.char_embeds.scatter_grad(c_rows.grad.contiguous(), char_ids.to(torch.int32))
        for tab in self._ce_tables:
            tab.apply(self.args.learning_rate)
        return loss.detach()

    def _attribute_batch(self, step):
        """generate_attribute_triple_batch (batch.py:214-225) with is_fixed_size=True: wrap-around slices of both KGs'
        attribute triples and, per positive, the same (attribute, value) with another entity of the same KG."""
        dev = self.ent_embeds.device
        if getattr(self, "_attr_dev", None) is None:
            up = lambda a: torch.as_tensor(np.ascontiguousarray(a), device=dev)
            self._attr_dev = (up(self.attribute_triples_list1), up(self.attribute_triples_list2))
            self._ents_dev = (up(np.asarray(self.kgs.kg1.entities_list, dtype=np.int32)),
                              up(np.asarray(self.kgs.kg2.entities_list, dtype=np.int32)))
        t1, t2 = self._attr_dev
        b1 = int(t1.shape[0] / (t1.shape[0] + t2.shape[0]) * self.args.batch_size)
        pos, neg = [], []
        for tri, ents, b in ((t1, self._ents_dev[0], b1), (t2, self._ents_dev[1], self.args.batch_size - b1)):
            if b <= 0 or tri.shape[0] == 0:
                continue
            start = step * b
            p = tri[start:min(start + b, tri.shape[0])]
            if p.shape[0] < b:                                       # generate_pos_triples, is_fixed_size (batch.py:55-56)
                p = torch.cat([p, tri[:b - p.shape[0]]])
            q = p.clone()
            for _ in range(self.args.neg_triple_num - 1):
                q = torch.cat([q, p])
            draw = ents[torch.randint(ents.numel(), (q.shape[0],), device=dev)]
            again = draw == q[:, 0]                                  # the only triple with this value id is the positive
            while bool(again.any()) and ents.numel() > 1:
                draw[again] = ents[torch.randint(ents.numel(), (int(again.sum()),), device=dev)]
                again = draw == q[:, 0]
            q[:, 0] = draw
            pos.append(p); neg.append(q)
        return torch.cat(pos).t().contiguous(), torch.cat(neg).t().contiguous()

    def launch_triple_training_1epo_ce(self, epoch, triple_steps, steps_tasks, batch_queue):
        start = time.time()
        total, trained = torch.zeros((), dtype=torch.float64, device=self.ent_embeds.device), 0
        for step in range(triple_steps):
            pos, neg = self._attribute_batch(step)
            total += self.ce_step(pos, neg).double()
            trained += pos.shape[1]
        epoch_loss = float(total.item()) / max(1, trained)
        print('epoch {}, CE, avg. triple loss: {:.4f}, cost time: {:.4f}s'.format(epoch, epoch_loss, time.time() - start))
        return epoch_loss

    # ---- joint step (attre.py:186-188,220-233) -------------------------------------------------------------------
    def joint_step(self, ents):
        se, ce = self._joint_tables
        a = se.lookup(ents).requires_grad_(True)
        b = ce.lookup(ents).requires_grad_(True)
        loss = (1.0 - (a * b).sum(1)).sum()
        loss.backward()
        se.scatter_grad(a.grad.contiguous(), ents)
        ce.scatter_grad(b.grad.contiguous(), ents)
        se.apply(self.args.learning_rate)
        ce.apply(self.args.learning_rate)
        return loss.detach()

    def launch_joint_training_1epo(self, epoch, entities):
        start = time.time()
        dev = self.ent_embeds.device
        if getattr(self, "_joint_ents", None) is None:
            self._joint_ents = torch.as_tensor(np.asarray(entities, dtype=np.int32), device=dev)
        n = self._joint_ents.numel()
        steps = int(math.ceil(n / self.args.batch_size))
        total = torch.zeros((), dtype=torch.float64, device=dev)
        for _ in range(steps):                                  # every step feeds ALL entities (attre.py:226-228)
            total += self.joint_step(self._joint_ents).double()
        epoch_loss = float(total.item()) / max(1, steps * n)
        print('epoch {}, joint learning loss: {:.4f}, time: {:.4f}s'.format(epoch, epoch_loss, time.time() - start))
        return epoch_loss

    def run(self):
        t = time.time()
        a = self.args
        relation_triple_steps = int(math.ceil(self._local_triples_num() / a.batch_size))
        attribute_triples_num = len(self.attribute_triples_list1) + len(self.attribute_triples_list2)
        attribute_triple_steps = int(math.ceil(attribute_triples_num / a.batch_size))
        relation_step_tasks = task_divide(list(range(relation_triple_steps)), a.batch_threads_num)
        entity_list = list(self.kgs.kg1.entities_list) + list(self.kgs.kg2.entities_list)
        every = getattr(a, "checkpoint_every", 0)
        for i in range(getattr(self, "_start_epoch", 1), a.max_epoch + 1):
            self.launch_triple_training_1epo(i, relation_triple_steps, relation_step_tasks, None, None, None)
            self.launch_triple_training_1epo_ce(i, attribute_triple_steps, None, None)
            self.launch_joint_training_1epo(i, entity_list)
            if every and i % every == 0:
                self.save_checkpoint(self.out_folder + "checkpoint.pt", i)
            if i >= a.start_valid and i % a.eval_freq == 0:
                flag = self.valid(a.stop_metric)
                self.flag1, self.flag2, self.early_stop = early_stop(self.flag1, self.flag2, flag)
                if self.early_stop or i == a.max_epoch:
                    break
        print("Training ends. Total time = {:.3f} s.".format(time.time() - t))
