"""IPTransE on the CUDA engine (approaches/iptranse.py of the reference; SURVEY §8f-2).

Three losses over the shared entity / relation tables, all margin-based with one negative per positive:

  triple loss      Σ relu(m + s(h,r,t) − s(h',r,t'))                       iptranse.py:155-163   k_score_sampled (K1)
  path loss        path_parm · Σ (1/w) · relu(m + ‖r̂x + r̂y − r̂‖² − ‖r̂x + r̂y − r̂'‖²)   :176-185   weighted margin kernel,
                   both tables of the call = the relation table
  alignment loss   Σ w · relu(m + s(pos) − s(neg)) on the triples of newly aligned entities   :170-174,208-226

The triple and path losses share one Adagrad instance (one `apply` per step); the alignment loss has its own slots.
The reference builds the two-step paths with three pandas merges and feeds Python lists per step; here the path table
is built with sorted-key joins on arrays, lives on the device, and every batch (path samples, corrupted paths, the
triples of latent aligned entities and their corruptions) is index arithmetic on device tensors.
"""
import math
import time

import numpy as np
import torch

from openea_b200 import engine as eng
from openea_b200 import finding
from openea_b200 import parallel as par
from openea_b200.models.basic_model import BasicModel
from openea_b200.modules.finding.evaluation import early_stop
from openea_b200.modules.utils.util import load_session, task_divide


def two_step_paths(triples, chunk=4_000_000):
    """generate_2steps_path (iptranse.py:98-121) on arrays.  For every pair of triples (h, r_x, m), (m, r_y, t) with
    size(h, r_x) · size(m, r_y) < 101 — size(a, r) = number of triples with head a and relation r — and every direct
    triple (h, r, t): one row (r_x, r_y, r) with weight size·size.  Returns (int32 [P, 3], float32 [P]); row order is
    unspecified (the reference samples rows at random)."""
    tri = np.asarray(triples, dtype=np.int64).reshape(-1, 3)
    if len(tri) == 0:
        return np.zeros((0, 3), np.int32), np.zeros(0, np.float32)
    n_rel = int(tri[:, 1].max()) + 1
    n_ent = int(max(tri[:, 0].max(), tri[:, 2].max())) + 1
    _, inv, cnt = np.unique(tri[:, 0] * n_rel + tri[:, 1], return_inverse=True, return_counts=True)
    size = cnt[inv]                                              # per triple: |{(h, r, ·)}|
    by_head = np.argsort(tri[:, 0], kind="stable")
    th, tsize = tri[by_head], size[by_head]
    start = np.searchsorted(th[:, 0], np.arange(n_ent + 1))
    ht_order = np.argsort(tri[:, 0] * n_ent + tri[:, 2], kind="stable")
    ht_keys = (tri[:, 0] * n_ent + tri[:, 2])[ht_order]
    ht_rel = tri[ht_order, 1]
    fan = (start[1:] - start[:-1])[tri[:, 2]]                   # second hops of every first hop
    bounds = np.concatenate([[0], np.cumsum(fan)])
    rows, weights = [], []
    lo = 0
    while lo < len(tri):
        hi = max(int(np.searchsorted(bounds, bounds[lo] + chunk, side="right")) - 1, lo + 1)
        f = fan[lo:hi]
        total = int(f.sum())
        if total:
            first = np.repeat(np.arange(lo, hi), f)
            second = start[tri[first, 2]] + (np.arange(total) - np.repeat(bounds[lo:hi] - bounds[lo], f))
            w = size[first] * tsize[second]
            keep = w < 101
            first, second, w = first[keep], second[keep], w[keep]
            key = tri[first, 0] * n_ent + th[second, 2]
            a, b = np.searchsorted(ht_keys, key, side="left"), np.searchsorted(ht_keys, key, side="right")
            direct = b - a
            m = int(direct.sum())
            if m:
                src = np.repeat(np.arange(len(key)), direct)
                pos = np.repeat(a, direct) + (np.arange(m) - np.repeat(np.cumsum(direct) - direct, direct))
                rows.append(np.stack([tri[first[src], 1], th[second[src], 1], ht_rel[pos]], 1).astype(np.int32))
                weights.append(w[src].astype(np.float32))
        lo = hi
    if not rows:
        return np.zeros((0, 3), np.int32), np.zeros(0, np.float32)
    return np.concatenate(rows), np.concatenate(weights)


def latent_triples(tri_by_head, tri_by_tail, src, dst, w):
    """generate_newly_triples for a batch of aligned pairs in one KG (iptranse.py:30-47): every triple with head src[p]
    yields (dst[p], r, t, w[p]) and every triple with tail src[p] yields (h, r, dst[p], w[p]).  tri_by_head /
    tri_by_tail: (sorted [T, 3] int32 triples, row pointer by head resp. tail) from `_by_column`.  → ([M, 3], [M])."""
    out, ws = [], []
    for (tri, ptr), col in ((tri_by_head, 0), (tri_by_tail, 2)):
        lo, hi = ptr[src], ptr[src + 1]
        cnt = hi - lo
        total = int(cnt.sum())
        if total == 0:
            continue
        pair = torch.repeat_interleave(torch.arange(src.numel(), device=src.device), cnt)
        within = torch.arange(total, device=src.device) - torch.repeat_interleave(torch.cumsum(cnt, 0) - cnt, cnt)
        rows = tri[lo[pair] + within].clone()
        rows[:, col] = dst[pair].to(rows.dtype)
        out.append(rows)
        ws.append(w[pair])
    if not out:
        dev = src.device
        return torch.zeros(0, 3, dtype=torch.int32, device=dev), torch.zeros(0, dtype=torch.float32, device=dev)
    return torch.cat(out), torch.cat(ws)


def _by_column(triples, col, n_ent):
    order = torch.argsort(triples[:, col].long(), stable=True)
    tri = triples[order].contiguous()
    ptr = torch.searchsorted(tri[:, col].long().contiguous(), torch.arange(n_ent + 1, device=triples.device))
    return tri, ptr


def distinct_weighted(tri, w, n_ent, n_rel):
    """The reference collects (h, r, t, w) tuples in a set (iptranse.py:38-47): drop exact repeats."""
    if tri.shape[0] == 0:
        return tri, w
    key = (tri[:, 0].long() * n_rel + tri[:, 1].long()) * n_ent + tri[:, 2].long()
    order = torch.argsort(key, stable=True)
    key, w_s = key[order], w[order]
    first = torch.ones_like(key, dtype=torch.bool)
    first[1:] = (key[1:] != key[:-1]) | (w_s[1:] != w_s[:-1])
    keep = order[first]
    return tri[keep], w[keep]


class IPTransE(BasicModel):

    def __init__(self):
        super().__init__()
        self.ref_entities1, self.ref_entities2 = None, None
        self.paths1, self.paths2 = None, None
        self.alignment_trainer = None

    def init(self):
        if par.world()[1] > 1:
            raise NotImplementedError("%s runs on one GPU: its extra training passes have no cross-rank exchange yet" %
                                      self.__class__.__name__)
        self.ref_entities1 = self.kgs.valid_entities1 + self.kgs.test_entities1
        self.ref_entities2 = self.kgs.valid_entities2 + self.kgs.test_entities2
        self.session = load_session()
        self._define_variables()
        self._define_embed_graph()
        self._define_alignment_graph()
        self._build_paths()
        # hyper-parameter guards of the reference (iptranse.py:138-151)
        required = dict(alignment_module='sharing', init='normal', neg_sampling='uniform', optimizer='Adagrad',
                        eval_metric='inner', loss_norm='L2', ent_l2_norm=True, rel_l2_norm=True, neg_triple_num=1)
        for key, want in required.items():
            assert getattr(self.args, key) == want, "IPTransE needs %s=%r" % (key, want)
        assert self.args.margin > 0.0
        assert self.args.sim_th > 0.0

    def _define_embed_graph(self):
        super()._define_embed_graph(loss='margin-based', neg_per_pos=1)
        self.train_loss = self.optimizer = self.triple_trainer

    def _define_alignment_graph(self):
        self.alignment_trainer = eng.TripleTrainer(self.ent_embeds.new_slots(), self.rel_embeds.new_slots(),
                                                   self.triple_trainer.loss, self.args.learning_rate)
        self.alignment_loss = self.alignment_optimizer = self.alignment_trainer

    def _build_paths(self):
        dev = self.ent_embeds.device
        t = time.time()
        self._paths = []
        for kg in (self.kgs.kg1, self.kgs.kg2):
            arr = getattr(kg, "relation_triples_array", None)
            rows, w = two_step_paths(kg.relation_triples_list if arr is None else arr)
            print("num of path:", len(rows))
            rels = torch.as_tensor(np.asarray(kg.relations_list, dtype=np.int32), device=dev)
            self._paths.append((torch.as_tensor(rows, device=dev), torch.as_tensor(w, device=dev), rels))
        self.paths1, self.paths2 = self._paths[0][0], self._paths[1][0]
        print("two-step paths built in {:.3f} s".format(time.time() - t))

    # ---- PTransE epoch (iptranse.py:228-259) -------------------------------------------------------------------
    def _path_batch(self, path_batch_size):
        """generate_batch's path half (iptranse.py:82-89): a uniform sample without replacement of each KG's paths and,
        per sampled path, the same (r_x, r_y) with a relation drawn from that KG's relation list."""
        n1, n2 = self.paths1.shape[0], self.paths2.shape[0]
        num1 = int(n1 / (n1 + n2) * path_batch_size)
        pos, neg, ws = [], [], []
        for (rows, w, rels), num in zip(self._paths, (num1, path_batch_size - num1)):
            num = min(num, rows.shape[0])
            if num <= 0:
                continue
            pick = torch.randperm(rows.shape[0], device=rows.device)[:num]
            p = rows[pick]
            q = p.clone()
            q[:, 2] = rels[torch.randint(rels.numel(), (num,), device=rows.device)]
            pos.append(p); neg.append(q); ws.append(w[pick])
        if not pos:
            return None
        return torch.cat(pos).t().contiguous(), torch.cat(neg).t().contiguous(), torch.cat(ws)

    def launch_ptranse_training_1epo(self, epoch, triple_steps, steps_tasks, batch_queue):
        start = time.time()
        kg1, kg2, tset = self._device_kgs()
        kg1.clear_candidates(); kg2.clear_candidates()
        n_paths = self.paths1.shape[0] + self.paths2.shape[0]
        path_batch_size = n_paths // triple_steps
        self._epoch_seed = (self._epoch_seed * 6364136223846793005 + 1442695040888963407) & ((1 << 63) - 1)
        tr = self.triple_trainer
        for step in range(triple_steps):
            tr.score_sampled(kg1, kg2, tset, self.args.batch_size, 1, step, self._epoch_seed)
            batch = self._path_batch(path_batch_size) if path_batch_size > 0 else None
            if batch is not None:
                tr.score_margin_weighted(batch[0], batch[1], batch[2], reciprocal=True, scale=self.args.path_parm,
                                         paths=True)
            tr.apply()
        epoch_loss = tr.read_loss() / self.args.batch_size          # the reference divides by the batch size (:255)
        print('epoch {}, avg. triple loss: {:.4f}, cost time: {:.4f}s'.format(epoch, epoch_loss, time.time() - start))
        return epoch_loss

    # ---- alignment epoch (iptranse.py:261-294) ----------------------------------------------------------------
    def _kg_indices(self):
        if getattr(self, "_kg_index", None) is None:
            kg1, kg2, _ = self._device_kgs()
            n = self.kgs.entities_num
            self._kg_index = [(_by_column(kg.triples, 0, n), _by_column(kg.triples, 2, n)) for kg in (kg1, kg2)]
            dev = self.ent_embeds.device
            ents = np.concatenate([np.asarray(self.kgs.kg1.entities_list), np.asarray(self.kgs.kg2.entities_list)])
            self._all_entities = torch.as_tensor(ents.astype(np.int32), device=dev)
            self._ref1 = torch.as_tensor(np.asarray(self.ref_entities1, dtype=np.int64), device=dev)
            self._ref2 = torch.as_tensor(np.asarray(self.ref_entities2, dtype=np.int64), device=dev)
        return self._kg_index

    def latent_aligned_triples(self):
        """find_potential_alignment_greedily on the reference-entity similarity (each row's nearest column when its
        similarity exceeds sim_th) and the triples those pairs induce, with the pair similarity as weight."""
        idx = self._kg_indices()
        e1 = self.ent_embeds.lookup(self.ref_entities1)
        e2 = self.ent_embeds.lookup(self.ref_entities2)
        rows, cols, vals = finding.find_alignment_device(e1, e2, self.args.sim_th, 1, "inner", False)
        if rows.numel() == 0:
            return None
        new1, new2 = self._ref1[rows.long()], self._ref2[cols.long()]
        a, wa = latent_triples(idx[0][0], idx[0][1], new1, new2, vals)
        b, wb = latent_triples(idx[1][0], idx[1][1], new2, new1, vals)
        tri, w = distinct_weighted(torch.cat([a, b]), torch.cat([wa, wb]), self.kgs.entities_num, self.kgs.relations_num)
        print("newly triples: {}".format(tri.shape[0]))
        return tri, w

    def launch_alignment_training_1epo(self, epoch):
        t1 = time.time()
        found = self.latent_aligned_triples()
        if found is None or found[0].shape[0] == 0:
            return
        tri, w = found
        n = tri.shape[0]
        steps = max(1, math.ceil(n / self.args.batch_size))
        tr = self.alignment_trainer
        dev = tri.device
        for _ in range(steps):
            # generate_triple_batch (iptranse.py:64-70): a fresh sample without replacement per step; every negative
            # replaces the head (p = ½) or the tail by an entity of either KG, unfiltered (:50-61)
            pick = torch.randperm(n, device=dev)[:min(self.args.batch_size, n)]
            pos = tri[pick]
            neg = pos.clone()
            repl = self._all_entities[torch.randint(self._all_entities.numel(), (pick.numel(),), device=dev)]
            head = torch.rand(pick.numel(), device=dev) < 0.5
            neg[:, 0] = torch.where(head, repl, neg[:, 0])
            neg[:, 2] = torch.where(head, neg[:, 2], repl)
            tr.score_margin_weighted(pos.t().contiguous(), neg.t().contiguous(), w[pick])
            tr.apply()
        alignment_loss = tr.read_loss() / n
        print('epoch {}, alignment loss: {:.4f}, cost time: {:.4f}s'.format(epoch, alignment_loss, time.time() - t1))
        return alignment_loss

    def run(self):
        t = time.time()
        a = self.args
        triples_num = self.kgs.kg1.relation_triples_num + self.kgs.kg2.relation_triples_num
        triple_steps = int(math.ceil(triples_num / a.batch_size))
        steps_tasks = task_divide(list(range(triple_steps)), a.batch_threads_num)
        for epoch in range(getattr(self, "_start_epoch", 1), a.max_epoch):         # the reference stops before max_epoch (:302)
            self.launch_ptranse_training_1epo(epoch, triple_steps, steps_tasks, None)
            if epoch >= a.start_valid and epoch % a.eval_freq == 0:
                flag = self.valid(a.stop_metric)
                self.flag1, self.flag2, self.early_stop = early_stop(self.flag1, self.flag2, flag)
                if self.early_stop or epoch == a.max_epoch:
                    break
            if epoch % a.bp_freq == 0:
                self.launch_alignment_training_1epo(epoch)
            every = getattr(a, "checkpoint_every", 0)
            if every and epoch % every == 0:
                self.save_checkpoint(self.out_folder + "checkpoint.pt", epoch)
        print("Training ends. Total time = {:.3f} s.".format(time.time() - t))
