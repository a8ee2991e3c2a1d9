"""BootEA on the CUDA engine (approaches/bootea.py): AlignE + bootstrapping of likely alignments.

Per iteration: `sub_epoch` epochs of fused triple steps → validation → bootstrapping (reference-entity
cosine similarity on the GPU, threshold ∧ top-k filter, matching, editing) → one pass of the alignment loss
−Σ log σ(−‖h+r−t‖²) on swapped triples (own Adagrad slots) → ε-truncated neighbour refresh.
run() keeps the bootstrapping working set on the device (modules/bootstrapping/device.py: matching, label editing and
swap-triple generation as tensor index arithmetic); the set / dict functions below are the reference's module-level
API (bootea_transh.py imports them) and the statement the device versions are tested against.
The likelihood graph of the reference (bootea.py:201-212) is never executed there (its call is commented
out, :293) and is not built here.
"""
import gc
import math
import time

import numpy as np
import torch

from openea_b200 import engine as eng
from openea_b200 import finding as F
from openea_b200.approaches.aligne import AlignE
from openea_b200.modules.bootstrapping import device as boot
from openea_b200.modules.bootstrapping.alignment_finder import find_alignment_from_embeds, mwgm, mwgm_graph_tool, \
    check_new_alignment
from openea_b200.modules.finding.evaluation import early_stop
from openea_b200.modules.load.kg import KG
from openea_b200.modules.utils.util import load_session, task_divide


class PairSim:
    """Similarity of selected (i, j) pairs of the reference-entity matrix without materialising it: what
    `sim_mat[i, j]` reads in bootea.py:35-78."""

    def __init__(self, embeds1, embeds2):
        self.e1, self.e2 = embeds1, embeds2          # row-normalised CUDA tensors

    def values(self, pairs):
        if not pairs:
            return {}
        idx = torch.as_tensor(list(pairs), dtype=torch.long, device=self.e1.device)
        v = (self.e1[idx[:, 0]] * self.e2[idx[:, 1]]).sum(1)   # gather + row dot (plumbing on a few thousand pairs)
        return dict(zip(pairs, v.cpu().tolist()))


def bootstrapping(sim_mat, unaligned_entities1, unaligned_entities2, labeled_alignment, sim_th, k):
    """sim_mat: PairSim over the reference entities.  Returns (labeled alignment set, newly aligned ids 1, 2)."""
    pairs, _ = find_alignment_from_embeds(sim_mat.e1, sim_mat.e2, sim_th, k, metric="inner", normalize=False)
    curr = None
    if pairs is not None:
        check_new_alignment(pairs, context="after filtering by sim and nearest k")
        t1 = time.time()
        curr = mwgm(pairs, sim_mat.values(list(pairs)), mwgm_graph_tool)
        check_new_alignment(curr, context="after mwgm")
        print("mwgm costs time: {:.3f} s".format(time.time() - t1))
    if curr is not None:
        labeled_alignment = update_labeled_alignment_x(labeled_alignment, curr, sim_mat)
        labeled_alignment = update_labeled_alignment_y(labeled_alignment, sim_mat)
    if labeled_alignment is not None:
        ents1 = [unaligned_entities1[p[0]] for p in labeled_alignment]
        ents2 = [unaligned_entities2[p[1]] for p in labeled_alignment]
    else:
        ents1, ents2 = None, None
    gc.collect()
    return labeled_alignment, ents1, ents2


def update_labeled_alignment_x(pre_labeled_alignment, curr_labeled_alignment, sim_mat):
    """Keep, for every KG1 index, the partner with the larger similarity between the previous and the new label."""
    labeled = dict(pre_labeled_alignment)
    need = [(i, labeled[i]) for i, _ in curr_labeled_alignment if i in labeled] + list(curr_labeled_alignment)
    val = sim_mat.values(list(set(need)))
    n1 = n2 = 0
    for i, j in curr_labeled_alignment:
        if labeled.get(i, -1) == i and j != i:
            n2 += 1
        if i in labeled:
            pre_j = labeled[i]
            if val[(i, j)] >= val[(i, pre_j)]:
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
    """Resolve KG2 indices claimed by several KG1 indices in favour of the most similar claimant."""
    by_j = {}
    for i, j in labeled_alignment:
        by_j.setdefault(j, set()).add(i)
    contested = [(i, j) for j, claim in by_j.items() if len(claim) > 1 for i in claim]
    val = sim_mat.values(contested)
    out = set()
    for j, claim in by_j.items():
        if len(claim) == 1:
            out.add((next(iter(claim)), j))
        else:
            best_i, best = -1, -10
            for i in claim:
                if val[(i, j)] > best:
                    best, best_i = val[(i, j)], i
            out.add((best_i, j))
    check_new_alignment(out, context="after editing (->)")
    return out


def generate_newly_triples(ent1, ent2, rt_dict1, hr_dict1):
    out = [(ent2, r, t) for r, t in rt_dict1.get(ent1, ())]
    out.extend((h, r, ent2) for h, r in hr_dict1.get(ent1, ()))
    return out


def generate_supervised_triples(rt_dict1, hr_dict1, rt_dict2, hr_dict2, ents1, ents2):
    assert len(ents1) == len(ents2)
    new1, new2 = [], []
    for a, b in zip(ents1, ents2):
        new1.extend(generate_newly_triples(a, b, rt_dict1, hr_dict1))
        new2.extend(generate_newly_triples(b, a, rt_dict2, hr_dict2))
    print("newly triples: {}, {}".format(len(new1), len(new2)))
    return new1, new2


def generate_pos_batch(triples1, triples2, step, batch_size):
    num1 = int(len(triples1) / (len(triples1) + len(triples2)) * batch_size)
    num2 = batch_size - num1
    return (triples1[step * num1:min(step * num1 + num1, len(triples1))],
            triples2[step * num2:min(step * num2 + num2, len(triples2))])


class BootEA(AlignE):

    def __init__(self):
        super().__init__()
        self.ref_ent1 = None
        self.ref_ent2 = None
        self.alignment_trainer = None

    def init(self):
        self.session = load_session()
        self._define_variables()
        self._define_embed_graph()
        self._define_alignment_graph()
        self.ref_ent1 = self.kgs.valid_entities1 + self.kgs.test_entities1
        self.ref_ent2 = self.kgs.valid_entities2 + self.kgs.test_entities2
        self._check_args()

    def _define_alignment_graph(self):
        # its own optimiser instance ⇒ its own Adagrad accumulators (bootea.py:198)
        self.alignment_trainer = eng.TripleTrainer(self.ent_embeds.new_slots(), self.rel_embeds.new_slots(),
                                                   eng.loss_cfg("logsigmoid", "L2"), self.args.learning_rate)
        self.alignment_loss = self.alignment_optimizer = self.alignment_trainer

    def eval_ref_sim_mat(self):
        """Cosine similarity of the reference entities (bootea.py:214-219) as a lazy PairSim."""
        e1, _ = F.to_device_rows(self.ent_embeds.lookup(self.ref_ent1), normalize=True)
        e2, _ = F.to_device_rows(self.ent_embeds.lookup(self.ref_ent2), normalize=True)
        d = self.ent_embeds.dim
        return PairSim(e1[:, :d].contiguous(), e2[:, :d].contiguous())

    def launch_training_k_epo(self, iter, iter_nums, triple_steps, steps_tasks, training_batch_queue, neighbors1,
                              neighbors2):
        for i in range(1, iter_nums + 1):
            epoch = (iter - 1) * iter_nums + i
            self.launch_triple_training_1epo(epoch, triple_steps, steps_tasks, training_batch_queue, neighbors1,
                                             neighbors2)
            self._sync_seed_rows()             # no-op on one GPU

    def train_alignment(self, kg1: KG, kg2: KG, entities1, entities2, training_epochs):
        if entities1 is None or len(entities1) == 0:
            return
        new1, new2 = generate_supervised_triples(kg1.rt_dict, kg1.hr_dict, kg2.rt_dict, kg2.hr_dict, entities1, entities2)
        total = len(new1) + len(new2)
        steps = max(1, math.ceil(total / self.args.batch_size))
        dev = self.ent_embeds.device
        for _ in range(training_epochs):
            t1 = time.time()
            for step in range(steps):
                b1, b2 = generate_pos_batch(new1, new2, step, self.args.batch_size)
                batch = b1 + b2
                if not batch:
                    continue
                pos = torch.as_tensor(np.asarray(batch, dtype=np.int32).T.copy(), device=dev)
                self.alignment_trainer.score_fed(pos)
                self.alignment_trainer.apply()
            alignment_loss = self.alignment_trainer.read_loss() / max(1, total)
            print("alignment_loss = {:.3f}, time = {:.3f} s".format(alignment_loss, time.time() - t1))

    # ---- device-resident bootstrapping (SURVEY §8f-1) ---------------------------------------------------------------
    def _local_triples_device(self, kg):
        """The KG's LOCAL relation triples (what rt_dict / hr_dict are built from, kg.py:86-91) as a device tensor."""
        arr = getattr(kg, "local_relation_triples_array", None)
        if arr is None:
            arr = np.asarray(kg.local_relation_triples_list, dtype=np.int32).reshape(-1, 3)
        return torch.as_tensor(np.ascontiguousarray(arr, dtype=np.int32), device=self.ent_embeds.device)

    def bootstrap_on_device(self):
        """bootstrapping() of bootea.py:19-32 without leaving the device: returns the labelled pairs as entity-id
        tensors (entities1, entities2), or (None, None) when nothing is labelled yet."""
        dev = self.ent_embeds.device
        if getattr(self, "_label", None) is None:
            self._label = torch.full((len(self.ref_ent1),), -1, dtype=torch.int64, device=dev)
            self._ref1 = torch.as_tensor(self.ref_ent1, dtype=torch.int64, device=dev)
            self._ref2 = torch.as_tensor(self.ref_ent2, dtype=torch.int64, device=dev)
        sim = self.eval_ref_sim_mat()
        cand = F.find_alignment_device(sim.e1, sim.e2, self.args.sim_th, max(self.args.k, 1), "inner", False)
        _, i, j = boot.bootstrap_labels(sim.e1, sim.e2, self._label, cand)
        if i.numel() == 0:
            return None, None
        return self._ref1[i], self._ref2[j]

    def train_alignment_device(self, entities1, entities2, training_epochs):
        """train_alignment (bootea.py:228-251) with the swap triples generated and batched on the device."""
        if entities1 is None or entities1.numel() == 0:
            return
        if getattr(self, "_local1", None) is None:
            self._local1 = self._local_triples_device(self.kgs.kg1)
            self._local2 = self._local_triples_device(self.kgs.kg2)
        n_ent = self.kgs.entities_num
        new1 = boot.swap_triples(self._local1, entities1, entities2, n_ent)
        new2 = boot.swap_triples(self._local2, entities2, entities1, n_ent)
        print("newly triples: {}, {}".format(new1.shape[0], new2.shape[0]))
        total = new1.shape[0] + new2.shape[0]
        if total == 0:
            return
        steps = max(1, math.ceil(total / self.args.batch_size))
        for _ in range(training_epochs):
            t1 = time.time()
            for step in range(steps):
                pos = boot.pos_batch(new1, new2, step, self.args.batch_size)
                if pos.shape[1] == 0:
                    continue
                self.alignment_trainer.score_fed(pos)
                self.alignment_trainer.apply()
            alignment_loss = self.alignment_trainer.read_loss() / total
            print("alignment_loss = {:.3f}, time = {:.3f} s".format(alignment_loss, time.time() - t1))

    # ---- checkpoint / resume at iteration granularity (BasicModel.save_checkpoint + the bootstrapped labels) ---------
    def _extra_state(self):
        label = getattr(self, "_label", None)
        return {"label": None if label is None else label.cpu()}

    def _load_extra_state(self, extra):
        if extra.get("label") is not None:
            dev = self.ent_embeds.device
            self._label = extra["label"].to(dev)
            self._ref1 = torch.as_tensor(self.ref_ent1, dtype=torch.int64, device=dev)
            self._ref2 = torch.as_tensor(self.ref_ent2, dtype=torch.int64, device=dev)

    def run(self):
        t = time.time()
        triples_num = self._local_triples_num()
        triple_steps = int(math.ceil(triples_num / self.args.batch_size))
        steps_tasks = task_divide(list(range(triple_steps)), self.args.batch_threads_num)
        neighbors1, neighbors2 = None, None
        sub_num = self.args.sub_epoch
        iter_nums = self.args.max_epoch // sub_num
        first_iter = (getattr(self, "_start_epoch", 1) - 1) // sub_num + 1       # checkpoints are written after whole iterations
        if first_iter > 1:
            neighbors1, neighbors2 = self._refresh_neighbours()                  # derived state: rebuilt, not stored
        every = getattr(self.args, "checkpoint_every", 0)
        for i in range(first_iter, iter_nums + 1):
            print("\niteration", i)
            self.launch_training_k_epo(i, sub_num, triple_steps, steps_tasks, None, neighbors1, neighbors2)
            if i * sub_num >= self.args.start_valid:
                flag = self.valid(self.args.stop_metric)
                self.flag1, self.flag2, self.early_stop = early_stop(self.flag1, self.flag2, flag)
                if self.early_stop or i == iter_nums:
                    break
            self._sync_replicas()              # under torchrun every rank must label the same pairs (no-op on one GPU)
            entities1, entities2 = self.bootstrap_on_device()
            self.train_alignment_device(entities1, entities2, 1)
            if i * sub_num >= self.args.start_valid:
                self.valid(self.args.stop_metric)
            t1 = time.time()
            neighbors1 = neighbors2 = None
            gc.collect()
            neighbors1, neighbors2 = self._refresh_neighbours()
            ent_num = len(self.kgs.kg1.entities_list) + len(self.kgs.kg2.entities_list)
            torch.cuda.synchronize()
            print("generating neighbors of {} entities costs {:.3f} s.".format(ent_num, time.time() - t1))
            if every and (i * sub_num) % every == 0:
                self.save_checkpoint(self.out_folder + "checkpoint.pt", i * sub_num)
        print("Training ends. Total time = {:.3f} s.".format(time.time() - t))
