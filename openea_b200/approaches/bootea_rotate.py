"""BootEA_RotatE (approaches/bootea_rotate.py of the reference): BootEA whose triple graph is RotatE's (real and
imaginary entity tables, relation phases, −Σ log σ(γ − d⁺) − Σ log σ(d⁻ − γ) with the negatives unweighted, :70-78) and
whose alignment loss is the positive half −Σ log σ(γ − d) on the swapped triples (:149-160, its own optimiser instance).
The reference-entity similarity, the ε-truncated neighbours, validation, test and save read re + im (:110-169).
Bootstrapping starts at epoch args.start_bp and runs args.align_times alignment epochs; early stopping waits for
args.min_iter iterations (:201-245)."""
import gc
import math
import time

import torch

from openea_b200 import engine as eng
from openea_b200 import finding as F
from openea_b200.approaches.bootea import BootEA, PairSim
from openea_b200.models.semantic.rotate import RotatE
from openea_b200.modules.finding.evaluation import early_stop
from openea_b200.modules.utils.util import load_session, task_divide


class BootEA_RotatE(BootEA):

    def __init__(self):
        super().__init__()
        self.pi = 3.14159265358979323846
        self.epsilon = 2.0
        self.embedding_range = None
        self.re_ent_embeds = self.im_ent_embeds = None

    def init(self):
        self.embedding_range = (self.args.gamma + self.epsilon) / self.args.dim
        self._define_variables()
        self._define_embed_graph()
        self._define_alignment_graph()
        self.session = load_session()
        self.ref_ent1 = self.kgs.valid_entities1 + self.kgs.test_entities1
        self.ref_ent2 = self.kgs.valid_entities2 + self.kgs.test_entities2
        assert self.args.alignment_module == 'swapping'
        assert self.args.neg_triple_num > 0.0
        assert self.args.truncated_epsilon > 0.0

    _define_variables = RotatE._define_variables
    _triple_trainer = RotatE._triple_trainer
    _both_parts = RotatE._both_parts
    _eval_valid_embeddings = RotatE._eval_valid_embeddings
    _eval_test_embeddings = RotatE._eval_test_embeddings
    save = RotatE.save

    def _define_embed_graph(self):
        self.triple_trainer = self._triple_trainer(None)           # negatives at weight 1 (bootea_rotate.py:77)
        self.neg_per_pos = self.args.neg_triple_num
        self.triple_loss = self.triple_optimizer = self.triple_trainer

    def _define_alignment_graph(self):
        # its own optimiser instance ⇒ its own slots (bootea_rotate.py:159-160)
        tables = (self.re_ent_embeds.new_slots(), self.rel_embeds.new_slots(), self.im_ent_embeds.new_slots())
        self.alignment_trainer = eng.ModelTrainer("RotatE", tables, eng.loss_cfg("logsigmoid", "L2"),
                                                  self.args.learning_rate, gamma=self.args.gamma)
        self.alignment_loss = self.alignment_optimizer = self.alignment_trainer

    def _normalised_sum(self, ids):
        """l2_normalize(re + im) of the given entities (bootea_rotate.py:129-140,163-168), device rows [n, dim]."""
        e, _ = F.to_device_rows(self._both_parts(ids), normalize=True)
        return e[:, :self.args.dim].contiguous()

    def eval_ref_sim_mat(self):
        return PairSim(self._normalised_sum(self.ref_ent1), self._normalised_sum(self.ref_ent2))

    def eval_kg1_useful_ent_embeddings(self):
        ids = self.kgs.useful_entities_list1
        return self._normalised_sum(ids) if self.args.ent_l2_norm else self._both_parts(ids)

    def eval_kg2_useful_ent_embeddings(self):
        ids = self.kgs.useful_entities_list2
        return self._normalised_sum(ids) if self.args.ent_l2_norm else self._both_parts(ids)

    # ---- checkpoint / resume: the labels (BootEA's) and the alignment optimiser's own slots --------------------------
    def _extra_state(self):
        state = super()._extra_state()
        state["alignment_slots"] = [tab.state_dict() for tab in self.alignment_trainer.live]
        return state

    def _load_extra_state(self, extra):
        super()._load_extra_state(extra)
        for tab, st in zip(self.alignment_trainer.live, extra.get("alignment_slots", [])):
            tab.load_state_dict(st)

    def run(self):
        t = time.time()
        triples_num = self._local_triples_num()
        triple_steps = int(math.ceil(triples_num / self.args.batch_size))
        steps_tasks = task_divide(list(range(triple_steps)), self.args.batch_threads_num)
        truncated = self.args.neg_sampling == "truncated"
        neighbors1, neighbors2 = None, None
        sub_num = self.args.sub_epoch
        iter_nums = self.args.max_epoch // sub_num
        first_iter = (getattr(self, "_start_epoch", 1) - 1) // sub_num + 1       # checkpoints are written after whole iterations
        if first_iter > 1 and truncated:
            neighbors1, neighbors2 = self._refresh_neighbours()                  # derived state: rebuilt, not stored
        every = getattr(self.args, "checkpoint_every", 0)
        for i in range(first_iter, iter_nums + 1):
            print("\niteration", i)
            self.launch_training_k_epo(i, sub_num, triple_steps, steps_tasks, None, neighbors1, neighbors2)
            if i * sub_num >= self.args.start_valid:
                flag = self.valid(self.args.stop_metric)
                self.flag1, self.flag2, self.early_stop = early_stop(self.flag1, self.flag2, flag)
                if (self.early_stop and i >= self.args.min_iter) or i == iter_nums:
                    break
            if i * sub_num >= self.args.start_bp:
                print("bootstrapping")
                self._sync_replicas()          # under torchrun every rank must label the same pairs (no-op on one GPU)
                entities1, entities2 = self.bootstrap_on_device()
                self.train_alignment_device(entities1, entities2, self.args.align_times)
                if i * sub_num >= self.args.start_valid:
                    self.valid(self.args.stop_metric)
            if truncated:
                t1 = time.time()
                assert 0.0 < self.args.truncated_epsilon < 1.0
                neighbors1 = neighbors2 = None
                gc.collect()
                neighbors1, neighbors2 = self._refresh_neighbours()
                ent_num = len(self.kgs.kg1.entities_list) + len(self.kgs.kg2.entities_list)
                torch.cuda.synchronize()
                print("generating neighbors of {} entities costs {:.3f} s.".format(ent_num, time.time() - t1))
            if every and (i * sub_num) % every == 0:
                self.save_checkpoint(self.out_folder + "checkpoint.pt", i * sub_num)
        print("Training ends. Total time = {:.3f} s.".format(time.time() - t))
