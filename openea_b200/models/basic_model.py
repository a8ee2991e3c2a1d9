"""BasicModel: the 6-call lifecycle set_args / set_kgs / init / run / test / save of the reference
(models/basic_model.py) over the CUDA engine.

What changed underneath (the lifecycle, printed lines and files on disk are the reference's):
  * variables are device tables (openea_b200.engine.EmbeddingTable), the "graph" is a TripleTrainer;
  * one training step = oea_triple_score_sampled (batch slicing + negative sampling + forward/backward in one
    kernel, replacing the mp.Process batch producers of basic_model.py:213-219 and session.run :224-230)
    + oea_rowopt_apply on both tables;
  * validation / test / ε-truncated neighbour refresh never leave the GPU (K3 kernels).
"""
import gc
import math
import os
import random
import time

import numpy as np
import torch

import openea_b200.modules.load.read as rd
import openea_b200.modules.train.batch as bat
from openea_b200 import engine as eng
from openea_b200 import parallel as par
from openea_b200.modules.base.initializers import init_embeddings, set_default_optimizer
from openea_b200.modules.base.mapping import add_mapping_variables, add_mapping_module
from openea_b200.modules.finding.alignment import stable_alignment
from openea_b200.modules.finding.evaluation import valid, test, early_stop
from openea_b200.modules.finding.similarity import sim
from openea_b200.modules.utils.util import generate_out_folder, load_session, task_divide


def _loss_from_args(args, loss=None):
    """args.loss / loss_norm / margins → engine loss config (get_loss_func, losses.py:4-12)."""
    kind = loss or args.loss
    if kind == 'margin-based':
        return eng.loss_cfg(kind, args.loss_norm, margin=args.margin)
    if kind == 'limited':
        # the approaches that name the limited loss themselves pass balance=args.neg_margin_balance (aligne.py:63-65,
        # bootea_transh.py:94-96); get_loss_func does not, so the default balance = 1.0 applies there (losses.py:10,44)
        balance = getattr(args, "neg_margin_balance", 1.0) if loss is not None else 1.0
        return eng.loss_cfg(kind, args.loss_norm, margin=args.pos_margin, neg_margin=args.neg_margin, balance=balance)
    return eng.loss_cfg(kind, getattr(args, "loss_norm", "L2"))


class BasicModel:

    def __init__(self):
        self.out_folder = None
        self.args = None
        self.kgs = None
        self.session = None
        self.rel_embeds = None
        self.ent_embeds = None
        self.mapping_mat = None
        self.eye_mat = None
        self.triple_optimizer = None
        self.triple_loss = None
        self.mapping_optimizer = None
        self.mapping_loss = None
        self.mapping_trainer = None
        self.triple_trainer = None
        self.neg_per_pos = None
        self._dkg1 = self._dkg2 = self._tset = None
        self._epoch_seed = random.getrandbits(48)
        self.flag1 = -1
        self.flag2 = -1
        self.early_stop = False

    # ---- lifecycle -----------------------------------------------------------------------------------
    def set_kgs(self, kgs):
        self.kgs = kgs

    def set_args(self, args):
        self.args = args
        self.out_folder = generate_out_folder(self.args.output, self.args.training_data, self.args.dataset_division,
                                              self.__class__.__name__)

    def init(self):
        pass  # to be overridden

    # ---- "graph" definition --------------------------------------------------------------------------
    def _define_variables(self):
        set_default_optimizer(self.args.optimizer)
        self.ent_embeds = init_embeddings([self.kgs.entities_num, self.args.dim], 'ent_embeds',
                                          self.args.init, self.args.ent_l2_norm, optimizer=self.args.optimizer)
        self.rel_embeds = init_embeddings([self.kgs.relations_num, self.args.dim], 'rel_embeds',
                                          self.args.init, self.args.rel_l2_norm, optimizer=self.args.optimizer)

    def _define_embed_graph(self, loss=None, neg_per_pos=None):
        self.triple_trainer = eng.TripleTrainer(self.ent_embeds, self.rel_embeds, _loss_from_args(self.args, loss),
                                                self.args.learning_rate)
        self.neg_per_pos = self.args.neg_triple_num if neg_per_pos is None else neg_per_pos
        self.triple_loss = self.triple_trainer       # handles kept under the reference's attribute names
        self.triple_optimizer = self.triple_trainer

    def _define_mapping_variables(self):
        add_mapping_variables(self)

    def _define_mapping_graph(self):
        add_mapping_module(self)

    def _device_kgs(self):
        """Device copies of both KGs' triple/entity lists + the triple membership set (built once)."""
        if self._dkg1 is None:
            dev = self.ent_embeds.device

            def device_kg(kg):     # the array-backed loader hands its int32 arrays over without building Python lists
                triples = getattr(kg, "relation_triples_array", None)
                entities = getattr(kg, "entities_array", None)
                return eng.DeviceKG(kg.relation_triples_list if triples is None else triples,
                                    kg.entities_list if entities is None else entities, self.kgs.entities_num, dev)
            self._dkg1, self._dkg2 = device_kg(self.kgs.kg1), device_kg(self.kgs.kg2)
            self._tset = eng.DeviceTripleSet([self._dkg1.triples, self._dkg2.triples], self.kgs.entities_num,
                                             self.kgs.relations_num, dev)       # membership test: ALL triples, every rank
            rank, world = par.world()
            if world > 1 and self._multi_mode() == "seed":   # this rank trains on the triples whose head row it owns (id mod G)
                for dkg in (self._dkg1, self._dkg2):
                    mine = par.shard_triples(dkg.triples.cpu().numpy(), rank, world)
                    dkg.triples = torch.as_tensor(np.ascontiguousarray(mine, dtype=np.int32), device=dev)
        return self._dkg1, self._dkg2, self._tset

    # ---- one process per GPU (SURVEY §8e-i) ----------------------------------------------------------------------
    def _multi_mode(self):
        """How path (i) trains under torchrun (DESIGN.md §6).  'exact' (default): replicated tables, every step's batch
        sharded over the ranks, gradients all-reduced, identical updates — the accuracy of one GPU, no speed-up at these
        table sizes.  'seed': the north-star's stale-replica scheme that bench.py
        times (head-owner triple shards, seed-pair rows exchanged once per epoch over NVLink) — fast, but it loses accuracy,
        more as N grows, so it is opt-in: args.multi_gpu_mode or OEA_MULTI_MODE."""
        mode = getattr(self.args, "multi_gpu_mode", None) or os.environ.get("OEA_MULTI_MODE") or "exact"
        if mode not in ("exact", "seed"):
            raise ValueError("multi_gpu_mode must be 'exact' or 'seed', not %r" % (mode,))
        return mode

    def _sync_seed_rows(self):
        """'seed' mode, end of a local epoch: the owners' copies of the seed-pair rows go to every replica (the only
        data-path collective of that mode); replicas are otherwise stale."""
        rank, world = par.world()
        if world == 1 or self._multi_mode() != "seed":
            return
        if getattr(self, "_seed_sync", None) is None:
            seeds = np.asarray(self.kgs.train_links, dtype=np.int64).reshape(-1)
            self._seed_sync = par.SeedRowSync(self.ent_embeds.weight, seeds, rank, world)
        self._seed_sync.sync()

    def _sync_replicas(self):
        """Before anything that must agree across ranks (validation and its early-stop decision, test, bootstrapping,
        saving): every entity row from its owner, every other table averaged.  Afterwards the replicas are identical."""
        rank, world = par.world()
        if world == 1:
            return False
        if not isinstance(self.ent_embeds, eng.EmbeddingTable):
            return par.replicas_in_sync()     # the row-sharded GNN approaches keep every rank's outputs identical themselves
        import torch.distributed as dist
        par.assemble_owned_rows(self.ent_embeds.weight, rank, world)
        for name, tab in vars(self).items():
            if isinstance(tab, eng.EmbeddingTable) and tab is not self.ent_embeds:
                dist.all_reduce(tab.weight)
                tab.weight /= world
        return True

    # ---- evaluation ------------------------------------------------------------------------------------
    def _mapping_array(self):
        return None if self.mapping_mat is None else self.mapping_mat.raw()

    def _eval_valid_embeddings(self):
        if len(self.kgs.valid_links) > 0:
            embeds1 = self.ent_embeds.lookup(self.kgs.valid_entities1)
            embeds2 = self.ent_embeds.lookup(self.kgs.valid_entities2 + self.kgs.test_entities2)
        else:
            embeds1 = self.ent_embeds.lookup(self.kgs.test_entities1)
            embeds2 = self.ent_embeds.lookup(self.kgs.test_entities2)
        return embeds1, embeds2, self._mapping_array()

    def _eval_test_embeddings(self):
        embeds1 = self.ent_embeds.lookup(self.kgs.test_entities1)
        embeds2 = self.ent_embeds.lookup(self.kgs.test_entities2)
        return embeds1, embeds2, self._mapping_array()

    def valid(self, stop_metric):
        par.mark_replicas_in_sync(self._sync_replicas())
        embeds1, embeds2, mapping = self._eval_valid_embeddings()
        hits1_12, mrr_12 = valid(embeds1, embeds2, mapping, self.args.top_k,
                                 self.args.test_threads_num, metric=self.args.eval_metric,
                                 normalize=self.args.eval_norm, csls_k=0, accurate=False)
        return hits1_12 if stop_metric == 'hits1' else mrr_12

    def test(self, save=True):
        par.mark_replicas_in_sync(self._sync_replicas())
        embeds1, embeds2, mapping = self._eval_test_embeddings()
        rest_12, _, _ = test(embeds1, embeds2, mapping, self.args.top_k, self.args.test_threads_num,
                             metric=self.args.eval_metric, normalize=self.args.eval_norm, csls_k=0, accurate=True)
        test(embeds1, embeds2, mapping, self.args.top_k, self.args.test_threads_num,
             metric=self.args.eval_metric, normalize=self.args.eval_norm, csls_k=self.args.csls, accurate=True)
        if save:
            ent_ids_rest_12 = [(self.kgs.test_entities1[i], self.kgs.test_entities2[j]) for i, j in rest_12]
            rd.save_results(self.out_folder, ent_ids_rest_12)

    def retest(self):
        parts = self.out_folder.split("/")
        new_dir = "".join(p + "/" for p in parts[:len(parts) - 2])
        new_dir = new_dir + os.listdir(new_dir)[0] + "/"
        embeds = np.load(new_dir + "ent_embeds.npy")
        embeds1 = embeds[self.kgs.test_entities1]
        embeds2 = embeds[self.kgs.test_entities2]
        mapping = None
        print(self.__class__.__name__, type(self.__class__.__name__))
        if self.__class__.__name__ == "GCN_Align":
            print(self.__class__.__name__, "loads attr embeds")
            attr_embeds = np.load(new_dir + "attr_embeds.npy")
            beta = self.args.beta
            embeds1 = np.concatenate([embeds1 * beta, attr_embeds[self.kgs.test_entities1] * (1.0 - beta)], axis=1)
            embeds2 = np.concatenate([embeds2 * beta, attr_embeds[self.kgs.test_entities2] * (1.0 - beta)], axis=1)
        if os.path.exists(new_dir + "mapping_mat.npy"):
            print(self.__class__.__name__, "loads mapping mat")
            mapping = np.load(new_dir + "mapping_mat.npy")
        kw = dict(metric=self.args.eval_metric, normalize=self.args.eval_norm, csls_k=0, accurate=True)
        print("conventional test:")
        test(embeds1, embeds2, mapping, self.args.top_k, self.args.test_threads_num, **kw)
        print("conventional reversed test:")
        if mapping is not None:
            embeds1 = np.matmul(embeds1, mapping)
            test(embeds2, embeds1, None, self.args.top_k, self.args.test_threads_num, **kw)
        else:
            test(embeds2, embeds1, mapping, self.args.top_k, self.args.test_threads_num, **kw)
        print("stable test:")
        stable_alignment(embeds1, embeds2, self.args.eval_metric, self.args.eval_norm, csls_k=0,
                         nums_threads=self.args.test_threads_num)
        print("stable test with csls:")
        stable_alignment(embeds1, embeds2, self.args.eval_metric, self.args.eval_norm, csls_k=self.args.csls,
                         nums_threads=self.args.test_threads_num)

    def save(self):
        self._sync_replicas()          # under torchrun: the owners' rows everywhere; only rank 0 writes the files
        if par.world()[0] != 0:
            return
        ent_embeds = self.ent_embeds.lookup().cpu().numpy()      # what `self.ent_embeds.eval()` returns in TF
        rel_embeds = self.rel_embeds.lookup().cpu().numpy()
        mapping_mat = self.mapping_mat.raw().cpu().numpy() if self.mapping_mat is not None else None
        rd.save_embeddings(self.out_folder, self.kgs, ent_embeds, rel_embeds, None, mapping_mat=mapping_mat)

    def eval_kg1_ent_embeddings(self):
        return self.ent_embeds.lookup(self.kgs.kg1.entities_list).cpu().numpy()

    def eval_kg2_ent_embeddings(self):
        return self.ent_embeds.lookup(self.kgs.kg2.entities_list).cpu().numpy()

    def eval_kg1_useful_ent_embeddings(self):
        return self.ent_embeds.lookup(self.kgs.useful_entities_list1)

    def eval_kg2_useful_ent_embeddings(self):
        return self.ent_embeds.lookup(self.kgs.useful_entities_list2)

    # ---- training --------------------------------------------------------------------------------------
    def launch_training_1epo(self, epoch, triple_steps, steps_tasks, training_batch_queue, neighbors1, neighbors2):
        self.launch_triple_training_1epo(epoch, triple_steps, steps_tasks, training_batch_queue, neighbors1, neighbors2)
        if self.args.alignment_module == 'mapping':
            self.launch_mapping_training_1epo(epoch, triple_steps)
        self._sync_seed_rows()

    @staticmethod
    def _slice_count(n_triples, batch_kg, step):
        lo = min(step * batch_kg, n_triples)
        return max(0, min(lo + batch_kg, n_triples) - lo)

    def _install_candidates(self, kg1, kg2, neighbors1, neighbors2):
        """Hand the ε-truncated candidate tensors (or None) to the device KG views of the sampler."""
        for kg, nb, ents in ((kg1, neighbors1, self.kgs.useful_entities_list1),
                             (kg2, neighbors2, self.kgs.useful_entities_list2)):
            if nb is None:
                kg.clear_candidates()
            elif kg.cand_src is not nb:
                kg.set_candidates(nb, ents)

    def launch_triple_training_1epo(self, epoch, triple_steps, steps_tasks, batch_queue, neighbors1, neighbors2):
        """One epoch of fused device steps.  `steps_tasks` / `batch_queue` belong to the reference's producer
        processes and are ignored; neighbors1/2 are the ε-truncated candidate tensors (or None)."""
        start = time.time()
        kg1, kg2, tset = self._device_kgs()
        self._install_candidates(kg1, kg2, neighbors1, neighbors2)
        t1, t2 = kg1.triples.shape[0], kg2.triples.shape[0]
        b1 = int(t1 / (t1 + t2) * self.args.batch_size)
        b2 = self.args.batch_size - b1
        self._epoch_seed = (self._epoch_seed * 6364136223846793005 + 1442695040888963407) & ((1 << 63) - 1)
        trained_samples_num = 0
        trainer = self.triple_trainer
        # the first epoch of a process runs eagerly (module loading, occupancy queries and allocator warm-up must not
        # happen inside a stream capture; a resumed run starts at epoch > 1); the multi-table trainers read the step's
        # size back and are not captured
        # Adam's bias-corrected step size is a host-computed launch argument that changes every step: a replayed graph
        # would freeze it, so Adam-optimised models run their epochs eagerly
        use_graph = getattr(self.args, "cuda_graph", True) and getattr(self, "_ran_eager_epoch", False) and \
            hasattr(trainer, "capture_epoch") and getattr(self.ent_embeds, "optimizer", None) != "Adam"
        self._ran_eager_epoch = True
        exact = None
        if par.world()[1] > 1 and self._multi_mode() == "exact" and isinstance(trainer, eng.TripleTrainer):
            # batch sharded over the ranks, gradients all-reduced between scorer and optimiser (two launches + NCCL per step:
            # not graph-captured).  Trainers without a shardable scorer (the multi-table score family) run the whole batch
            # on every rank instead: replicas stay equal up to the order of the float reductions, and _sync_replicas
            # re-unifies them before anything that must agree.
            exact = getattr(self, "_exact_step", None)
            if exact is None or exact.trainer is not trainer:
                exact = self._exact_step = par.ExactReplicaStep(trainer)
            use_graph = False
        if use_graph:
            key = (triple_steps, trainer._views(kg1, kg2, tset) and trainer._view_key)
            if getattr(self, "_epoch_graph_key", None) != key:      # (re)capture: first use, or new candidate lists
                self._epoch_graph = trainer.capture_epoch(kg1, kg2, tset, self.args.batch_size, self.neg_per_pos,
                                                          triple_steps)
                self._epoch_graph_key = key
            self._epoch_graph.replay(self._epoch_seed)
        for step in range(triple_steps):
            if exact is not None:
                exact.step(kg1, kg2, tset, self.args.batch_size, self.neg_per_pos, step, self._epoch_seed)
            elif not use_graph:
                trainer.step_sampled(kg1, kg2, tset, self.args.batch_size, self.neg_per_pos, step, self._epoch_seed)
            trained_samples_num += self._slice_count(t1, b1, step) + self._slice_count(t2, b2, step)
        epoch_loss = trainer.read_loss() / max(1, trained_samples_num)     # one device→host read per epoch
        print('epoch {}, avg. triple loss: {:.4f}, cost time: {:.4f}s'.format(epoch, epoch_loss, time.time() - start))
        return epoch_loss

    def launch_mapping_training_1epo(self, epoch, triple_steps):
        start = time.time()
        # every step draws len(train_links) // triple_steps distinct seed pairs, independently of the other steps
        # (random.sample per step, basic_model.py:241-243): all steps' index sets in one device draw — the per-row
        # m largest of n random keys — and one loss read per epoch instead of one host sync per step
        dev = self.ent_embeds.device
        if getattr(self, "_links_dev", None) is None:
            self._links_dev = torch.as_tensor(np.asarray(self.kgs.train_links, dtype=np.int32).reshape(-1, 2), device=dev)
        n, m = self._links_dev.shape[0], len(self.kgs.train_links) // triple_steps
        picks = torch.rand(triple_steps, n, device=dev).topk(m, dim=1).indices if m > 0 else None
        self.mapping_trainer.loss_dev.zero_()
        for step in range(triple_steps if m > 0 else 0):
            batch = self._links_dev[picks[step]]
            self.mapping_trainer.step(batch[:, 0], batch[:, 1], read_loss=False)
        trained_samples_num = triple_steps * m
        epoch_loss = self.mapping_trainer.read_loss() / max(1, trained_samples_num)
        print('epoch {}, avg. mapping loss: {:.4f}, cost time: {:.4f}s'.format(epoch, epoch_loss, time.time() - start))
        return epoch_loss

    def _refresh_neighbours(self):
        """ε-truncated candidate lists of both KGs (basic_model.py:267-289), as device tensors."""
        assert 0.0 < self.args.truncated_epsilon < 1.0
        num1 = int((1 - self.args.truncated_epsilon) * self.kgs.kg1.entities_num)
        num2 = int((1 - self.args.truncated_epsilon) * self.kgs.kg2.entities_num)
        n1 = bat.neighbours_device(self.eval_kg1_useful_ent_embeddings(), self.kgs.useful_entities_list1, num1)
        n2 = bat.neighbours_device(self.eval_kg2_useful_ent_embeddings(), self.kgs.useful_entities_list2, num2)
        return n1, n2

    # ---- checkpoint / resume (absent in the reference, SURVEY §5 / §8f-4) -----------------------------------------
    def _checkpoint_tables(self):
        """Every optimiser instance that holds state: the model's tables by attribute name, plus the separate slot
        views of the mapping / alignment trainers (they share the weights of the tables above)."""
        tables = {name: v for name, v in vars(self).items() if isinstance(v, eng.EmbeddingTable)}
        for tname in ("mapping_trainer", "alignment_trainer"):
            trainer = getattr(self, tname, None)
            for slot in ("ent", "rel"):
                tab = getattr(trainer, slot, None)
                if isinstance(tab, eng.EmbeddingTable):
                    tables["%s.%s" % (tname, slot)] = tab
        return tables

    def save_checkpoint(self, path, epoch):
        """Everything a run needs to continue after `epoch`: variables, optimiser slots, the sampler's epoch seed,
        early-stopping state and the host RNG streams (mapping batches, GNN negatives)."""
        # RNG streams as plain ints / tensors so that the file loads with torch.load(weights_only=True): a checkpoint
        # from an untrusted source cannot run code at load time
        pr = random.getstate()
        nr = np.random.get_state()
        state = {"epoch": int(epoch), "epoch_seed": int(self._epoch_seed), "flag1": self.flag1, "flag2": self.flag2,
                 "class": self.__class__.__name__,
                 "python_random": {"version": int(pr[0]), "state": [int(x) for x in pr[1]], "gauss": pr[2]},
                 "numpy_random": {"kind": str(nr[0]), "keys": torch.from_numpy(np.asarray(nr[1], dtype=np.int64).copy()),
                                  "pos": int(nr[2]), "has_gauss": int(nr[3]), "cached": float(nr[4])},
                 "tables": {name: tab.state_dict() for name, tab in self._checkpoint_tables().items()},
                 "extra": self._extra_state()}
        # under torchrun every rank reaches this point with identical replicas (the callers sync first): rank 0 writes
        if par.world()[0] != 0:
            return path
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        tmp = path + ".tmp"
        torch.save(state, tmp)
        os.replace(tmp, path)
        return path

    def load_checkpoint(self, path):
        """Restore a save_checkpoint() file into an initialised model (call after init()); returns the epoch to
        continue from and makes run() start there."""
        state = torch.load(path, map_location="cpu", weights_only=True)
        if state["class"] != self.__class__.__name__:
            raise ValueError("checkpoint of %s loaded into %s" % (state["class"], self.__class__.__name__))
        tables = self._checkpoint_tables()
        if set(tables) != set(state["tables"]):
            raise ValueError("checkpoint tables %s do not match the model's %s" % (sorted(state["tables"]), sorted(tables)))
        for name, tab in tables.items():
            tab.load_state_dict(state["tables"][name])
        self._epoch_seed, self.flag1, self.flag2 = state["epoch_seed"], state["flag1"], state["flag2"]
        pr, nr = state["python_random"], state["numpy_random"]
        random.setstate((pr["version"], tuple(pr["state"]), pr["gauss"]))
        np.random.set_state((nr["kind"], nr["keys"].numpy().astype(np.uint32), nr["pos"], nr["has_gauss"], nr["cached"]))
        self._load_extra_state(state.get("extra") or {})
        self._start_epoch = state["epoch"] + 1
        return self._start_epoch

    def _extra_state(self):
        """Approach-specific state beyond tables and seeds (host tensors / plain Python), e.g. BootEA's labels."""
        return {}

    def _load_extra_state(self, extra):
        pass

    def _local_triples_num(self):
        """Training triples of this process: all of them, or this rank's head-owned shard under torchrun."""
        if par.world()[1] == 1:
            return self.kgs.kg1.relation_triples_num + self.kgs.kg2.relation_triples_num
        kg1, kg2, _ = self._device_kgs()
        return int(kg1.triples.shape[0] + kg2.triples.shape[0])

    def run(self):
        t = time.time()
        triples_num = self._local_triples_num()
        triple_steps = int(math.ceil(triples_num / self.args.batch_size))
        steps_tasks = task_divide(list(range(triple_steps)), self.args.batch_threads_num)
        neighbors1, neighbors2 = None, None
        start_epoch = getattr(self, "_start_epoch", 1)
        # ProjE's configuration names no neg_sampling (its batches are positives only)
        truncated = getattr(self.args, "neg_sampling", None) == 'truncated'
        if start_epoch > 1 and truncated and (start_epoch - 1) >= self.args.truncated_freq:
            neighbors1, neighbors2 = self._refresh_neighbours()     # the candidate lists are derived state: rebuild them
        every = getattr(self.args, "checkpoint_every", 0)
        for i in range(start_epoch, self.args.max_epoch + 1):
            self.launch_training_1epo(i, triple_steps, steps_tasks, None, neighbors1, neighbors2)
            if every and i % every == 0:
                self._sync_replicas()          # under torchrun: identical tables on every rank, rank 0 writes the file
                self.save_checkpoint(self.out_folder + "checkpoint.pt", i)
            if i >= self.args.start_valid and i % self.args.eval_freq == 0:
                flag = self.valid(self.args.stop_metric)
                self.flag1, self.flag2, self.early_stop = early_stop(self.flag1, self.flag2, flag)
                if self.early_stop or i == self.args.max_epoch:
                    break
            if truncated and i % self.args.truncated_freq == 0:
                t1 = time.time()
                neighbors1 = neighbors2 = None
                gc.collect()
                neighbors1, neighbors2 = self._refresh_neighbours()
                ent_num = len(self.kgs.kg1.entities_list) + len(self.kgs.kg2.entities_list)
                torch.cuda.synchronize()
                print("\ngenerating neighbors of {} entities costs {:.3f} s.".format(ent_num, time.time() - t1))
        print("Training ends. Total time = {:.3f} s.".format(time.time() - t))

    # ---- prediction --------------------------------------------------------------------------------------
    def predict(self, top_k=1, min_sim_value=None, output_file_name=None):
        """Correspondences that are in the top_k of their KG1 row or KG2 column (optionally above a confidence);
        returns [(uri1, uri2, similarity)] and optionally writes a TSV (basic_model.py:292-352)."""
        from openea_b200 import finding as F
        embeds1 = self.ent_embeds.lookup(self.kgs.kg1.entities_list)
        embeds2 = self.ent_embeds.lookup(self.kgs.kg2.entities_list)
        if self.mapping_mat is not None:
            embeds1 = embeds1 @ self.mapping_mat.raw()
        e1, e2, d = F._prep_pair(embeds1, embeds2, self.args.eval_metric, self.args.eval_norm)
        matched = {}
        if top_k:
            assert top_k > 0
            fwd = F.topk(e1, e2, d, self.args.eval_metric, top_k, want=("val", "idx"))
            bwd = F.topk(e2, e1, d, self.args.eval_metric, top_k, want=("val", "idx"))
            fi, fv = fwd["idx"].cpu().numpy(), fwd["val"].cpu().numpy()
            bi, bv = bwd["idx"].cpu().numpy(), bwd["val"].cpu().numpy()
            for i in range(fi.shape[0]):
                for j, v in zip(fi[i], fv[i]):
                    matched[(i, int(j))] = float(v)
            for j in range(bi.shape[0]):
                for i, v in zip(bi[j], bv[j]):
                    matched[(int(i), j)] = float(v)
        elif min_sim_value:
            s = F.sim_matrix(e1, e2, d, self.args.eval_metric)
            rows, cols = torch.nonzero(s > min_sim_value, as_tuple=True)
            vals = s[rows, cols].cpu().numpy()
            matched = {(int(i), int(j)): float(v) for i, j, v in zip(rows.cpu().numpy(), cols.cpu().numpy(), vals)}
        else:
            raise ValueError("Either top_k or min_sim_value should have a value")
        kg1_id_to_uri = {v: k for k, v in self.kgs.kg1.entities_id_dict.items()}
        kg2_id_to_uri = {v: k for k, v in self.kgs.kg2.entities_id_dict.items()}
        out = [(kg1_id_to_uri[self.kgs.kg1.entities_list[i]], kg2_id_to_uri[self.kgs.kg2.entities_list[j]], v)
               for (i, j), v in matched.items()]
        self._write_predictions(out, output_file_name)
        return out

    def predict_entities(self, entities_file_path, output_file_name=None):
        """Confidence of the given (entity1 \\t entity2) pairs (basic_model.py:354-412)."""
        from openea_b200 import finding as F
        kg1_entities, kg2_entities = [], []
        with open(entities_file_path, 'r', encoding='utf-8') as fh:
            for line in fh:
                a, b = line.strip('\n').split('\t')[:2]
                kg1_entities.append(self.kgs.kg1.entities_id_dict[a])
                kg2_entities.append(self.kgs.kg2.entities_id_dict[b])
        d1, d2 = sorted(set(kg1_entities)), sorted(set(kg2_entities))
        pos1 = {e: i for i, e in enumerate(d1)}
        pos2 = {e: i for i, e in enumerate(d2)}
        embeds1, embeds2 = self.ent_embeds.lookup(d1), self.ent_embeds.lookup(d2)
        if self.mapping_mat is not None:
            embeds1 = embeds1 @ self.mapping_mat.raw()
        e1, e2, d = F._prep_pair(embeds1, embeds2, self.args.eval_metric, self.args.eval_norm)
        s = F.sim_matrix(e1, e2, d, self.args.eval_metric).cpu().numpy()
        kg1_id_to_uri = {v: k for k, v in self.kgs.kg1.entities_id_dict.items()}
        kg2_id_to_uri = {v: k for k, v in self.kgs.kg2.entities_id_dict.items()}
        out = [(kg1_id_to_uri[a], kg2_id_to_uri[b], s[pos1[a], pos2[b]]) for a, b in zip(kg1_entities, kg2_entities)]
        self._write_predictions(out, output_file_name)
        return out

    def _write_predictions(self, rows, output_file_name):
        if output_file_name is None:
            return
        os.makedirs(self.out_folder, exist_ok=True)
        with open(self.out_folder + output_file_name, 'w', encoding='utf8') as fh:
            fh.writelines("%s\t%s\t%s\n" % (a, b, c) for a, b, c in rows)
        print(self.out_folder + output_file_name, "saved")
