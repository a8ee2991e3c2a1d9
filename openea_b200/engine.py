"""Host side of path (i): device-resident embedding tables, the triple trainer and device KG views.

PyTorch is used for device memory and streams only; every numeric operation goes through the C-ABI
of liboea.so (openea_b200.lib).  Nothing here falls back to PyTorch maths.

Reference boundary this mirrors: the TF variables + placeholders + session.run of
models/basic_model.py:73-98,211-236 (variables live on the device, index batches are fed).
"""
import ctypes as C
import math

import numpy as np
import torch

from . import lib as L

ADAGRAD_INIT_ACC = 0.1  # tf.train.AdagradOptimizer initial_accumulator_value (TF1 default)


def _stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def pitch_for(dim):
    """Internal row pitch: next multiple of 4 floats (16 B) so rows are float4-addressable (d=75 → 76)."""
    return (int(dim) + 3) // 4 * 4


def _grown(buf, need, device):
    """`buf` if it holds `need` bytes, else a new byte buffer of that size (at least 1 B) on `device`."""
    if buf is None or buf.numel() < need:
        buf = torch.empty(max(1, need), dtype=torch.uint8, device=device)
    return buf


class EmbeddingTable:
    """A TF-style embedding variable + optimiser slots on the device.

    `weight` is the RAW variable; when `l2_norm` every lookup goes through l2_normalize and gradients
    flow through it (modules/base/initializers.py:26,34,41,50).
    """

    def __init__(self, init, l2_norm, optimizer="Adagrad", device="cuda"):
        init = torch.as_tensor(init, dtype=torch.float32)
        rows, dim = init.shape
        self.rows, self.dim, self.pitch = int(rows), int(dim), pitch_for(dim)
        self.l2_norm = bool(l2_norm)
        self.device = torch.device(device)
        self.weight = torch.zeros(rows, self.pitch, dtype=torch.float32, device=self.device)
        self.weight[:, :dim] = init.to(self.device)
        self.grad = torch.zeros_like(self.weight)
        self.touched = torch.zeros(rows, dtype=torch.int32, device=self.device)
        self.optimizer = optimizer
        self.state1 = None
        self.state2 = None
        self.adam_t = 0
        self._make_state()
        self._struct = None

    def _make_state(self):
        if self.optimizer == "Adagrad":
            self.state1 = torch.full_like(self.weight, ADAGRAD_INIT_ACC)
            self.state1[:, self.dim:] = 1.0  # padding columns: g = 0 there, keep rsqrt finite
        elif self.optimizer == "Adam":
            self.state1 = torch.zeros_like(self.weight)
            self.state2 = torch.zeros_like(self.weight)
        elif self.optimizer == "Adadelta":       # tf.train.AdadeltaOptimizer: accum and accum_update start at 0
            self.state1 = torch.zeros_like(self.weight)
            self.state2 = torch.zeros_like(self.weight)
        elif self.optimizer in ("SGD", "GradientDescent"):
            self.optimizer = "SGD"
        else:
            raise ValueError("unsupported optimizer for the fused row optimiser: %s" % self.optimizer)

    def new_slots(self):
        """A second optimiser instance over the same variable (each generate_optimizer call in the
        reference owns its slot variables, SURVEY A.3): returns a view sharing weight/grad/touched."""
        other = object.__new__(EmbeddingTable)
        other.__dict__.update(self.__dict__)
        other._struct = None
        other._make_state()
        other.adam_t = 0
        return other

    def state_dict(self):
        """Variable + this optimiser instance's slots as host tensors (checkpointing; the reference has none, SURVEY §5)."""
        cpu = lambda t: None if t is None else t.detach().cpu().clone()
        return {"weight": cpu(self.weight), "state1": cpu(self.state1), "state2": cpu(self.state2),
                "adam_t": int(self.adam_t), "optimizer": self.optimizer, "l2_norm": self.l2_norm, "dim": self.dim}

    def load_state_dict(self, state):
        """Restore in place (device buffers keep their addresses, so cached C structs and CUDA graphs stay valid)."""
        if state["optimizer"] != self.optimizer or state["dim"] != self.dim or tuple(state["weight"].shape) != tuple(self.weight.shape):
            raise ValueError("checkpoint does not match this table (optimizer %s/%s, shape %s/%s)" % (
                state["optimizer"], self.optimizer, tuple(state["weight"].shape), tuple(self.weight.shape)))
        self.weight.copy_(state["weight"])
        for name in ("state1", "state2"):
            if getattr(self, name) is not None:
                getattr(self, name).copy_(state[name])
        self.adam_t = int(state["adam_t"])
        self.grad.zero_()
        self.touched.zero_()

    def c_struct(self):
        if self._struct is None:
            self._struct = L.Table(self.weight.data_ptr(), self.grad.data_ptr(),
                                   0 if self.state1 is None else self.state1.data_ptr(),
                                   0 if self.state2 is None else self.state2.data_ptr(),
                                   self.touched.data_ptr(), self.rows, self.dim, self.pitch, int(self.l2_norm))
        return self._struct

    def raw(self):
        return self.weight[:, :self.dim]

    def lookup(self, ids=None, padded=False):
        """Normalised rows as TF's `embedding_lookup(self.ent_embeds, ids).eval()` → device tensor [n, dim]
        (or [n, pitch] zero-padded when `padded`, the layout the SpMM / similarity kernels take)."""
        lib = L.load()
        if ids is None:
            n, ids_t = self.rows, None
        else:
            ids_t = torch.as_tensor(ids, dtype=torch.int32, device=self.device).contiguous()
            n = ids_t.numel()
        width = self.pitch if padded else self.dim
        out = torch.empty(n, width, dtype=torch.float32, device=self.device)
        L.check(lib.oea_table_lookup(C.byref(self.c_struct()), _ptr(ids_t), n, _ptr(out), width, _stream_ptr()),
                "oea_table_lookup")
        return out

    def scatter_grad(self, grad_rows, ids=None):
        """Backward of lookup(): push d loss / d (normalised rows) through the normalisation into self.grad."""
        lib = L.load()
        if ids is None:
            if getattr(self, "_all_ids", None) is None:
                self._all_ids = torch.arange(self.rows, dtype=torch.int32, device=self.device)
            ids_t = self._all_ids
        else:
            ids_t = torch.as_tensor(ids, dtype=torch.int32, device=self.device).contiguous()
        L.check(lib.oea_table_scatter_grad(C.byref(self.c_struct()), _ptr(ids_t), ids_t.numel(), _ptr(grad_rows),
                                           grad_rows.stride(0), _stream_ptr()), "oea_table_scatter_grad")

    def apply(self, lr):
        """One optimiser step on this table with its own slots (oea_rowopt_apply)."""
        lib = L.load()
        if self.optimizer == "Adam":
            self.adam_t += 1
        cfg = opt_cfg(self, lr)
        L.check(lib.oea_rowopt_apply(C.byref(self.c_struct()), C.byref(cfg), _stream_ptr()), "oea_rowopt_apply")


def loss_cfg(loss, loss_norm, margin=0.0, neg_margin=0.0, balance=1.0):
    kinds = {"margin-based": L.LOSS_MARGIN, "limited": L.LOSS_LIMITED, "logistic": L.LOSS_LOGISTIC,
             "positive": L.LOSS_POSITIVE, "logsigmoid": L.LOSS_LOGSIGMOID}
    if loss not in kinds:
        raise ValueError("unknown loss %r" % (loss,))
    score = L.SCORE_L1 if loss_norm == "L1" else L.SCORE_L2SQ  # losses.py: anything but 'L1' is squared L2
    return L.LossCfg(score, kinds[loss], float(margin), float(neg_margin), float(balance))


def opt_cfg(table, lr):
    kind = {"SGD": L.OPT_SGD, "Adagrad": L.OPT_ADAGRAD, "Adam": L.OPT_ADAM, "Adadelta": L.OPT_ADADELTA}[table.optimizer]
    if kind == L.OPT_ADADELTA:      # TF1 defaults rho = 0.95, epsilon = 1e-8 (beta1 carries rho)
        return L.OptCfg(kind, float(lr), 0.95, 0.0, 1e-8, 1)
    return L.OptCfg(kind, float(lr), 0.9, 0.999, 1e-8, max(1, table.adam_t))


class DeviceKG:
    """Device copy of one KG's training triples + candidate lists (oea_kg_view)."""

    def __init__(self, triples, entities, ent_rows, device="cuda"):
        self.device = torch.device(device)
        tri = np.asarray(triples, dtype=np.int32).reshape(-1, 3)
        self.triples = torch.from_numpy(np.ascontiguousarray(tri)).to(self.device)
        self.entities = torch.as_tensor(np.asarray(entities, dtype=np.int32), device=self.device)
        self.ent_rows = int(ent_rows)
        self.cand = None
        self.ent2row = None
        self.cand_src = None

    def set_candidates(self, cand, row_entities, direct=True):
        """cand: [rows, n_cand] int32 device tensor of ε-truncated neighbour ids; row_entities: the entity id
        owning each row (batch.py:145-165 builds dict entity → list)."""
        rows = torch.as_tensor(row_entities, dtype=torch.int64, device=self.device)
        self.cand_src = cand          # identity of the caller's tensor (lets callers skip redundant re-installs)
        if direct:   # candidate matrix indexed by entity id: the sampler skips the ent2row indirection
            full = torch.full((self.ent_rows, cand.shape[1]), -1, dtype=torch.int32, device=self.device)
            full[rows] = cand
            self.cand, self.ent2row = full, None
            return
        self.cand = cand.contiguous()
        e2r = torch.full((self.ent_rows,), -1, dtype=torch.int32, device=self.device)
        e2r[rows] = torch.arange(rows.numel(), dtype=torch.int32, device=self.device)
        self.ent2row = e2r

    def clear_candidates(self):
        self.cand = None
        self.ent2row = None
        self.cand_src = None

    def view(self):
        return L.KgView(self.triples.data_ptr(), self.triples.shape[0], self.entities.data_ptr(),
                        self.entities.numel(), 0 if self.cand is None else self.cand.data_ptr(),
                        0 if self.ent2row is None else self.ent2row.data_ptr(),
                        0 if self.cand is None else self.cand.shape[1])


def _pcg32(x):
    """pcg32 of oea_common.cuh on int64 tensors holding 32-bit values (every product stays below 2^63)."""
    x = (x * 747796405 + 2891336453) & 0xFFFFFFFF
    w = (((x >> ((x >> 28) + 4)) ^ x) * 277803737) & 0xFFFFFFFF
    return (w >> 22) ^ w


def tripleset_filter(slots):
    """The blocked Bloom filter of the keys held in `slots` (int64, empty = -1): int64 words, a power of two of them
    and at least 16 bits per key.  Restates tset_filter_hash / tset_filter_bits of oea_common.cuh: a key sets four
    bits of one word."""
    keys = slots[slots != -1]
    n_words = 1 << (max(1, (keys.numel() + 3) // 4) - 1).bit_length()
    fh = _pcg32((keys >> 32) ^ _pcg32((keys & 0xFFFFFFFF) ^ 0x2545F491))
    b = _pcg32(fh ^ 0x68E31DA4)
    word = (fh & (n_words - 1)) * 64
    bitmap = torch.zeros(n_words * 64, dtype=torch.bool, device=slots.device)
    for shift in (0, 6, 12, 18):
        bitmap[word + ((b >> shift) & 63)] = True
    weights = torch.ones(64, dtype=torch.int64, device=slots.device) << torch.arange(64, device=slots.device)
    return (bitmap.view(n_words, 64).to(torch.int64) * weights).sum(1)


class DeviceTripleSet:
    """Open-addressing membership set of (h, r, t) built on device (oea_tripleset_build), with the blocked Bloom
    filter that answers most "absent" queries from L2 (tripleset_filter)."""

    def __init__(self, triple_tensors, n_ent, n_rel, device="cuda"):
        lib = L.load()
        self.device = torch.device(device)
        allt = torch.cat([t.reshape(-1, 3) for t in triple_tensors], dim=0).contiguous()
        n = allt.shape[0]
        self.ent_bits = max(1, int(math.ceil(math.log2(max(2, n_ent)))))
        self.rel_bits = max(1, int(math.ceil(math.log2(max(2, n_rel)))))
        cap = 1 << max(4, int(math.ceil(math.log2(max(2, 2 * n)))))
        self.slots = torch.empty(cap, dtype=torch.int64, device=self.device)
        self.capacity = cap
        L.check(lib.oea_tripleset_build(_ptr(allt), n, _ptr(self.slots), cap, self.ent_bits, self.rel_bits,
                                        _stream_ptr()), "oea_tripleset_build")
        self.filter = tripleset_filter(self.slots)

    def view(self):
        return L.TripleSet(self.slots.data_ptr(), self.capacity, self.ent_bits, self.rel_bits, self.filter.data_ptr(),
                           self.filter.numel())


class TripleTrainer:
    """Forward/backward + optimiser for one (loss, optimiser instance) over the entity/relation tables."""

    def __init__(self, ent, rel, loss, lr):
        self.lib = L.load()
        self.ent, self.rel = ent, rel
        self.loss = loss
        self.lr = float(lr)
        dev = ent.device
        self.loss_dev = torch.zeros(1, dtype=torch.float64, device=dev)
        self._idx_ws = None
        self._loss_pinned = torch.zeros(1, dtype=torch.float64).pin_memory() if dev.type == "cuda" else None

    # -- device-index API -------------------------------------------------------------------------
    def score_fed(self, pos, neg=None, loss_out=None, grouped=False):
        """pos/neg: int32 device tensors [3, n] (h | r | t rows).  Accumulates gradients; adds the batch
        loss into loss_out (device fp64 scalar tensor, default self.loss_dev).  grouped: the negatives of positive p are
        columns p·k … p·k+k−1 (the reference's batch layout) → one warp per positive and its negatives
        (oea_triple_score_fed_grouped; same result)."""
        out = self.loss_dev if loss_out is None else loss_out
        n_pos = pos.shape[1]
        n_neg = 0 if neg is None else neg.shape[1]
        np_ = lambda t, i: C.c_void_p(0 if t is None or t.shape[1] == 0 else t[i].data_ptr())
        fn = self.lib.oea_triple_score_fed_grouped if grouped else self.lib.oea_triple_score_fed
        L.check(fn(
            C.byref(self.ent.c_struct()), C.byref(self.rel.c_struct()),
            np_(pos, 0), np_(pos, 1), np_(pos, 2), n_pos, np_(neg, 0), np_(neg, 1), np_(neg, 2), n_neg,
            C.byref(self.loss), _ptr(out), _stream_ptr()), "oea_triple_score_fed")

    def step_fed_grouped(self, pos, neg=None, loss_out=None):
        """score_fed(grouped=True) + apply() as one cooperative launch (oea_triple_step_fed_grouped); raises OeaError
        where the one-launch kernel does not apply (L1 score, pitch > 256, Adam / Adadelta)."""
        out = self.loss_dev if loss_out is None else loss_out
        n_pos = pos.shape[1]
        n_neg = 0 if neg is None else neg.shape[1]
        np_ = lambda t, i: C.c_void_p(0 if t is None or t.shape[1] == 0 else t[i].data_ptr())
        cfg = opt_cfg(self.ent, self.lr)
        L.check(self.lib.oea_triple_step_fed_grouped(
            C.byref(self.ent.c_struct()), C.byref(self.rel.c_struct()),
            np_(pos, 0), np_(pos, 1), np_(pos, 2), n_pos, np_(neg, 0), np_(neg, 1), np_(neg, 2), n_neg,
            C.byref(self.loss), C.byref(cfg), _ptr(out), _stream_ptr()), "oea_triple_step_fed_grouped")

    def score_margin_weighted(self, pos, neg, weights=None, reciprocal=False, scale=1.0, paths=False, loss_out=None):
        """scale · Σ wᵢ · relu(margin + s(posᵢ) − s(negᵢ)) forward + backward (oea_triple_score_margin_weighted;
        iptranse.py:170-180).  pos / neg: int32 device tensors [3, n]; weights: float32 device tensor [n] or None;
        reciprocal: wᵢ = 1 / weights[i]; paths: the columns are (r_x, r_y, r) relation ids and all three rows come from
        the relation table (the path loss).  margin and norm are this trainer's loss configuration."""
        out = self.loss_dev if loss_out is None else loss_out
        n = pos.shape[1]
        if neg.shape[1] != n or (weights is not None and weights.numel() != n):
            raise ValueError("weighted margin loss pairs positive i with negative i and weight i")
        if weights is not None:
            weights = weights.to(torch.float32).contiguous()
        a = self.rel if paths else self.ent
        np_ = lambda t, i: C.c_void_p(0 if n == 0 else t[i].data_ptr())
        L.check(self.lib.oea_triple_score_margin_weighted(
            C.byref(a.c_struct()), C.byref(self.rel.c_struct()), np_(pos, 0), np_(pos, 1), np_(pos, 2),
            np_(neg, 0), np_(neg, 1), np_(neg, 2), n, _ptr(weights), L.WEIGHT_RECIPROCAL if reciprocal else L.WEIGHT_DIRECT,
            float(scale), C.byref(self.loss), _ptr(out), _stream_ptr()), "oea_triple_score_margin_weighted")

    def score_pairs(self, ids_a, ids_b, weights=None, scale=1.0, loss_out=None):
        """scale · Σ wᵢ · ‖ê_a − ê_b‖² over entity pairs, forward + backward (oea_pair_distance_loss; imuse.py:303-306)."""
        out = self.loss_dev if loss_out is None else loss_out
        dev = self.ent.device
        a = torch.as_tensor(ids_a, dtype=torch.int32, device=dev).contiguous()
        b = torch.as_tensor(ids_b, dtype=torch.int32, device=dev).contiguous()
        if a.numel() != b.numel() or (weights is not None and weights.numel() != a.numel()):
            raise ValueError("pair loss needs one id of each side (and one weight) per pair")
        if weights is not None:
            weights = weights.to(torch.float32).contiguous()
        L.check(self.lib.oea_pair_distance_loss(C.byref(self.ent.c_struct()), _ptr(a), _ptr(b), a.numel(), _ptr(weights),
                                                float(scale), _ptr(out), _stream_ptr()), "oea_pair_distance_loss")

    def apply(self):
        for tab in (self.ent, self.rel):
            if tab.optimizer == "Adam":
                tab.adam_t += 1
        cfg = opt_cfg(self.ent, self.lr)
        L.check(self.lib.oea_rowopt_apply_pair(C.byref(self.ent.c_struct()), C.byref(self.rel.c_struct()), C.byref(cfg),
                                               _stream_ptr()), "oea_rowopt_apply_pair")

    def step_sampled(self, kg1, kg2, tset, batch_size, neg_per_pos, step, epoch_seed, max_try=10, n_pos_out=None,
                     dev_seed=None):
        """One whole training step in one C call (fused sampler+scorer, then one optimiser launch)."""
        smp = L.SampleCfg(int(batch_size), int(neg_per_pos), int(step), int(max_try), int(epoch_seed) & (2**64 - 1),
                          0 if dev_seed is None else dev_seed.data_ptr())
        views = self._views(kg1, kg2, tset)
        for tab in (self.ent, self.rel):
            if tab.optimizer == "Adam":
                tab.adam_t += 1
        cfg = opt_cfg(self.ent, self.lr)
        L.check(self.lib.oea_triple_step_sampled(
            C.byref(self.ent.c_struct()), C.byref(self.rel.c_struct()), C.byref(views[0]), C.byref(views[1]),
            C.byref(views[2]), C.byref(smp), C.byref(self.loss), C.byref(cfg), _ptr(self.loss_dev), _ptr(n_pos_out),
            _stream_ptr()), "oea_triple_step_sampled")

    def capture_epoch(self, kg1, kg2, tset, batch_size, neg_per_pos, steps, max_try=10):
        """CUDA graph of one whole epoch (`steps` × [fused sampler/scorer, optimiser]).  The per-epoch seed lives in
        a device scalar, so the same graph is replayed every epoch: `EpochGraph.replay(seed)`.  Must be re-captured
        when the candidate lists (device pointers) change."""
        return EpochGraph(self, kg1, kg2, tset, batch_size, neg_per_pos, steps, max_try)

    def _views(self, kg1, kg2, tset):
        """ctypes views of the KGs / triple set, cached until their device buffers change."""
        key = (kg1.triples.data_ptr(), kg2.triples.data_ptr(), 0 if kg1.cand is None else kg1.cand.data_ptr(),
               0 if kg2.cand is None else kg2.cand.data_ptr(), tset.slots.data_ptr())
        if getattr(self, "_view_key", None) != key:
            self._view_key = key
            self._view_val = (kg1.view(), kg2.view(), tset.view())
        return self._view_val

    def score_sampled(self, kg1, kg2, tset, batch_size, neg_per_pos, step, epoch_seed, max_try=10,
                      loss_out=None, dbg=None, n_pos_out=None, shard=None):
        """Fused sampler + scorer, gradients accumulated (no optimiser).  shard = (rank, world): score only the positives
        p ≡ rank (mod world) of the step's batch — the exact-parity multi-GPU mode (parallel.ExactReplicaStep)."""
        out = self.loss_dev if loss_out is None else loss_out
        sr, sw = (0, 0) if shard is None else (int(shard[0]), int(shard[1]))
        smp = L.SampleCfg(int(batch_size), int(neg_per_pos), int(step), int(max_try), int(epoch_seed) & (2**64 - 1), 0, sr, sw)
        k1, k2, ts = kg1.view(), kg2.view(), tset.view()
        L.check(self.lib.oea_triple_score_sampled(
            C.byref(self.ent.c_struct()), C.byref(self.rel.c_struct()), C.byref(k1), C.byref(k2), C.byref(ts),
            C.byref(smp), C.byref(self.loss), _ptr(out), _ptr(n_pos_out), _ptr(dbg), _stream_ptr()),
            "oea_triple_score_sampled")

    # -- host-index API (the session.run(feed_dict) boundary) --------------------------------------
    def step_fed_host(self, pos_hrt, neg_hrt=None):
        """pos_hrt / neg_hrt: host int32 arrays [3, n] (pinned torch tensors or numpy).  Synchronous; returns
        the batch loss as a Python float (what session.run returns for `triple_loss`)."""
        pos_t = _as_host_i32(pos_hrt)
        neg_t = _as_host_i32(neg_hrt) if neg_hrt is not None else None
        n_pos = pos_t.shape[1]
        n_neg = 0 if neg_t is None else neg_t.shape[1]
        need = 3 * (n_pos + n_neg)
        if self._idx_ws is None or self._idx_ws.numel() < need:
            self._idx_ws = torch.empty(max(need, 1), dtype=torch.int32, device=self.ent.device)
        for tab in (self.ent, self.rel):
            if tab.optimizer == "Adam":
                tab.adam_t += 1
        cfg = opt_cfg(self.ent, self.lr)
        loss = C.c_float(0.0)
        L.check(self.lib.oea_triple_step_fed_host(
            C.byref(self.ent.c_struct()), C.byref(self.rel.c_struct()),
            C.c_void_p(pos_t.data_ptr()), n_pos, C.c_void_p(0 if neg_t is None else neg_t.data_ptr()), n_neg,
            C.byref(self.loss), C.byref(cfg), _ptr(self._idx_ws), _ptr(self.loss_dev),
            C.c_void_p(self._loss_pinned.data_ptr()), C.byref(loss), _stream_ptr()), "oea_triple_step_fed_host")
        return float(loss.value)

    def read_loss(self, reset=True):
        v = float(self.loss_dev.item())
        if reset:
            self.loss_dev.zero_()
        return v


MODEL_KINDS = {"TransE": L.MODEL_TRANSE, "TransH": L.MODEL_TRANSH, "TransD": L.MODEL_TRANSD,
               "DistMult": L.MODEL_DISTMULT, "SimplE": L.MODEL_SIMPLE, "RotatE": L.MODEL_ROTATE, "HolE": L.MODEL_HOLE,
               "TransR": L.MODEL_TRANSR}

ROTATE_EPSILON = 2.0      # rotate.py:25: the embedding range is (γ + ε) / dim


def rotate_phase(gamma, dim):
    """π/ρ with ρ = (γ + 2)/dim: the factor that turns a relation entry into its phase (rotate.py:37,86,90)."""
    return math.pi / ((float(gamma) + ROTATE_EPSILON) / int(dim))


class ModelTrainer:
    """Forward/backward + optimiser for the score functions beyond plain translation (oea_model_score_fed):
    TransH / TransD / DistMult / SimplE / RotatE / HolE / TransR graphs of the reference's models/ (SURVEY §8f-2).

    tables = (ent, rel, ent_aux, rel_aux) EmbeddingTables in the slot order of `oea_model` (None where a model has
    no such table).  A step = device batch producer (oea_triple_sample_batch) → fed scorer → one row-optimiser
    launch per table; `mean_loss` applies DistMult's reduce_mean (distmult.py:58).  `gamma`: RotatE's γ (the phase
    scale follows from it and the dimension).  `neg_weight`: weight of the negatives' loss relative to the positives'
    (RotatE's 1/k, rotate.py:81); None = the same weight.  TransR (rel_aux = the matrix table, R·d rows of width d)
    is scored by oea_transr_score_fed, in a workspace the trainer owns and grows on demand."""

    def __init__(self, model, tables, loss, lr, mean_loss=False, sampler="fast", gamma=None, neg_weight=None):
        self.lib = L.load()
        self.kind = MODEL_KINDS[model]
        self.tables = tuple(tables) + (None,) * (4 - len(tables))
        self.live = [t for t in self.tables if t is not None]
        self.loss, self.lr = loss, float(lr)
        self.mean_loss = bool(mean_loss)
        self.sampler = {"fast": 0, "independent": 1}[sampler]
        if self.kind == L.MODEL_ROTATE and gamma is None:
            raise ValueError("RotatE needs its margin gamma")
        self.gamma = 0.0 if gamma is None else float(gamma)
        self.phase = rotate_phase(gamma, self.tables[0].dim) if self.kind == L.MODEL_ROTATE else 0.0
        self.neg_weight = None if neg_weight is None else float(neg_weight)
        dev = self.tables[0].device
        self.loss_dev = torch.zeros(1, dtype=torch.float64, device=dev)
        self._idx = None
        self._n_pos = C.c_int32(0)
        self._ws = None

    def _workspace(self, n_pos, n_neg):
        """TransR's scratch (bucketed triple ids, chunk list, scores, projections) for a batch of this size."""
        need = self.lib.oea_transr_workspace_bytes(n_pos, n_neg, self.tables[0].dim, self.tables[1].rows)
        self._ws = _grown(self._ws, need, self.tables[0].device)
        return self._ws

    def _c_model(self):
        # the Table structs are owned by the EmbeddingTables (cached there), so the pointers stay valid
        ptr = lambda t: C.pointer(t.c_struct()) if t is not None else None
        return L.Model(self.kind, *[ptr(t) for t in self.tables], self.gamma, self.phase)

    def score_fed(self, pos, neg=None, loss_out=None, scale=None, neg_scale=None):
        """pos / neg: int32 device tensors [3, n] (h | r | t rows); accumulates gradients into every table and adds
        the batch loss into loss_out (default self.loss_dev).  `scale` multiplies loss and gradient (default 1, or
        1 / batch for `mean_loss`); it may be negative (JAPE's −α·Σ s⁻ term).  `neg_scale` (default scale·neg_weight,
        or scale when the trainer has no neg_weight) multiplies the negatives' part instead: the positives and the
        negatives are then scored by two calls."""
        out = self.loss_dev if loss_out is None else loss_out
        n_pos = pos.shape[1]
        n_neg = 0 if neg is None else neg.shape[1]
        if scale is None:
            scale = 1.0 / max(1, n_pos + n_neg) if self.mean_loss else 1.0
        if neg_scale is None and self.neg_weight is not None:
            neg_scale = scale * self.neg_weight
        np_ = lambda t, i: C.c_void_p(0 if t is None or t.shape[1] == 0 else t[i].data_ptr())
        model = self._c_model()

        def call(p, n_p, n, n_n, s):
            if self.kind == L.MODEL_TRANSR:
                ws = self._workspace(n_p, n_n)
                L.check(self.lib.oea_transr_score_fed(
                    C.byref(model), np_(p, 0), np_(p, 1), np_(p, 2), n_p, np_(n, 0), np_(n, 1), np_(n, 2), n_n,
                    C.byref(self.loss), s, _ptr(ws), ws.numel(), _ptr(out), _stream_ptr()), "oea_transr_score_fed")
                return
            L.check(self.lib.oea_model_score_fed(
                C.byref(model), np_(p, 0), np_(p, 1), np_(p, 2), n_p, np_(n, 0), np_(n, 1), np_(n, 2), n_n,
                C.byref(self.loss), s, _ptr(out), _stream_ptr()), "oea_model_score_fed")
        if neg_scale is None or n_neg == 0 or neg_scale == scale:
            call(pos, n_pos, neg, n_neg, scale)
        else:
            call(pos, n_pos, None, 0, scale)
            call(None, 0, neg, n_neg, neg_scale)

    def apply(self):
        for tab in self.live:
            tab.apply(self.lr)

    def sample_batch(self, kg1, kg2, tset, batch_size, neg_per_pos, step, epoch_seed, max_try=10):
        """The device batch producer: returns (pos [3, n_pos], neg [3, n_pos·k] or None) int32 device tensors."""
        need = 3 * batch_size * (1 + neg_per_pos)
        if self._idx is None or self._idx.numel() < need:
            self._idx = torch.empty(need, dtype=torch.int32, device=self.tables[0].device)
        smp = L.SampleCfg(int(batch_size), int(neg_per_pos), int(step), int(max_try), int(epoch_seed) & (2**64 - 1), 0)
        k1, k2, ts = kg1.view(), kg2.view(), tset.view()
        pos_buf, neg_buf = self._idx[:3 * batch_size], self._idx[3 * batch_size:]
        L.check(self.lib.oea_triple_sample_batch(
            C.byref(k1), C.byref(k2), C.byref(ts), C.byref(smp), self.sampler, C.byref(self.tables[0].c_struct()),
            _ptr(pos_buf), _ptr(neg_buf), C.byref(self._n_pos), _stream_ptr()), "oea_triple_sample_batch")
        n = int(self._n_pos.value)
        pos = pos_buf[:3 * n].view(3, n)
        neg = neg_buf[:3 * n * neg_per_pos].view(3, n * neg_per_pos) if neg_per_pos > 0 else None
        return pos, neg

    def step_sampled(self, kg1, kg2, tset, batch_size, neg_per_pos, step, epoch_seed, max_try=10, **_):
        """One whole training step (what one session.run([triple_loss, triple_optimizer]) does)."""
        pos, neg = self.sample_batch(kg1, kg2, tset, batch_size, neg_per_pos, step, epoch_seed, max_try)
        if pos.shape[1] == 0:
            return 0
        self.score_fed(pos, neg)
        self.apply()
        return pos.shape[1]

    def read_loss(self, reset=True):
        v = float(self.loss_dev.item())
        if reset:
            self.loss_dev.zero_()
        return v


class SampledNceTrainer:
    """What every step on the sampled-NCE head shares: TF's unique log-uniform sampler on the device
    (oea_logu_sample_unique; one set of `num_sampled` classes per step, seeded from the epoch seed and the step) into
    `sampled` / `num_tries`, the loss accumulated on the device (`loss_dev`, read_loss), a workspace that grows on demand
    and one optimiser step over every table.  `n_classes` is the rows of the class table."""

    def __init__(self, tables, num_sampled, lr, n_classes):
        self.lib = L.load()
        self.tables = tuple(tables)
        self.num_sampled = int(num_sampled)
        self.n_classes = int(n_classes)
        if not 1 <= self.num_sampled <= self.n_classes:
            raise ValueError("nce_loss samples %d distinct classes out of %d: the sampler's range is too small"
                             % (self.num_sampled, self.n_classes))
        self.lr = float(lr)
        dev = self.tables[0].device
        self.loss_dev = torch.zeros(1, dtype=torch.float64, device=dev)
        self.sampled = torch.zeros(self.num_sampled, dtype=torch.int32, device=dev)
        self.num_tries = torch.zeros(1, dtype=torch.int32, device=dev)
        self._ws = None

    def _workspace(self, n):
        """The step's scratch for a batch of n (n = 0: the sampler's alone); _workspace_bytes(n) sizes it."""
        self._ws = _grown(self._ws, self._workspace_bytes(n), self.tables[0].device)
        return self._ws

    def sample(self, seed):
        """Draw the step's sampled set into self.sampled / self.num_tries (device; no host synchronisation)."""
        ws = self._workspace(0)
        L.check(self.lib.oea_logu_sample_unique(self.n_classes, self.num_sampled, int(seed) & (2**64 - 1),
                                                _ptr(self.sampled), _ptr(self.num_tries), _ptr(ws), ws.numel(),
                                                _stream_ptr()), "oea_logu_sample_unique")

    def _score(self, fn, model, ids, n, sampled, num_tries, loss_out, *step_args):
        """fn(model, *ids, n, sampled, num_tries, S, *step_args, workspace, its bytes, loss_out, stream): sampled /
        num_tries default to the last sample(), loss_out to loss_dev."""
        sampled = self.sampled if sampled is None else sampled
        num_tries = self.num_tries if num_tries is None else num_tries
        ws = self._workspace(n)
        L.check(getattr(self.lib, fn)(C.byref(model), *ids, n, _ptr(sampled), _ptr(num_tries), sampled.numel(),
                                      *step_args, _ptr(ws), ws.numel(),
                                      _ptr(self.loss_dev if loss_out is None else loss_out), _stream_ptr()), fn)

    def apply(self):
        for tab in self.tables:
            tab.apply(self.lr)

    @staticmethod
    def step_seed(epoch_seed, step):
        """The sampler's seed of one step: a function of (epoch seed, step) only, so that a resumed run draws the same."""
        return (int(epoch_seed) * 0x9E3779B97F4A7C15 + int(step) + 1) & (2**64 - 1)

    def read_loss(self, reset=True):
        v = float(self.loss_dev.item())
        if reset:
            self.loss_dev.zero_()
        return v


def _pos_rows(pos):
    """The h, r and t rows of a [3, n] int32 device batch as C pointers (NULL for an empty batch)."""
    return [C.c_void_p(0 if pos.shape[1] == 0 else pos[i].data_ptr()) for i in range(3)]


class ProjETrainer(SampledNceTrainer):
    """ProjE's step (models/neural/proje.py:46-96): device batch producer (oea_triple_sample_batch, positives only) →
    the sampler → the projection layer and the NCE head (oea_proje_score_fed) → Adam on the five tables.
    tables = (ent, rel, cls_w, cls_b, params) EmbeddingTables: entity_w, entity_b as [E, 1], and the [4, d] table of
    mlp_w, mlp_bias and the two batch-norm betas."""

    def __init__(self, tables, num_sampled, lr, sampler="fast"):
        super().__init__(tables, num_sampled, lr, tables[2].rows)
        self.sampler = {"fast": 0, "independent": 1}[sampler]
        self._idx = None
        self._n_pos = C.c_int32(0)

    def _workspace_bytes(self, n_pos):
        return self.lib.oea_proje_workspace_bytes(n_pos, self.num_sampled, self.tables[0].dim, self.n_classes)

    def score_fed(self, pos, sampled=None, num_tries=None, loss_out=None):
        """pos: int32 device tensor [3, n] (h | r | t rows); sampled / num_tries: int32 device tensors (default: the
        last sample()).  Accumulates gradients into the five tables and adds the batch loss into loss_out."""
        self._score("oea_proje_score_fed", L.Proje(*[C.pointer(t.c_struct()) for t in self.tables]), _pos_rows(pos),
                    pos.shape[1], sampled, num_tries, loss_out)

    def sample_batch(self, kg1, kg2, tset, batch_size, step, epoch_seed, max_try=10):
        """The device batch producer with no negatives: pos [3, n_pos] int32 device tensor."""
        if self._idx is None or self._idx.numel() < 3 * batch_size:
            self._idx = torch.empty(3 * batch_size, dtype=torch.int32, device=self.tables[0].device)
        smp = L.SampleCfg(int(batch_size), 0, int(step), int(max_try), int(epoch_seed) & (2**64 - 1), 0)
        k1, k2, ts = kg1.view(), kg2.view(), tset.view()
        L.check(self.lib.oea_triple_sample_batch(
            C.byref(k1), C.byref(k2), C.byref(ts), C.byref(smp), self.sampler, C.byref(self.tables[0].c_struct()),
            _ptr(self._idx), C.c_void_p(0), C.byref(self._n_pos), _stream_ptr()), "oea_triple_sample_batch")
        n = int(self._n_pos.value)
        return self._idx[:3 * n].view(3, n)

    def step_sampled(self, kg1, kg2, tset, batch_size, neg_per_pos, step, epoch_seed, max_try=10, **_):
        """One session.run([triple_loss, triple_optimizer]) of proje.py:87-90; neg_per_pos is ignored (positives only)."""
        pos = self.sample_batch(kg1, kg2, tset, batch_size, step, epoch_seed, max_try)
        if pos.shape[1] == 0:
            return 0
        self.sample(self.step_seed(epoch_seed, step))
        self.score_fed(pos)
        self.apply()
        return pos.shape[1]


class ConvETrainer(ProjETrainer):
    """ConvE's step (models/neural/conve.py:42-79): ProjE's batch producer, sampler, Adam and loss accumulator, with the
    convolution tower in front of the NCE head (oea_conve_score_fed).  tables = (ent, rel, cls_w, cls_b, conv, bn_in,
    fc_w, fc_out) EmbeddingTables (include/oea.h oea_conve).  The dropout masks are keyed by a seed derived from the
    sampler's, so a step's masks, like its sampled set, are a function of (epoch seed, step) only."""

    def __init__(self, tables, num_sampled, lr, keep_prob, sampler="fast"):
        super().__init__(tables, num_sampled, lr, sampler)
        self.keep_prob = float(keep_prob)
        if not 0.0 < self.keep_prob <= 1.0:
            raise ValueError("output_keep_prob = %r is not in (0, 1]" % keep_prob)
        self.filters = self.tables[4].rows

    def _workspace_bytes(self, n_pos):
        return self.lib.oea_conve_workspace_bytes(n_pos, self.num_sampled, self.tables[0].dim, self.filters,
                                                  self.n_classes)

    def score_fed(self, pos, sampled=None, num_tries=None, dropout_seed=0, loss_out=None):
        """pos: int32 device tensor [3, n] (h | r | t rows); sampled / num_tries: int32 device tensors (default: the
        last sample()).  Accumulates gradients into the eight tables and adds the batch loss into loss_out."""
        self._score("oea_conve_score_fed", L.Conve(*[C.pointer(t.c_struct()) for t in self.tables]), _pos_rows(pos),
                    pos.shape[1], sampled, num_tries, loss_out, self.keep_prob, int(dropout_seed) & (2**64 - 1))

    def step_sampled(self, kg1, kg2, tset, batch_size, neg_per_pos, step, epoch_seed, max_try=10, **_):
        """One session.run([triple_loss, triple_optimizer]) of conve.py:42-79; neg_per_pos is ignored (positives only)."""
        pos = self.sample_batch(kg1, kg2, tset, batch_size, step, epoch_seed, max_try)
        if pos.shape[1] == 0:
            return 0
        seed = self.step_seed(epoch_seed, step)
        self.sample(seed)
        self.score_fed(pos, dropout_seed=self.step_seed(seed, 0))
        self.apply()
        return pos.shape[1]


class NceTrainer(SampledNceTrainer):
    """tf.nn.nce_loss applied to an embedding lookup, one reduce_mean step of approaches/attr2vec.py:113-124,145-161:
    B distinct pairs drawn on the device (oea_pairs_draw, keyed by (seed, epoch, step)) → the sampler, seeded from the
    seed, the epoch and the step → oea_nce_score_fed with loss_scale 1/B → Adagrad (or the tables' optimiser) on the
    three tables.  tables = (inputs, cls_w, cls_b) EmbeddingTables, cls_b as [C, 1]."""

    def __init__(self, tables, num_sampled, lr):
        super().__init__(tables, num_sampled, lr, tables[1].rows)
        self.pairs = None
        self._batch = None

    def _workspace_bytes(self, n):
        return self.lib.oea_nce_workspace_bytes(n, self.num_sampled, self.tables[0].dim, self.n_classes)

    def set_pairs(self, pairs):
        """The training pairs the steps draw from: [n, 2] (input id, label id), copied to the device once."""
        self.pairs = torch.as_tensor(np.asarray(pairs, dtype=np.int32).reshape(-1, 2), device=self.tables[0].device)

    def draw(self, batch, seed, epoch, step):
        """random.sample(pairs, batch) of attr2vec.py:150 as a keyed permutation: (inputs [B], labels [B]) device int32."""
        if self._batch is None or self._batch.shape[1] < batch:
            self._batch = torch.empty(2, batch, dtype=torch.int32, device=self.tables[0].device)
        L.check(self.lib.oea_pairs_draw(_ptr(self.pairs), self.pairs.shape[0], int(batch), int(seed) & (2**64 - 1),
                                        int(epoch), int(step), _ptr(self._batch[0]), _ptr(self._batch[1]),
                                        _stream_ptr()), "oea_pairs_draw")
        return self._batch[0, :batch], self._batch[1, :batch]

    def score_fed(self, inputs, labels, sampled=None, num_tries=None, scale=None, loss_out=None):
        """inputs / labels: int32 device tensors [n]; sampled / num_tries: int32 device tensors (default: the last
        sample()); scale: default 1/n (reduce_mean).  Accumulates gradients into the three tables and adds the scaled
        batch loss into loss_out."""
        n = inputs.numel()
        scale = 1.0 / max(1, n) if scale is None else float(scale)
        self._score("oea_nce_score_fed", L.Nce(*[C.pointer(t.c_struct()) for t in self.tables]),
                    (_ptr(inputs), _ptr(labels)), n, sampled, num_tries, loss_out, scale)

    def step(self, batch, seed, epoch, step):
        """One session.run([loss, optimizer]) of attr2vec.py:156-158 on pairs drawn from set_pairs()."""
        inputs, labels = self.draw(batch, seed, epoch, step)
        self.sample(self.step_seed(self.step_seed(seed, epoch), step))
        self.score_fed(inputs, labels)
        self.apply()


class FedHostPipeline:
    """Depth-2 pipeline over TripleTrainer's host-index step (oea_triple_step_fed_host_submit / _collect): the copy of
    step i+1 overlaps the kernels of step i; losses come back one step late.  Owns two streams, four events and the
    per-slot buffers.  Usage: `for i, (pos, neg) in enumerate(batches): p.submit(i % 2, pos, neg); …; p.collect(i % 2)`
    with the host buffers of a submitted step left untouched until it is collected."""

    def __init__(self, trainer, max_indices):
        self.trainer = trainer
        dev = trainer.ent.device
        torch.cuda.synchronize(dev)                          # tables were initialised on the default stream
        self.copy_stream, self.compute_stream = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
        self.events = [torch.cuda.Event() for _ in range(4)]
        for ev in self.events:                               # a torch event gets its CUDA handle at the first record
            ev.record(self.compute_stream)
        self.compute_stream.synchronize()
        self.idx = [torch.empty(max(1, max_indices), dtype=torch.int32, device=dev) for _ in range(2)]
        self.loss_dev = [torch.zeros(1, dtype=torch.float64, device=dev) for _ in range(2)]
        self.loss_host = [torch.zeros(1, dtype=torch.float64).pin_memory() for _ in range(2)]
        vp2 = lambda a, b: (C.c_void_p * 2)(a, b)
        self.struct = L.FedPipeline(self.copy_stream.cuda_stream, self.compute_stream.cuda_stream,
                                    vp2(self.events[0].cuda_event, self.events[1].cuda_event),
                                    vp2(self.events[2].cuda_event, self.events[3].cuda_event),
                                    vp2(self.idx[0].data_ptr(), self.idx[1].data_ptr()),
                                    vp2(self.loss_dev[0].data_ptr(), self.loss_dev[1].data_ptr()),
                                    vp2(self.loss_host[0].data_ptr(), self.loss_host[1].data_ptr()))

    def submit(self, slot, pos_hrt, neg_hrt=None):
        t = self.trainer
        pos_t = _as_host_i32(pos_hrt)
        neg_t = _as_host_i32(neg_hrt) if neg_hrt is not None else None
        n_pos, n_neg = pos_t.shape[1], 0 if neg_t is None else neg_t.shape[1]
        assert 3 * (n_pos + n_neg) <= self.idx[slot].numel() and pos_t.is_pinned()
        for tab in (t.ent, t.rel):
            if tab.optimizer == "Adam":
                tab.adam_t += 1
        cfg = opt_cfg(t.ent, t.lr)
        L.check(t.lib.oea_triple_step_fed_host_submit(
            C.byref(t.ent.c_struct()), C.byref(t.rel.c_struct()), C.byref(self.struct), int(slot),
            C.c_void_p(pos_t.data_ptr()), n_pos, C.c_void_p(0 if neg_t is None else neg_t.data_ptr()), n_neg,
            C.byref(t.loss), C.byref(cfg)), "oea_triple_step_fed_host_submit")

    def collect(self, slot):
        loss = C.c_float(0.0)
        L.check(self.trainer.lib.oea_triple_step_fed_host_collect(C.byref(self.struct), int(slot), C.byref(loss)),
                "oea_triple_step_fed_host_collect")
        return float(loss.value)


def _as_host_i32(a):
    if isinstance(a, torch.Tensor):
        assert a.dtype == torch.int32 and not a.is_cuda and a.is_contiguous()
        return a
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.int32)))


class MappingTrainer:
    """MTransE-style mapping module: loss alpha·(Σ‖e2 − e1·M‖² + Σ(MMᵀ − I)²) over seed pairs
    (modules/base/mapping.py:9-19, losses.py:76-80) with its OWN optimiser slots on the entity table and on M."""

    def __init__(self, ent, mapping, alpha, lr):
        self.lib = L.load()
        self.ent = ent.new_slots()          # a separate optimiser instance ⇒ separate accumulators (SURVEY A.3)
        self.M = mapping
        self.alpha, self.lr = float(alpha), float(lr)
        self.loss_dev = torch.zeros(1, dtype=torch.float64, device=ent.device)
        ws = self.lib.oea_mapping_workspace_bytes(ent.dim)
        self.ws = torch.empty(max(1, ws), dtype=torch.uint8, device=ent.device)

    def step(self, ents1, ents2, read_loss=True):
        """One session.run([mapping_loss, mapping_optimizer]) (basic_model.py:244-246); returns the batch loss, or —
        with read_loss=False — leaves it accumulated on the device for `read_loss()` (no host sync per step).
        ents1 / ents2: entity id lists or int32 device tensors."""
        dev = self.ent.device
        i1 = torch.as_tensor(ents1, dtype=torch.int32, device=dev).contiguous()
        i2 = torch.as_tensor(ents2, dtype=torch.int32, device=dev).contiguous()
        n, d, p = i1.numel(), self.ent.dim, self.ent.pitch
        e1 = torch.empty(n, p, dtype=torch.float32, device=dev)
        e2 = torch.empty(n, p, dtype=torch.float32, device=dev)
        st = _stream_ptr()
        es, ms = self.ent.c_struct(), self.M.c_struct()
        L.check(self.lib.oea_table_lookup(C.byref(es), _ptr(i1), n, _ptr(e1), p, st), "oea_table_lookup")
        L.check(self.lib.oea_table_lookup(C.byref(es), _ptr(i2), n, _ptr(e2), p, st), "oea_table_lookup")
        g1, g2 = torch.empty_like(e1), torch.empty_like(e2)
        if read_loss:
            self.loss_dev.zero_()
        L.check(self.lib.oea_mapping_fwd_bwd(_ptr(e1), _ptr(e2), n, d, p, _ptr(self.M.weight), self.M.pitch, self.alpha,
                                             _ptr(self.loss_dev), _ptr(g1), _ptr(g2), _ptr(self.M.grad), _ptr(self.ws),
                                             self.ws.numel(), st), "oea_mapping_fwd_bwd")
        L.check(self.lib.oea_table_scatter_grad(C.byref(es), _ptr(i1), n, _ptr(g1), p, st), "oea_table_scatter_grad")
        L.check(self.lib.oea_table_scatter_grad(C.byref(es), _ptr(i2), n, _ptr(g2), p, st), "oea_table_scatter_grad")
        self.M.touched.fill_(1)
        for tab in (self.ent, self.M):
            if tab.optimizer == "Adam":
                tab.adam_t += 1
            cfg = opt_cfg(tab, self.lr)
            L.check(self.lib.oea_rowopt_apply(C.byref(tab.c_struct()), C.byref(cfg), st), "oea_rowopt_apply")
        return float(self.loss_dev.item()) if read_loss else None

    def read_loss(self, reset=True):
        v = float(self.loss_dev.item())
        if reset:
            self.loss_dev.zero_()
        return v


class EpochGraph:
    """One training epoch captured as a CUDA graph (launch-bound inner loop → one graph launch per epoch)."""

    def __init__(self, trainer, kg1, kg2, tset, batch_size, neg_per_pos, steps, max_try=10):
        self.trainer = trainer
        dev = trainer.ent.device
        self.seed_dev = torch.zeros(1, dtype=torch.int64, device=dev)
        self.key = trainer._views(kg1, kg2, tset) and trainer._view_key
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            for step in range(steps):
                trainer.step_sampled(kg1, kg2, tset, batch_size, neg_per_pos, step, 0, max_try=max_try,
                                     dev_seed=self.seed_dev)

    def replay(self, epoch_seed):
        self.seed_dev.fill_(int(epoch_seed) & ((1 << 63) - 1))
        self.graph.replay()
