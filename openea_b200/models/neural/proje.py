"""ProjE (models/neural/proje.py of the reference): the head and relation embeddings through a shared-beta batch norm, a
shared-weight combination and an output batch norm, scored by tf.nn.nce_loss against entity_w / entity_b over one set
of dnn_neg_nums log-uniform classes per step — engine.ProjETrainer over csrc/oea_proje.cu.  Adam on all variables.
Evaluation and save are BasicModel's (entity and relation embeddings)."""
import math

import torch

from openea_b200 import engine as eng
from openea_b200.models.basic_model import BasicModel
from openea_b200.modules.base import initializers
from openea_b200.modules.utils.util import load_session


class ProjE(BasicModel):

    def __init__(self):
        super().__init__()
        self.entity_w = None
        self.entity_b = None
        self.proje_params = None

    def init(self):
        a = self.args
        # proje.py:28-34, checked before anything is allocated
        for ok, what in ((a.init == 'xavier', "init 'xavier'"), (a.alignment_module == 'sharing', "alignment 'sharing'"),
                         (a.optimizer == 'Adam', "optimizer 'Adam'"), (a.eval_metric == 'inner', "eval_metric 'inner'"),
                         (a.ent_l2_norm is True and a.rel_l2_norm is True, "ent_l2_norm and rel_l2_norm"),
                         (a.dnn_neg_nums > 1, "dnn_neg_nums > 1")):
            if not ok:
                raise ValueError("%s needs %s" % (type(self).__name__, what))
        if a.dnn_neg_nums > self.kgs.entities_num:
            raise ValueError("dnn_neg_nums = %d exceeds the %d entities: the sampler's range is too small"
                             % (a.dnn_neg_nums, self.kgs.entities_num))
        self.session = load_session()
        self._define_variables()
        self._define_embed_graph()

    def _define_variables(self):
        super()._define_variables()                      # ent_embeds, rel_embeds: xavier, l2-normalised, Adam slots
        self._define_head_variables()
        # mlp/mlp_w and mlp/mlp_bias: get_variable's default glorot-uniform on [d] (limit sqrt(3/d)); both batch-norm
        # betas start at 0.  One [4, d] table: rows mlp_w, mlp_bias, input beta, output beta
        d = self.args.dim
        lim = math.sqrt(3.0 / d)
        glorot = lambda: torch.rand(d, generator=initializers._GEN, dtype=torch.float32) * (2 * lim) - lim
        params = torch.stack([glorot(), glorot(), torch.zeros(d), torch.zeros(d)])
        self.proje_params = initializers._make(params, False, 'Adam')

    def _define_head_variables(self):
        """entity_w and entity_b, the NCE head's variables (proje.py:42-44)."""
        n_ent, d = self.kgs.entities_num, self.args.dim
        self.entity_w = initializers.init_embeddings([n_ent, d], 'entity_w', 'xavier', False, optimizer='Adam')
        # entity_b: xavier on the 1-D shape [E] (σ = sqrt(1.3/E)), stored as an [E, 1] table
        self.entity_b = initializers._make(initializers.init_values([n_ent], 'xavier').reshape(n_ent, 1), False, 'Adam')

    def _define_embed_graph(self):
        self.triple_trainer = eng.ProjETrainer((self.ent_embeds, self.rel_embeds, self.entity_w, self.entity_b,
                                                self.proje_params), self.args.dnn_neg_nums, self.args.learning_rate)
        self.neg_per_pos = 0                             # generate_pos_batch: positives only
        self.triple_loss = self.triple_optimizer = self.triple_trainer
