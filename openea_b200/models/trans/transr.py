"""TransR (models/trans/transr.py of the reference): h' = l2_normalize(M_r·ĥ), t' = l2_normalize(M_r·t̂) with one d×d
matrix per relation, loss chosen by get_loss_func(args) on (h', r̂, t') — oea_transr_score_fed, the relation-grouped
kernel of csrc/oea_triple_transr.cu.  Evaluation and save are BasicModel's (entity and relation embeddings)."""
from openea_b200 import engine as eng
from openea_b200.models.basic_model import _loss_from_args
from openea_b200.models.trans.transe import TransE
from openea_b200.modules.base import initializers


class TransR(TransE):

    def __init__(self):
        super().__init__()
        self.rel_matrix = None

    def _define_variables(self):
        super()._define_variables()
        a = self.args
        n_rel, d = self.kgs.relations_num, a.dim
        # transr.py:20-21: init_embeddings([R, d·d], 'rel_matrix', init, False) — drawn with that shape (σ = 1/d for
        # 'normal', fan R + d² for 'xavier'), stored as R·d rows of width d: row r·d + i is row i of M_r
        values = initializers.init_values([n_rel, d * d], a.init).reshape(n_rel * d, d)
        self.rel_matrix = initializers._make(values, False, a.optimizer)

    def _define_embed_graph(self):
        self.triple_trainer = eng.ModelTrainer("TransR", (self.ent_embeds, self.rel_embeds, None, self.rel_matrix),
                                               _loss_from_args(self.args), self.args.learning_rate)
        self.neg_per_pos = self.args.neg_triple_num
        self.triple_loss = self.triple_optimizer = self.triple_trainer
