"""HolE (models/semantic/hole.py of the reference): entity and relation tables, energy E = −σ(<l2n(r̂), ccorr(ĥ, t̂)>)
with the circular correlation ccorr_k = Σ_i ĥ_i·t̂_{(i+k) mod dim}, and the margin loss Σ relu(m + E⁺ − mean_k E⁻) over
the k negatives of every positive (hole.py:77-84) — the OEA_MODEL_HOLE instance of oea_model_score_fed (the reference
correlates through the FFT; the kernel sums directly, O(dim²) per triple).  Evaluation and save are BasicModel's."""
from openea_b200 import engine as eng
from openea_b200.models.basic_model import BasicModel
from openea_b200.modules.utils.util import load_session


class HolE(BasicModel):
    """
    A small margin, such as 0.2 or 0.3, works!
    """

    def init(self):
        self._define_variables()
        self._define_embed_graph()
        self.session = load_session()
        assert self.args.init == 'xavier'
        assert self.args.alignment_module == 'sharing'
        assert self.args.neg_sampling == 'uniform'
        assert self.args.optimizer == 'Adagrad'
        assert self.args.eval_metric == 'inner'
        assert self.args.loss_norm == 'L2'
        assert self.args.ent_l2_norm is True
        assert self.args.rel_l2_norm is True
        assert self.args.margin > 0.0

    def _define_embed_graph(self):
        self.triple_trainer = eng.ModelTrainer("HolE", (self.ent_embeds, self.rel_embeds),
                                               eng.loss_cfg("margin-based", "L2", margin=self.args.margin),
                                               self.args.learning_rate)
        self.neg_per_pos = self.args.neg_triple_num
        self.triple_loss = self.triple_optimizer = self.triple_trainer
