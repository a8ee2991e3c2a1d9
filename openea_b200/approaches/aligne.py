"""AlignE on the CUDA engine (approaches/aligne.py): limited loss, ε-truncated negatives, swapping."""
from openea_b200.models.basic_model import BasicModel
from openea_b200.modules.utils.util import load_session


class AlignE(BasicModel):

    def __init__(self):
        super().__init__()

    def _check_args(self):
        a = self.args
        assert a.init == 'normal'
        assert a.alignment_module == 'swapping'
        assert a.loss == 'limited'
        assert a.neg_sampling == 'truncated'
        assert a.optimizer == 'Adagrad'
        assert a.eval_metric == 'inner'
        assert a.loss_norm == 'L2'
        assert a.ent_l2_norm is True
        assert a.rel_l2_norm is True
        assert a.pos_margin >= 0.0
        assert a.neg_margin > a.pos_margin
        assert a.neg_triple_num > 1
        assert a.truncated_epsilon > 0.0
        assert a.learning_rate >= 0.01

    def init(self):
        self.session = load_session()
        self._define_variables()
        self._define_embed_graph()
        self._check_args()

    def _define_embed_graph(self):
        # limited_loss(..., pos_margin, neg_margin, loss_norm, balance=neg_margin_balance) (aligne.py:63-65)
        super()._define_embed_graph(loss='limited')
