"""RotatE (models/semantic/rotate.py of the reference): real and imaginary entity tables and a relation table of phases;
a relation rotates the head, E = Σ_i |ĥ_i·e^{iθ_i} − t̂_i| − γ with θ = r̂·π/ρ, ρ = (γ + 2)/dim, and the loss
−Σ log σ(γ − d⁺) − (1/k)·Σ log σ(d⁻ − γ) (rotate.py:61-82) — the OEA_MODEL_ROTATE instance of oea_model_score_fed,
positives and negatives weighted separately.  The reference keeps these variables in float64; here they are fp32 like
every table of the engine.  Evaluation and save use re + im (rotate.py:121-144)."""
import openea_b200.modules.load.read as rd
from openea_b200 import engine as eng
from openea_b200 import finding as F
from openea_b200 import parallel as par
from openea_b200.models.basic_model import BasicModel
from openea_b200.modules.base.initializers import init_embeddings, set_default_optimizer
from openea_b200.modules.utils.util import load_session


class RotatE(BasicModel):

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
        self.session = load_session()
        assert self.args.init == 'uniform'
        assert self.args.alignment_module == 'sharing'
        assert self.args.neg_sampling == 'uniform'
        assert self.args.optimizer == 'Adam'
        assert self.args.eval_metric == 'inner'
        assert self.args.gamma > 0.0

    def _define_variables(self):
        a = self.args
        set_default_optimizer(a.optimizer)
        mk = lambda rows, name, norm: init_embeddings([rows, a.dim], name, a.init, norm, optimizer=a.optimizer)
        self.re_ent_embeds = mk(self.kgs.entities_num, 're_ent_embeds', a.ent_l2_norm)
        self.im_ent_embeds = mk(self.kgs.entities_num, 'im_ent_embeds', a.ent_l2_norm)
        self.rel_embeds = mk(self.kgs.relations_num, 'rel_embeds', a.rel_l2_norm)
        self.ent_embeds = self.re_ent_embeds          # device / shape queries of the base class

    def _triple_trainer(self, neg_weight):
        return eng.ModelTrainer("RotatE", (self.re_ent_embeds, self.rel_embeds, self.im_ent_embeds),
                                eng.loss_cfg("logistic", "L2"), self.args.learning_rate, gamma=self.args.gamma,
                                neg_weight=neg_weight)

    def _define_embed_graph(self):
        self.triple_trainer = self._triple_trainer(1.0 / self.args.neg_triple_num)      # rotate.py:81
        self.neg_per_pos = self.args.neg_triple_num
        self.triple_loss = self.triple_optimizer = self.triple_trainer

    def _both_parts(self, ids=None):
        return self.re_ent_embeds.lookup(ids) + self.im_ent_embeds.lookup(ids)   # device row add (plumbing)

    def _eval_valid_embeddings(self):
        return (self._both_parts(self.kgs.valid_entities1),
                self._both_parts(self.kgs.valid_entities2 + self.kgs.test_entities2), self._mapping_array())

    def _eval_test_embeddings(self):
        return self._both_parts(self.kgs.test_entities1), self._both_parts(self.kgs.test_entities2), self._mapping_array()

    def save(self):
        self._sync_replicas()          # under torchrun: the owners' rows everywhere; only rank 0 writes the files
        if par.world()[0] != 0:
            return
        ent, _ = F.to_device_rows(self._both_parts(), normalize=True)      # preprocessing.normalize (rotate.py:141)
        ent_embeds = ent[:, :self.args.dim].cpu().numpy()
        rel_embeds = self.rel_embeds.lookup().cpu().numpy()
        mapping_mat = self.mapping_mat.raw().cpu().numpy() if self.mapping_mat is not None else None
        rd.save_embeddings(self.out_folder, self.kgs, ent_embeds, rel_embeds, None, mapping_mat=mapping_mat)
