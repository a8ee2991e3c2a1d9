"""ConvE (models/neural/conve.py of the reference): ProjE's variables, batches and NCE head with a convolution tower in
front of the head — the head and relation embeddings stacked into one image, an inference-mode batch norm, dropout, a
3×3 convolution, a batch norm per filter, ReLU, dropout, a fully connected ReLU layer and an output batch norm —
engine.ConvETrainer over csrc/oea_proje.cu.  Adam on all variables.  Evaluation and save are BasicModel's (entity and
relation embeddings), so dropout never reaches them."""
import math

import torch

from openea_b200 import engine as eng
from openea_b200 import parallel as par
from openea_b200.models.basic_model import BasicModel
from openea_b200.models.neural.proje import ProjE
from openea_b200.modules.base import initializers

MAX_DIM = 128                                            # the NCE head's row width (include/oea.h oea_conve)


def dim_factorization(d):
    """conve.py:10-18: the image of one d-vector is x × y, x the largest divisor of d not above ⌊√d⌋ + 1."""
    half = int(math.sqrt(d)) + 1
    while d % half > 0:
        half -= 1
    return half, d // half


def _uniform(shape, lim):
    return torch.rand(*shape, generator=initializers._GEN, dtype=torch.float32) * (2 * lim) - lim


class ConvE(ProjE):

    def __init__(self):
        super().__init__()
        self.kernel_size = (3, 3)
        self.conv = None
        self.bn_in = None
        self.fc_w = None
        self.fc_out = None

    def init(self):
        if par.world()[1] > 1:
            raise NotImplementedError("ConvE runs on one GPU")
        a = self.args
        for ok, what in ((0 < a.output_keep_prob <= 1, "0 < output_keep_prob <= 1"), (a.filter_num >= 1, "filter_num >= 1"),
                         (a.dim <= MAX_DIM, "dim <= %d" % MAX_DIM)):
            if not ok:
                raise ValueError("ConvE needs %s" % what)
        super().init()                                   # proje.py's guards (conve.py:34-40), then the variables

    def _define_variables(self):
        BasicModel._define_variables(self)               # ent_embeds, rel_embeds: xavier, l2-normalised, Adam slots
        self._define_head_variables()                    # entity_w, entity_b; ConvE builds no mlp variables
        d, F = self.args.dim, self.args.filter_num
        _, y = dim_factorization(d)
        # cnn/conv2d: kernel [3, 3, 1, F] glorot-uniform (fan_in 9, fan_out 9F), bias 0; stored per filter as its 9
        # taps, the bias, and the gamma (1) and beta (0) of the batch norm over filters
        taps = _uniform([3, 3, F], math.sqrt(6.0 / (9 + 9 * F))).permute(2, 0, 1).reshape(F, 9)
        self.conv = initializers._make(torch.cat([taps, torch.zeros(F, 1), torch.ones(F, 1), torch.zeros(F, 1)], 1),
                                       False, 'Adam')
        # the image's batch norm over its y columns: gamma 1, beta 0
        self.bn_in = initializers._make(torch.stack([torch.ones(y), torch.zeros(y)]), False, 'Adam')
        # fully_connected: weights [2Fd, d] xavier-uniform, bias 0; then the output batch norm's gamma 1 and beta 0
        self.fc_w = initializers._make(_uniform([2 * F * d, d], math.sqrt(6.0 / (2 * F * d + d))), False, 'Adam')
        self.fc_out = initializers._make(torch.stack([torch.zeros(d), torch.ones(d), torch.zeros(d)]), False, 'Adam')

    def _define_embed_graph(self):
        self.triple_trainer = eng.ConvETrainer((self.ent_embeds, self.rel_embeds, self.entity_w, self.entity_b,
                                                self.conv, self.bn_in, self.fc_w, self.fc_out), self.args.dnn_neg_nums,
                                               self.args.learning_rate, self.args.output_keep_prob)
        self.neg_per_pos = 0                             # generate_pos_batch: positives only
        self.triple_loss = self.triple_optimizer = self.triple_trainer
