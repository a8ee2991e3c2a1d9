"""MTransE on the CUDA engine (approaches/mtranse.py of the reference): positive-only squared-L2 TransE loss
on relation triples + the orthogonal mapping loss on seed pairs, each with its own Adagrad slots."""
import math
import time

from openea_b200.models.basic_model import BasicModel
from openea_b200.modules.finding.evaluation import early_stop
from openea_b200.modules.utils.util import load_session, task_divide


class MTransE(BasicModel):

    def __init__(self):
        super().__init__()

    def init(self):
        self.session = load_session()
        self._define_variables()
        self._define_mapping_variables()
        self._define_embed_graph()
        self._define_mapping_graph()
        # hyper-parameter guards of the reference (mtranse.py:31-37)
        required = dict(init='unit', alignment_module='mapping', optimizer='Adagrad', eval_metric='inner',
                        ent_l2_norm=True)
        for key, want in required.items():
            assert getattr(self.args, key) == want, "MTransE needs %s=%r" % (key, want)
        assert self.args.alpha > 1

    def _define_embed_graph(self):
        # positive_loss(phs, prs, pts, 'L2'): no negatives (mtranse.py:56)
        self.args.loss_norm = getattr(self.args, "loss_norm", "L2")
        super()._define_embed_graph(loss='positive', neg_per_pos=0)

    def launch_training_1epo(self, epoch, triple_steps, steps_tasks, training_batch_queue, neighbors1, neighbors2):
        self.launch_triple_training_1epo(epoch, triple_steps, steps_tasks, training_batch_queue, neighbors1, neighbors2)
        self.launch_mapping_training_1epo(epoch, triple_steps)

    def run(self):
        started = time.time()
        a = self.args
        n_triples = self.kgs.kg1.relation_triples_num + self.kgs.kg2.relation_triples_num
        triple_steps = int(math.ceil(n_triples / a.batch_size))
        steps_tasks = task_divide(list(range(triple_steps)), a.batch_threads_num)
        for epoch in range(1, a.max_epoch + 1):
            self.launch_training_1epo(epoch, triple_steps, steps_tasks, None, None, None)
            if epoch < a.start_valid or epoch % a.eval_freq:
                continue
            flag = self.valid(a.stop_metric)
            self.flag1, self.flag2, self.early_stop = early_stop(self.flag1, self.flag2, flag)
            if self.early_stop or epoch == a.max_epoch:
                break
        print("Training ends. Total time = {:.3f} s.".format(time.time() - started))
