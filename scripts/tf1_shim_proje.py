"""TEST INFRASTRUCTURE: what ProjE's graph (models/neural/proje.py:36-74) needs from TensorFlow 1 beyond
oracle/tf1_shim.py, installed onto that shim module by `install()` before the reference is imported
(scripts/make_golden_proje.py).  Restated from the TF 1.x documentation and op definitions:

  * variable_scope(name, reuse=None | True | AUTO_REUSE): scopes nest; reuse is inherited by inner scopes.  get_variable
    returns the variable already made under the same scoped name only when reuse is requested (True, or AUTO_REUSE);
    otherwise it makes a new one, as the plain shim does.  get_variable's default initializer is glorot-uniform, and a
    1-D shape [n] has fan_in = fan_out = n (so does contrib.layers.xavier_initializer's).  A variable keeps the plain
    name the shim gives it; its scoped name is `scoped_name`.
  * contrib.layers.batch_norm defaults: training mode (the batch's mean and biased variance over axis 0),
    epsilon = 1e-3, center=True (a beta under <scope>/beta, zeros), scale=False (no gamma).  The moving statistics are
    not trainable and never read in training mode, so they are not made.
  * nn.log_uniform_candidate_sampler(unique=True): P(c) = log((c+2)/(c+1)) / log(E+1), ⌊exp(u·log(E+1))⌋ − 1 mod E
    per draw, draws until num_sampled distinct classes are held; expected counts in fp32 as RangeSampler computes
    them, −expm1(num_tries·log1p(−P)) or P·S when num_tries == S.  Drawn once per session.run from a seeded NumPy
    stream, and every draw is recorded in SAMPLED as (sampled ids, num_tries).
  * nn.nce_loss: one sampler call per graph evaluation over the labels, logits x·w_c + b_c − log q(c) (subtract_log_q),
    accidental hits kept, sigmoid cross-entropy with the true class against 1 and each sampled class against 0, summed
    per example.

Installing changes nothing the existing golden generators see: `python scripts/make_golden_proje.py --check-existing`
regenerates their goldens with the extension installed and compares them array by array with the committed files."""
import contextlib
import math

import numpy as np
import torch

SAMPLED = []              # (sampled ids int32 [S], num_tries) of every sampler evaluation, in order


class _AutoReuse:
    def __repr__(self):
        return "AUTO_REUSE"


AUTO_REUSE = _AutoReuse()


def install(tf, seed=0):
    """Adds the ops above to the shim module `tf` (idempotent)."""
    if getattr(tf, "_proje_ops", False):
        return tf
    tf._proje_ops = True
    scopes = []                                  # [(name, reuse)]
    scoped = {}                                  # scoped name → Variable
    rng = np.random.default_rng(seed)
    base_reset = tf.reset_default_graph

    def reset_default_graph():
        base_reset()
        scoped.clear()
        SAMPLED.clear()
    tf.reset_default_graph = reset_default_graph

    def current_reuse():
        return scopes[-1][1] if scopes else None

    @contextlib.contextmanager
    def variable_scope(name_or_scope, default_name=None, values=None, reuse=None, **kw):
        name = name_or_scope if name_or_scope is not None else default_name
        scopes.append((name, reuse if reuse is not None else current_reuse()))
        try:
            yield
        finally:
            scopes.pop()
    tf.variable_scope = variable_scope
    tf.AUTO_REUSE = AUTO_REUSE

    def fans(shape):
        return (shape[0], shape[1]) if len(shape) > 1 else (shape[0], shape[0])

    def glorot_uniform(shape):
        fan_in, fan_out = fans(shape)
        lim = math.sqrt(6.0 / (fan_in + fan_out))
        return rng.uniform(-lim, lim, shape)

    base_xavier = tf.contrib.layers.xavier_initializer

    def xavier_initializer(uniform=True, **kw):
        two_d = base_xavier(uniform=uniform, **kw)

        def init(shape):
            if len(shape) > 1:
                return two_d(shape)
            fan = float(shape[0])
            if uniform:
                return rng.uniform(-math.sqrt(3.0 / fan), math.sqrt(3.0 / fan), shape)
            return tf._truncated_normal(stddev=math.sqrt(1.3 / fan))(shape)
        return init

    def get_variable(name, shape=None, dtype=None, initializer=None, regularizer=None, trainable=True, **kw):
        full = "/".join([s for s, _ in scopes] + [name])
        reuse = current_reuse()
        if reuse is True or reuse is AUTO_REUSE:
            if full in scoped:
                return scoped[full]
            if reuse is True:
                raise ValueError("Variable %s does not exist, or was not created with tf.get_variable()" % full)
        init = initializer if initializer is not None else glorot_uniform
        v = tf.Variable(init(list(shape)), name=name, dtype=dtype, trainable=trainable)
        v.scoped_name = full
        scoped[full] = v
        return v
    tf.get_variable = get_variable

    def width(x):
        """The static last dimension of a node fed by index placeholders: evaluated once with every placeholder fed [0]."""
        env, stack, seen = {}, [x], set()
        while stack:
            n = stack.pop()
            if id(n) in seen:
                continue
            seen.add(id(n))
            if isinstance(n, tf.Placeholder):
                env[id(n)] = torch.zeros(1, dtype=torch.long)
            stack.extend(n.inputs)
        return int(x._eval(env).shape[-1])

    def batch_norm(inputs, decay=0.999, center=True, scale=False, epsilon=0.001, is_training=True, reuse=None,
                   scope=None, **kw):
        assert center and not scale and is_training, "only contrib.layers.batch_norm's defaults are restated"
        x = tf._wrap(inputs)
        with variable_scope(scope, "BatchNorm", reuse=reuse):
            beta = get_variable("beta", [width(x)], initializer=tf.zeros_initializer())

        def f(a, b):
            mean = a.mean(0, keepdim=True)
            var = ((a - mean) ** 2).mean(0, keepdim=True)
            return (a - mean) / torch.sqrt(var + epsilon) + b
        return tf.Tensor(f, (x, beta), "batch_norm")

    tf.contrib.layers.xavier_initializer = xavier_initializer
    tf.contrib.layers.batch_norm = batch_norm

    def probability(ids, range_max):
        ids = np.asarray(ids, dtype=np.float64)
        return (np.log((ids + 2.0) / (ids + 1.0)) / math.log1p(range_max)).astype(np.float32)

    def expected_count(ids, range_max, num_sampled, num_tries):
        p = probability(ids, range_max)
        if num_tries == num_sampled:
            return p * np.float32(num_sampled)
        return (-np.expm1(np.float32(num_tries) * np.log1p(-p))).astype(np.float32)

    def log_uniform_candidate_sampler(true_classes, num_true, num_sampled, unique, range_max, seed=None, name=None):
        assert unique, "only the unique sampler is restated"
        log_range = math.log1p(range_max)

        def draw(labels):
            seen, out, tries = set(), [], 0
            while len(out) < num_sampled:
                tries += 1
                c = (int(math.exp(rng.random() * log_range)) - 1) % range_max
                if c not in seen:
                    seen.add(c)
                    out.append(c)
            ids = np.asarray(out, dtype=np.int32)
            SAMPLED.append((ids, tries))
            true_q = expected_count(labels.numpy().reshape(-1, num_true), range_max, num_sampled, tries)
            return (torch.as_tensor(ids.astype(np.int64)), torch.as_tensor(true_q.astype(np.float64)),
                    torch.as_tensor(expected_count(ids, range_max, num_sampled, tries).astype(np.float64)))
        node = tf.Tensor(draw, (tf._wrap(true_classes),), "log_uniform_candidate_sampler")
        return tuple(tf.Tensor(lambda t, i=i: t[i], (node,), "sampler_out") for i in range(3))

    def nce_loss(weights, biases, labels, inputs, num_sampled, num_classes, num_true=1, sampled_values=None,
                 remove_accidental_hits=False, partition_strategy="mod", name="nce_loss"):
        assert num_true == 1 and sampled_values is None and not remove_accidental_hits
        sampled, true_q, sampled_q = log_uniform_candidate_sampler(labels, num_true, num_sampled, True, num_classes)

        def f(w, b, lab, x, s, tq, sq):
            t = lab.reshape(-1).long()
            true_logit = (x * w[t]).sum(1) + b[t] - torch.log(tq.reshape(-1))
            samp_logit = x @ w[s].T + b[s] - torch.log(sq)
            # sigmoid_cross_entropy_with_logits: max(z, 0) − z·y + log(1 + e^{−|z|})
            return torch.nn.functional.softplus(-true_logit) + torch.nn.functional.softplus(samp_logit).sum(1)
        return tf.Tensor(f, tuple(tf._wrap(v) for v in (weights, biases, labels, inputs, sampled, true_q, sampled_q)),
                         "nce_loss")

    tf.nn.log_uniform_candidate_sampler = log_uniform_candidate_sampler
    tf.nn.nce_loss = nce_loss
    return tf
