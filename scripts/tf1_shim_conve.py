"""TEST INFRASTRUCTURE: what ConvE's graph (models/neural/conve.py:42-79) needs from TensorFlow 1 beyond
oracle/tf1_shim.py and scripts/tf1_shim_proje.py, installed onto the shim module by `install()` before the reference is
imported (scripts/make_golden_conve.py).  Restated from the TF 1.x documentation and op definitions:

  * layers.batch_normalization(inputs, axis=-1, training=False): inference mode — the moving mean (0) and variance (1)
    normalise and are never updated, so y = x·γ/√(1 + ε) + β with ε = 1e-3 and γ (ones), β (zeros) of shape
    [inputs.shape[axis]], broadcast along that axis.  Variables batch_normalization[_i]/gamma, /beta in creation order.
  * layers.conv2d(inputs, filters, kernel_size, padding='same', use_bias=True, data_format='channels_first'): a
    cross-correlation (the kernel is not flipped), stride 1, 'same' zero padding of (k − 1)/2 on each side; kernel
    [kh, kw, in, filters] glorot-uniform (fan_in = kh·kw·in, fan_out = kh·kw·filters), bias zeros.  Variables
    <scope>/conv2d[_i]/kernel, /bias.
  * contrib.layers.fully_connected(inputs, num_outputs): activation ReLU, weights [in, out] xavier-uniform, biases
    zeros.  Variables <scope>/fully_connected[_i]/weights, /biases.
  * nn.dropout(x, keep_prob): x / keep_prob · mask with a Bernoulli(keep_prob) mask.  keep_prob = 1 is the plain shim's
    identity.  Otherwise the mask of each call is drawn from a counter stream: per session.run a seed is drawn from a
    seeded NumPy generator, and element i of the run's k-th dropout call is kept iff (pcg32(key_k ^ i) >> 8)·2⁻²⁴ <
    keep_prob (the stream include/oea.h documents for oea_conve_score_fed).  Every run's seed and masks are recorded in
    DROPOUT as (seed, [mask of call 0, mask of call 1, …]).  TF's ⌊keep_prob + U⌋ and `u < keep_prob` are the same
    Bernoulli draw; the counter stream lets the engine, given the recorded seed, draw the very masks the graph used.

Installing changes nothing the existing golden generators see: `python scripts/make_golden_conve.py --check-existing`
regenerates their goldens with the extension installed and compares them array by array with the committed files."""
import math

import numpy as np
import torch

DROPOUT = []              # (seed, [bool mask per dropout call, in the call's flat element order]) per session.run
M32 = 0xFFFFFFFF


def _pcg32(x):
    x = (np.asarray(x, dtype=np.uint64) * np.uint64(747796405) + np.uint64(2891336453)) & np.uint64(M32)
    w = (((x >> ((x >> np.uint64(28)) + np.uint64(4))) ^ x) * np.uint64(277803737)) & np.uint64(M32)
    return (w >> np.uint64(22)) ^ w


def counter_mask(seed, site, count, keep):
    key = int(_pcg32(np.uint64(seed & M32) ^ _pcg32(((seed >> 32) + site * 0x9E3779B9) & M32)))
    h = _pcg32(np.uint64(key) ^ np.arange(count, dtype=np.uint64))
    return (h >> np.uint64(8)).astype(np.float64) * 2.0 ** -24 < float(np.float32(keep))


def install(tf, seed=0):
    """Adds the ops above to the shim module `tf`, on top of scripts/tf1_shim_proje.py's (idempotent)."""
    if getattr(tf, "_conve_ops", False):
        return tf
    tf._conve_ops = True
    rng = np.random.default_rng(seed)
    counts = {}
    base_reset = tf.reset_default_graph

    def reset_default_graph():
        base_reset()
        counts.clear()
        DROPOUT.clear()
    tf.reset_default_graph = reset_default_graph

    def layer_scope(kind):
        i = counts.get(kind, 0)
        counts[kind] = i + 1
        return kind if i == 0 else "%s_%d" % (kind, i)

    def static_shape(x):
        """The shape of a node fed by index placeholders: evaluated once with every placeholder fed [0]."""
        env, stack, seen = {}, [x], set()
        while stack:
            n = stack.pop()
            if id(n) in seen:
                continue
            seen.add(id(n))
            if isinstance(n, tf.Placeholder):
                env[id(n)] = torch.zeros(1, dtype=torch.long)
            stack.extend(n.inputs)
        return tuple(x._eval(env).shape)

    def glorot(fan_in, fan_out, shape):
        lim = math.sqrt(6.0 / (fan_in + fan_out))
        return rng.uniform(-lim, lim, shape)

    def batch_normalization(inputs, axis=-1, momentum=0.99, epsilon=1e-3, center=True, scale=True, training=False,
                            **kw):
        assert center and scale and training is False, "only the inference-mode defaults are restated"
        x = tf._wrap(inputs)
        shape = static_shape(x)
        ax = axis % len(shape)
        scope = layer_scope("batch_normalization")
        gamma = tf.get_variable(scope + "/gamma", [shape[ax]], initializer=tf.ones_initializer())
        beta = tf.get_variable(scope + "/beta", [shape[ax]], initializer=tf.zeros_initializer())
        view = [1] * len(shape)
        view[ax] = -1

        def f(a, g, b):
            return a * (g / math.sqrt(1.0 + epsilon)).reshape(view) + b.reshape(view)
        return tf.Tensor(f, (x, gamma, beta), scope)

    def conv2d(inputs, filters, kernel_size, strides=(1, 1), padding="valid", data_format="channels_last",
               use_bias=True, **kw):
        assert padding == "same" and data_format == "channels_first" and tuple(strides) == (1, 1)
        kh, kw_ = kernel_size
        assert kh % 2 == 1 and kw_ % 2 == 1
        x = tf._wrap(inputs)
        cin = static_shape(x)[1]
        scope = layer_scope("conv2d")
        kernel = tf.get_variable(scope + "/kernel", [kh, kw_, cin, filters],
                                 initializer=lambda s: glorot(kh * kw_ * cin, kh * kw_ * filters, s))
        # cross-correlation, channels first: torch's conv2d weight is [out, in, kh, kw]
        conv = lambda a, k: torch.nn.functional.conv2d(a, k.permute(3, 2, 0, 1), padding=(kh // 2, kw_ // 2))
        if not use_bias:
            return tf.Tensor(conv, (x, kernel), scope)
        bias = tf.get_variable(scope + "/bias", [filters], initializer=tf.zeros_initializer())
        return tf.Tensor(lambda a, k, b: conv(a, k) + b.reshape(1, -1, 1, 1), (x, kernel, bias), scope)

    def fully_connected(inputs, num_outputs, activation_fn=tf.nn.relu, **kw):
        x = tf._wrap(inputs)
        cin = static_shape(x)[-1]
        scope = layer_scope("fully_connected")
        w = tf.get_variable(scope + "/weights", [cin, num_outputs], initializer=lambda s: glorot(cin, num_outputs, s))
        b = tf.get_variable(scope + "/biases", [num_outputs], initializer=tf.zeros_initializer())
        y = tf.Tensor(lambda a, ww, bb: a @ ww + bb, (x, w, b), scope)
        return y if activation_fn is None else activation_fn(y)

    base_dropout = tf.nn.dropout

    def dropout(x, keep_prob=None, rate=None, noise_shape=None, seed=None, name=None):
        kp = 1.0 - rate if keep_prob is None else keep_prob
        if float(kp) == 1.0:
            return base_dropout(x, keep_prob=1.0)
        kp = float(kp)

        def f(a):
            if not DROPOUT:                       # a shape-only evaluation while the graph is built
                return a / kp
            run = DROPOUT[-1]
            site = len(run[1])
            mask = counter_mask(run[0], site, a.numel(), kp)
            run[1].append(mask)
            return a / kp * torch.as_tensor(mask.reshape(tuple(a.shape)), dtype=a.dtype)
        return tf.Tensor(f, (tf._wrap(x),), "dropout")

    def new_run():
        """Called by the generator before each session.run: draws the run's dropout seed."""
        DROPOUT.append((int(rng.integers(0, 2 ** 63)), []))
    tf.dropout_new_run = new_run

    tf.layers.batch_normalization = batch_normalization
    tf.layers.conv2d = conv2d
    tf.contrib.layers.fully_connected = fully_connected
    tf.nn.dropout = dropout
    return tf
