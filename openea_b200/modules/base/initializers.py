"""Embedding initialisers → device tables (interface of modules/base/initializers.py:9-56 of the reference).

`init_embeddings(shape, name, init, is_l2_norm)` returns an `openea_b200.engine.EmbeddingTable`: the RAW
variable plus the `is_l2_norm` flag.  As in the reference, every lookup of a normalised table goes through
l2_normalize and gradients flow back through it (initializers.py:26,34,41,50).
Random streams cannot match TensorFlow's; parity tests start both sides from explicit tensors.
"""
import math

import numpy as np
import torch

from openea_b200.engine import EmbeddingTable

_GEN = torch.Generator(device="cpu")
_DEFAULT_OPT = "Adagrad"


def set_seed(seed):
    _GEN.manual_seed(int(seed))


def set_default_optimizer(opt):
    """Optimiser whose slot variables new tables allocate (TF creates slots lazily per optimiser)."""
    global _DEFAULT_OPT
    _DEFAULT_OPT = opt


def _trunc_normal(shape, std):
    t = torch.empty(*shape, dtype=torch.float32)
    return torch.nn.init.trunc_normal_(t, mean=0.0, std=std, a=-2 * std, b=2 * std, generator=_GEN)


def _make(values, is_l2_norm, optimizer=None):
    dev = "cuda" if torch.cuda.is_available() else None
    if dev is None:
        from openea_b200.lib import OeaError
        raise OeaError("embedding tables live on the GPU; no CUDA device is visible (no CPU fallback)")
    return EmbeddingTable(values, bool(is_l2_norm), optimizer or _DEFAULT_OPT, dev)


def init_embeddings(shape, name, init, is_l2_norm, dtype=None, optimizer=None):
    if init == 'xavier':
        return xavier_init(shape, name, is_l2_norm, optimizer=optimizer)
    if init == 'normal':
        return truncated_normal_init(shape, name, is_l2_norm, optimizer=optimizer)
    if init == 'uniform':
        return random_uniform_init(shape, name, is_l2_norm, optimizer=optimizer)
    if init == 'unit':
        return random_unit_init(shape, name, is_l2_norm, optimizer=optimizer)
    return None


def init_values(shape, init):
    """The values init_embeddings(shape, name, init, ...) holds, as a host tensor of `shape`, drawn with that shape's
    distribution (TransR draws its [R, d²] matrix table this way and stores it as R·d rows of width d)."""
    draw = {'xavier': _xavier_values, 'normal': _normal_values, 'uniform': _uniform_values, 'unit': _unit_values}
    if init not in draw:
        raise ValueError("unknown init %r" % (init,))
    return draw[init](shape)


def _xavier_values(shape):
    # tf.contrib.layers.xavier_initializer(uniform=False): truncated normal, σ = sqrt(1.3·2/(fan_in+fan_out)); a 1-D
    # shape [n] has fan_in = fan_out = n (ProjE's entity_b), so σ = sqrt(1.3/n)
    fan_in, fan_out = (shape[0], shape[1]) if len(shape) > 1 else (shape[0], shape[0])
    return _trunc_normal(shape, math.sqrt(1.3 * 2.0 / (fan_in + fan_out)))


def _normal_values(shape):
    return _trunc_normal(shape, 1.0 / math.sqrt(shape[1]))


def _uniform_values(shape, minval=0, maxval=None):
    hi = 1.0 if maxval is None else float(maxval)
    return torch.rand(*shape, generator=_GEN, dtype=torch.float32) * (hi - minval) + minval


def _unit_values(shape):
    t = torch.randn(*shape, generator=_GEN, dtype=torch.float32)
    return t / t.norm(dim=1, keepdim=True).clamp_min(1e-12)       # sklearn.preprocessing.normalize


def xavier_init(shape, name, is_l2_norm, dtype=None, optimizer=None):
    return _make(_xavier_values(shape), is_l2_norm, optimizer)


def truncated_normal_init(shape, name, is_l2_norm, dtype=None, optimizer=None):
    return _make(_normal_values(shape), is_l2_norm, optimizer)


def random_uniform_init(shape, name, is_l2_norm, minval=0, maxval=None, dtype=None, optimizer=None):
    return _make(_uniform_values(shape, minval, maxval), is_l2_norm, optimizer)


def random_unit_init(shape, name, is_l2_norm, dtype=None, optimizer=None):
    return _make(_unit_values(shape), is_l2_norm, optimizer)


def orthogonal_init(shape, name, dtype=None, optimizer=None):
    t = torch.empty(*shape, dtype=torch.float32)
    torch.nn.init.orthogonal_(t, generator=_GEN)
    return _make(t, False, optimizer)


def from_array(values, is_l2_norm, optimizer=None):
    """Table from explicit values (parity tests start engine and oracle from the same tensors)."""
    return _make(torch.as_tensor(np.asarray(values), dtype=torch.float32), is_l2_norm, optimizer)
