"""CPU ORACLE (test infrastructure only) for the general sampled-NCE step (oea_nce_score_fed) and Attr2Vec's step.

loss = scale · Σ_b tf.nn.nce_loss(ŵ, b, label_b, x̂[input_b]) in float64 torch autograd, through jape.nce_loss (the
torch restatement of tf.nn.nce_loss with closed-form tests in tests/test_jape.py) over l2-normalised or raw tables.
jape.nce_loss takes the expected count 1 − (1 − p)^num_tries in float64; TF (and the kernel) compute it in fp32 and
switch to p·S when num_tries == S (proje_oracle.expected_count).  A per-class shift of the biases by the difference of
the two log counts makes the logits TF's; a constant shift leaves every gradient unchanged.

Tables: {"in" [A, d], "w" [C, d], "b" [C] or [C, 1]}.
"""
import math

import numpy as np
import torch

from oracle.triple_ext import DenseState, l2n  # noqa: F401  (DenseState: dense TF-1 Adagrad steps)
from openea_b200.approaches import jape
from tests import proje_oracle as po


def fwd_bwd(tabs, norms, inputs, labels, sampled, num_tries, scale, device="cpu"):
    """→ (loss, {name: d loss / d variable, float64 arrays in the shape given})."""
    tv = {k: torch.tensor(np.asarray(v), dtype=torch.float64, device=device, requires_grad=True) for k, v in tabs.items()}
    n_classes, S = tv["w"].shape[0], len(sampled)
    X = (l2n(tv["in"]) if norms["in"] else tv["in"])[torch.as_tensor(np.asarray(inputs), device=device).long()]
    W = l2n(tv["w"]) if norms["w"] else tv["w"]
    b = tv["b"].reshape(-1)
    c = torch.arange(n_classes, dtype=torch.float64, device=device)
    p = torch.log((c + 2.0) / (c + 1.0)) / math.log(n_classes + 1.0)
    tf_q = torch.as_tensor(po.expected_count(np.arange(n_classes), n_classes, S, num_tries).astype(np.float64),
                           device=device)
    b = b - torch.log(tf_q) + torch.log(-torch.expm1(num_tries * torch.log1p(-p)))
    lab = torch.as_tensor(np.asarray(labels), device=device).long()
    smp = torch.as_tensor(np.asarray(sampled), device=device).long()
    val = scale * jape.nce_loss(W, b, lab, X, smp, num_tries, n_classes).sum()
    val.backward()
    return float(val.detach()), {k: (v.grad.cpu().numpy() if v.grad is not None else np.zeros(v.shape))
                                 for k, v in tv.items()}


def step(state, norms, inputs, labels, sampled, num_tries, lr):
    """One session.run([loss, optimizer]) of attr2vec.py:156 (reduce_mean, dense TF-1 Adagrad); returns the loss."""
    val, grads = fwd_bwd(state.w, norms, inputs, labels, sampled, num_tries, 1.0 / len(inputs))
    state.apply(grads, lr)
    return val
