"""CPU ORACLE (test infrastructure only) for ProjE on path (i).

float64 torch-autograd restatement, TF op by TF op, of the graph models/neural/proje.py:46-74 builds, given the sampled
set and num_tries of TF's unique log-uniform candidate sampler:
  x_h = ê[h], x_r = r̂[r] (l2-normalised lookups); y = batch_norm(x) in training mode (batch mean, biased variance,
  ε = 1e-3, beta, no gamma) with one beta shared by both inputs; z = y_h·w + y_r·w + b (the same mlp_w twice);
  X = batch_norm_out(z); loss = Σ_b nce_loss: sigmoid cross-entropy of x·w_c + b_c − log q(c), true class against 1 and
  every sampled class against 0, accidental hits kept.
q(c) is computed in fp32 as TF's RangeSampler does, including its shortcut P(c)·S when num_tries == S.
The CUDA kernels (openea_b200/csrc/oea_proje.cu) run the same maths in fp32; tests/test_emu_proje.py and
tests/test_zz_proje_gpu.py compare them with this file.

Tables: {"ent" [E, d], "rel" [R, d], "w" [E, d], "b" [E] or [E, 1], "params" [4, d]} with params rows mlp_w, mlp_bias,
the input beta and the output beta.
"""
import math

import numpy as np
import torch

from oracle.triple_ext import DenseState, l2n  # noqa: F401  (DenseState: dense TF-1 Adam steps)

BN_EPS = 1e-3


def probability(ids, n_classes):
    """LogUniformSampler::Probability in fp32: log((c+2)/(c+1)) / log(E+1)."""
    ids = np.asarray(ids, dtype=np.float64)
    return (np.log((ids + 2.0) / (ids + 1.0)) / math.log1p(n_classes)).astype(np.float32)


def expected_count(ids, n_classes, num_sampled, num_tries):
    """ExpectedCountHelper in fp32."""
    p = probability(ids, n_classes)
    if num_tries == num_sampled:
        return p * np.float32(num_sampled)
    return (-np.expm1(np.float32(num_tries) * np.log1p(-p))).astype(np.float32)


def draw_classes(seed, j, n_classes):
    """The device sampler's draw j (oea_logu_sample_unique): ⌊exp(u·log(E+1))⌋ − 1 mod E, u from mix64."""
    M = (1 << 64) - 1

    def mix64(z):
        z = (z + 0x9E3779B97F4A7C15) & M
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
        return z ^ (z >> 31)
    r = mix64((seed & M) ^ mix64(j))
    u = (r >> 11) * 2.0 ** -53
    return (int(math.exp(u * math.log1p(n_classes))) - 1) % n_classes


def sample_unique(seed, n_classes, num_sampled):
    """The sequential loop of TF's unique sampler over the device's draw stream: (sampled ids, num_tries)."""
    seen, out, j = set(), [], 0
    while len(out) < num_sampled:
        c = draw_classes(seed, j, n_classes)
        j += 1
        if c not in seen:
            seen.add(c)
            out.append(c)
    return np.asarray(out, dtype=np.int32), j


def _bn(x, beta):
    mu = x.mean(0, keepdim=True)
    var = ((x - mu) ** 2).mean(0, keepdim=True)
    return (x - mu) / torch.sqrt(var + BN_EPS) + beta


def loss_of(tv, norms, pos, sampled, num_tries, drop_true=None):
    """The batch loss of float64 tensors `tv` (on any device) for host index arrays.  drop_true: a row whose true-class
    term is left out (tests/nce_edge_cases.py checks that its comparisons can see one term missing)."""
    dev = tv["ent"].device
    h, r, t = (torch.as_tensor(np.asarray(x), dtype=torch.long, device=dev) for x in pos)
    E = l2n(tv["ent"]) if norms["ent"] else tv["ent"]
    R = l2n(tv["rel"]) if norms["rel"] else tv["rel"]
    W, b, P = tv["w"], tv["b"].reshape(-1), tv["params"]
    n_classes, S = W.shape[0], len(sampled)
    y_h, y_r = _bn(E[h], P[2]), _bn(R[r], P[2])
    X = _bn(y_h * P[0] + y_r * P[0] + P[1], P[3])
    s = torch.as_tensor(np.asarray(sampled), dtype=torch.long, device=dev)
    lq = lambda ids: torch.as_tensor(np.log(expected_count(np.asarray(ids), n_classes, S, num_tries).astype(np.float64)),
                                     device=dev)
    lq_t, lq_s = lq(pos[2]), lq(sampled)
    true = (X * W[t]).sum(1) + b[t] - lq_t
    samp = X @ W[s].T + b[s] - lq_s
    true_terms = torch.nn.functional.softplus(-true)
    if drop_true is not None:
        true_terms = torch.cat([true_terms[:drop_true], true_terms[drop_true + 1:]])
    return true_terms.sum() + torch.nn.functional.softplus(samp).sum()


def fwd_bwd(tabs, norms, pos, sampled, num_tries, device="cpu", drop_true=None):
    """Returns (loss, {name: d loss / d variable as float64 arrays in the shape given}); `device`: where the float64
    graph runs (a 100K-shape batch is a [5 000, 4 096] product)."""
    tv = {k: torch.tensor(np.asarray(v), dtype=torch.float64, device=device, requires_grad=True) for k, v in tabs.items()}
    val = loss_of(tv, norms, pos, sampled, num_tries, drop_true)
    val.backward()
    return float(val.detach()), {k: (v.grad.cpu().numpy() if v.grad is not None else np.zeros(v.shape))
                                 for k, v in tv.items()}


def step(state, norms, pos, sampled, num_tries, lr):
    """One session.run([triple_loss, triple_optimizer]) with TF-1's dense Adam; returns the batch loss."""
    val, grads = fwd_bwd(state.w, norms, pos, sampled, num_tries)
    state.apply(grads, lr)
    return val
