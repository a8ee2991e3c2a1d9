"""CPU ORACLE (test infrastructure only) for ConvE on path (i).

float64 torch-autograd restatement, TF op by TF op, of the graph models/neural/conve.py:42-79 builds, given the sampled
set and num_tries of TF's unique log-uniform candidate sampler and the two dropout masks:
  x_h = ê[h], x_r = r̂[r] (l2-normalised lookups), reshaped row-major to x × y (dim_factorization) and stacked into a
  [2x, y] image; tf.layers.batch_normalization in inference mode (moving mean 0, variance 1, ε = 1e-3) over the image's
  columns: v·γ₁[j]/√(1+ε) + β₁[j]; dropout v/keep·m₀; conv2d with F 3×3 filters, 'same' padding, a bias, as a
  cross-correlation; the same batch norm per filter (γ₂, β₂); ReLU; dropout ·m₁/keep; flatten channel-first to 2Fd;
  fully_connected: relu(A·W + bias); the same batch norm per column (γ₃, β₃) → X; then Σ_b nce_loss as ProjE's head.
The CUDA kernels (openea_b200/csrc/oea_proje.cu) run the same maths in fp32.

Tables: {"ent" [E, d], "rel" [R, d], "w" [E, d], "b" [E, 1], "conv" [F, 12] (9 taps dy·3 + dx, bias, γ₂, β₂),
"bn_in" [2, y] (γ₁, β₁), "fc_w" [2Fd, d], "fc_out" [3, d] (bias, γ₃, β₃)}.
"""
import math

import numpy as np
import torch

from oracle.triple_ext import DenseState, l2n  # noqa: F401  (DenseState: dense TF-1 Adam steps)
from tests.proje_oracle import expected_count, sample_unique  # noqa: F401

BN_EPS = 1e-3
NAMES = ("ent", "rel", "w", "b", "conv", "bn_in", "fc_w", "fc_out")
M32 = 0xFFFFFFFF


def dim_factorization(d):
    half = int(math.sqrt(d)) + 1
    while d % half > 0:
        half -= 1
    return half, d // half


# ---- the device dropout mask, restated --------------------------------------------------------------------------------
def pcg32(x):
    x = (np.asarray(x, dtype=np.uint64) * np.uint64(747796405) + np.uint64(2891336453)) & np.uint64(M32)
    w = (((x >> ((x >> np.uint64(28)) + np.uint64(4))) ^ x) * np.uint64(277803737)) & np.uint64(M32)
    return (w >> np.uint64(22)) ^ w


def dropout_key(seed, site):
    seed &= (1 << 64) - 1
    inner = pcg32(((seed >> 32) + site * 0x9E3779B9) & M32)
    return int(pcg32(np.uint64(seed & M32) ^ inner))


def dropout_mask(seed, site, count, keep):
    """Kept flags of elements 0 … count − 1 of mask `site`: (pcg32(key ^ i) >> 8)·2⁻²⁴ < keep (fp32 keep)."""
    h = pcg32(np.uint64(dropout_key(seed, site)) ^ np.arange(count, dtype=np.uint64))
    return (h >> np.uint64(8)).astype(np.float64) * 2.0 ** -24 < float(np.float32(keep))


def masks(seed, n, d, F, keep):
    """(m₀ [n, 2d], m₁ [n, 2Fd]) of oea_conve_score_fed for a batch of n: flat indices b·2d + e and b·2Fd + o."""
    return (dropout_mask(seed, 0, n * 2 * d, keep).reshape(n, 2 * d),
            dropout_mask(seed, 1, n * 2 * F * d, keep).reshape(n, 2 * F * d))


# ---- the step ---------------------------------------------------------------------------------------------------------
def tower(tv, norms, h, r, keep, m0, m1):
    """X [n, d] and the pre-activations of both ReLUs (conv [n, 2Fd], dense [n, d])."""
    dev = tv["ent"].device
    E = l2n(tv["ent"]) if norms["ent"] else tv["ent"]
    R = l2n(tv["rel"]) if norms["rel"] else tv["rel"]
    n, d = len(h), E.shape[1]
    x, y = dim_factorization(d)
    F = tv["conv"].shape[0]
    s = 1.0 / math.sqrt(1.0 + BN_EPS)
    img = torch.cat([E[h].reshape(n, x, y), R[r].reshape(n, x, y)], 1)
    u = img * (tv["bn_in"][0] * s) + tv["bn_in"][1]
    u = u / keep * torch.as_tensor(m0, dtype=torch.float64, device=dev).reshape(n, 2 * x, y)
    C = tv["conv"]
    q = torch.nn.functional.conv2d(u[:, None], C[:, :9].reshape(F, 1, 3, 3), C[:, 9], padding=1)
    p = q * (C[:, 10] * s)[None, :, None, None] + C[:, 11][None, :, None, None]
    a = torch.relu(p) / keep * torch.as_tensor(m1, dtype=torch.float64, device=dev).reshape(n, F, 2 * x, y)
    zpre = a.reshape(n, 2 * F * d) @ tv["fc_w"] + tv["fc_out"][0]
    X = torch.relu(zpre) * (tv["fc_out"][1] * s) + tv["fc_out"][2]
    return X, p.reshape(n, -1), zpre


def loss_of(tv, norms, pos, sampled, num_tries, keep, m0, m1):
    dev = tv["ent"].device
    h, r, t = (torch.as_tensor(np.asarray(v), dtype=torch.long, device=dev) for v in pos)
    X, _, _ = tower(tv, norms, h, r, keep, m0, m1)
    W, b = tv["w"], tv["b"].reshape(-1)
    n_classes, S = W.shape[0], len(sampled)
    lq = lambda ids: torch.as_tensor(np.log(expected_count(np.asarray(ids), n_classes, S, num_tries).astype(np.float64)),
                                     device=dev)
    smp = torch.as_tensor(np.asarray(sampled), dtype=torch.long, device=dev)
    true = (X * W[t]).sum(1) + b[t] - lq(pos[2])
    samp = X @ W[smp].T + b[smp] - lq(sampled)
    return torch.nn.functional.softplus(-true).sum() + torch.nn.functional.softplus(samp).sum()


def tensors(tabs, device="cpu", grad=True):
    return {k: torch.tensor(np.asarray(v), dtype=torch.float64, device=device, requires_grad=grad) for k, v in tabs.items()}


def fwd_bwd(tabs, norms, pos, sampled, num_tries, keep, m0, m1, device="cpu"):
    """(loss, {name: d loss / d variable as float64 arrays in the shape given})."""
    tv = tensors(tabs, device)
    val = loss_of(tv, norms, pos, sampled, num_tries, keep, m0, m1)
    val.backward()
    return float(val.detach()), {k: (v.grad.cpu().numpy() if v.grad is not None else np.zeros(v.shape))
                                 for k, v in tv.items()}


def _gamma(k):
    u = 2.0 ** -24
    return k * u / (1 - k * u)


def kink_ratios(tabs, norms, pos, keep, m0, m1, device="cpu"):
    """|pre-activation| over its fp32 rounding bound, for every ReLU input that reaches the loss: (conv [kept
    elements], dense).  The bound is γ(k)·Σ|terms| of the element's own sum — k = 12 for a conv output (nine taps, the
    bias, the batch norm's FMA and the input's rounding), 2Fd + 13 for a dense one — evaluated on absolute values.  A
    ratio above 1 means fp32 takes the same ReLU branch as float64."""
    with torch.no_grad():
        tv = tensors(tabs, device, grad=False)
        h, r = (torch.as_tensor(np.asarray(v), dtype=torch.long, device=device) for v in pos[:2])
        _, p, z = tower(tv, norms, h, r, keep, m0, m1)
        av = {k: v.abs() for k, v in tv.items()}
        # tower() on absolute values, with the normalised tables' |x̂| in place of the raw rows, gives Σ|terms|
        E = l2n(tv["ent"]).abs() if norms["ent"] else av["ent"]
        R = l2n(tv["rel"]).abs() if norms["rel"] else av["rel"]
        av["ent"], av["rel"] = E, R
        _, pa, za = tower(av, {"ent": False, "rel": False}, h, r, keep, m0, m1)
        F, d = tv["conv"].shape[0], tv["fc_w"].shape[1]
        kept = torch.as_tensor(m1, device=device)
        conv = (p.abs() / (_gamma(12) * pa.abs()).clamp_min(1e-300))[kept]
        dense = z.abs() / (_gamma(2 * F * d + 13) * za.abs()).clamp_min(1e-300)
        return conv, dense


def kink_margin(tabs, norms, pos, keep, m0, m1, device="cpu"):
    """The smallest kink ratio of kink_ratios (> 1: no ReLU input lies within fp32 rounding of 0)."""
    conv, dense = kink_ratios(tabs, norms, pos, keep, m0, m1, device)
    return min(float(conv.min()) if conv.numel() else math.inf, float(dense.min()))


def near_kinks(tabs, norms, pos, keep, m0, m1, device="cpu"):
    """(number of ReLU inputs within fp32 rounding of 0, number of ReLU inputs that reach the loss)."""
    conv, dense = kink_ratios(tabs, norms, pos, keep, m0, m1, device)
    return int((conv <= 1).sum()) + int((dense <= 1).sum()), conv.numel() + dense.numel()


def step(state, norms, pos, sampled, num_tries, keep, m0, m1, lr):
    """One session.run([triple_loss, triple_optimizer]) with TF-1's dense Adam; returns the batch loss."""
    val, grads = fwd_bwd(state.w, norms, pos, sampled, num_tries, keep, m0, m1)
    state.apply(grads, lr)
    return val
