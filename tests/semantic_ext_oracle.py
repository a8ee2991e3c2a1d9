"""CPU ORACLE (test infrastructure only) for RotatE and HolE on path (i).

float64 torch-autograd restatement, TF op by TF op, of the graphs the reference builds for
  RotatE         models/semantic/rotate.py:52-93 (lookup_all, _generate_scores, _generate_loss)
  BootEA_RotatE  approaches/bootea_rotate.py:48-108 (the same graph, negatives unweighted) and :149-160 (alignment loss)
  HolE           models/semantic/hole.py:41-86 (_ccorr through the FFT, _calc, the averaged margin loss)
with tf.nn.embedding_lookup → indexing, tf.nn.l2_normalize(x, 1) → x·rsqrt(max(Σx², 1e-12)), and `init_embeddings(...,
is_l2_norm)` returning the normalised variable (modules/base/initializers.py:26-50), so gradients flow through the
normalisation into the raw variable.  The CUDA kernels (openea_b200/csrc/oea_triple_ext.cu) run the same maths in fp32
and compute HolE's correlation directly instead of through the FFT; tests/test_emu_semantic_ext.py and
tests/test_zz_semantic_ext_gpu.py compare them with this file, and tests/test_semantic_ext_goldens.py pins both to the
reference's own graph code (tests/golden/path_i_semantic_ext.npz).
"""
import numpy as np
import torch

from oracle.triple_ext import DenseState, l2n  # noqa: F401  (DenseState: the dense TF-1 optimiser steps)

PI = 3.14159265358979323846            # rotate.py:24
EPSILON = 2.0                          # rotate.py:25
# table slots in the order of the C-ABI struct oea_model: (ent, rel, ent_aux, rel_aux)
SLOTS = {"RotatE": ("re_ent", "rel", "im_ent"), "HolE": ("ent", "rel")}


def _var(tab, norm):
    return l2n(tab) if norm else tab


def rotate_phase_scale(gamma, dim):
    """1 / (embedding_range / π) with embedding_range = (γ + ε) / dim (rotate.py:37,90)."""
    return 1.0 / (((gamma + EPSILON) / dim) / PI)


def rotate_distance(tabs, norms, hrt, gamma):
    """Σ_i ‖(re_score_i, im_score_i)‖ of rotate.py:61-69 (before `gamma − ·`), per triple."""
    h, r, t = (torch.as_tensor(np.asarray(x), dtype=torch.long) for x in hrt)
    RE, IM = _var(tabs["re_ent"], norms["re_ent"]), _var(tabs["im_ent"], norms["im_ent"])
    R = _var(tabs["rel"], norms["rel"])
    dim = RE.shape[1]
    rh, rt, ih, it = RE[h], RE[t], IM[h], IM[t]                            # lookup_all, rotate.py:84-89
    phase = R[r] / (((gamma + EPSILON) / dim) / PI)                        # rotate.py:90
    rr, ir = torch.cos(phase), torch.sin(phase)                            # rotate.py:91-92
    re_score = rh * rr - ih * ir - rt                                      # rotate.py:62
    im_score = rh * ir + ih * rr - it                                      # rotate.py:63
    scores = torch.stack([re_score, im_score], 0)                          # rotate.py:65
    scores = torch.sqrt((scores * scores).sum(0))                          # tf.norm(axis=0), rotate.py:67
    return scores.sum(-1)                                                  # rotate.py:69


def rotate_loss(tabs, norms, pos, neg, gamma, neg_weight):
    """rotate.py:74-82: −Σ log σ(γ − d⁺) − neg_weight·Σ log σ(−(γ − d⁻)); neg_weight = 1/k there, 1 in
    bootea_rotate.py:77.  neg None: BootEA_RotatE's alignment loss −Σ log σ(γ − d) (bootea_rotate.py:153-158)."""
    pos_scores = gamma - rotate_distance(tabs, norms, pos, gamma)
    loss = -torch.log(torch.sigmoid(pos_scores)).sum()
    if neg is not None and np.asarray(neg).shape[1] > 0:
        neg_scores = -(gamma - rotate_distance(tabs, norms, neg, gamma))
        loss = loss - torch.log(torch.sigmoid(neg_scores)).sum() * neg_weight
    return loss


def ccorr(a, b):
    """hole.py:51-54: real(ifft(conj(fft(a)) · fft(b))) along the last axis."""
    a, b = a.to(torch.complex128), b.to(torch.complex128)
    return torch.real(torch.fft.ifft(torch.conj(torch.fft.fft(a)) * torch.fft.fft(b)))


def hole_energy(tabs, norms, hrt):
    """_calc of hole.py:56-60: −σ(Σ l2_normalize(r) ∘ ccorr(h, t)), shape [n, 1]."""
    h, r, t = (torch.as_tensor(np.asarray(x), dtype=torch.long) for x in hrt)
    E, R = _var(tabs["ent"], norms["ent"]), _var(tabs["rel"], norms["rel"])
    relation_mention = l2n(R[r])
    entity_mention = ccorr(E[h], E[t])
    return -torch.sigmoid((relation_mention * entity_mention).sum(1, keepdim=True))


def hole_loss(tabs, norms, pos, neg, margin):
    """hole.py:78-84: Σ relu(m + E⁺ − mean over the k negatives of each positive)."""
    pos_score = hole_energy(tabs, norms, pos)
    neg_score = hole_energy(tabs, norms, neg)
    k = neg_score.shape[0] // pos_score.shape[0]
    if k > 1:
        neg_score = neg_score.reshape(-1, k).mean(1, keepdim=True)
    return torch.relu(margin + pos_score - neg_score).sum()


def fwd_bwd(model, tabs, norms, pos, neg, gamma=12.0, neg_weight=1.0, margin=0.2):
    """tabs: {slot: float array [rows, d]} raw variables; norms: {slot: bool}.
    Returns (loss, {slot: d loss / d raw variable as float64 arrays})."""
    tv = {k: torch.tensor(np.asarray(v), dtype=torch.float64, requires_grad=True) for k, v in tabs.items()}
    if model == "RotatE":
        val = rotate_loss(tv, norms, pos, neg, gamma, neg_weight)
    elif model == "HolE":
        val = hole_loss(tv, norms, pos, neg, margin)
    else:
        raise ValueError(model)
    val.backward()
    grads = {k: (v.grad.numpy() if v.grad is not None else np.zeros(v.shape)) for k, v in tv.items()}
    return float(val.detach()), grads


def step(state, model, norms, pos, neg, lr, **kw):
    """One session.run([triple_loss, triple_optimizer]) with dense TF-1 optimiser rules; returns the batch loss."""
    val, grads = fwd_bwd(model, state.w, norms, pos, neg, **kw)
    state.apply(grads, lr)
    return val


def ccorr_direct(a, b):
    """The O(d²) form the kernel computes: ccorr_k = Σ_i a_i · b_{(i+k) mod d} (NumPy, float64)."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    d = a.shape[-1]
    idx = (np.arange(d)[None, :] + np.arange(d)[:, None]) % d           # [k, i] → (i + k) mod d
    return np.einsum("...i,...ki->...k", a, b[..., idx])
