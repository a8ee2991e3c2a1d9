"""CPU ORACLE (test infrastructure only) for TransR on path (i).

float64 torch-autograd restatement, TF op by TF op, of the graph models/trans/transr.py:14-52 builds: the looked-up
entity rows (normalised when ent_l2_norm) reshaped to [n, d, 1], tf.matmul with rel_matrix[r] reshaped row-major to
[d, d], tf.nn.l2_normalize of both projections (unconditionally), and get_loss_func on (h', r̂, t') — the losses of
modules/base/losses.py through oracle.triple_ext.loss_value.  rel_matrix is never normalised.  The CUDA kernels
(openea_b200/csrc/oea_triple_transr.cu) run the same maths in fp32; tests/test_emu_transr.py and
tests/test_zz_transr_gpu.py compare them with this file, and tests/test_transr_goldens.py pins it to the reference's own
graph code (tests/golden/path_i_transr.npz).

The matrix table `mat` may be given as [R, d²] (the reference's variable) or [R·d, d] (the engine's table): both are
the same row-major numbers.
"""
import numpy as np
import torch

from oracle.triple_ext import DenseState, _score, _var, l2n, loss_value  # noqa: F401  (DenseState: dense TF-1 steps)

SLOTS = ("ent", "rel", None, "mat")          # the order of the C-ABI struct oea_model: (ent, rel, ent_aux, rel_aux)


def projections(tabs, norms, hrt):
    """(l2n(M_r·ĥ), r̂, l2n(M_r·t̂)) per triple."""
    dev = tabs["ent"].device
    h, r, t = (torch.as_tensor(np.asarray(x), dtype=torch.long, device=dev) for x in hrt)
    E, R = _var(tabs["ent"], norms["ent"]), _var(tabs["rel"], norms["rel"])
    d = E.shape[1]
    M = tabs["mat"].reshape(-1, d, d)
    ph = l2n(torch.matmul(M[r], E[h].reshape(-1, d, 1)).reshape(-1, d))      # transr.py:38-44
    pt = l2n(torch.matmul(M[r], E[t].reshape(-1, d, 1)).reshape(-1, d))
    return ph, R[r], pt


def energies(tabs, norms, hrt, loss_norm="L2"):
    ph, rr, pt = projections(tabs, norms, hrt)
    return _score(ph + rr - pt, loss_norm)


def fwd_bwd(tabs, norms, pos, neg, loss, loss_norm="L2", margin=0.0, neg_margin=0.0, balance=1.0, scale=1.0,
            device="cpu"):
    """tabs: {"ent", "rel", "mat"} raw variables; norms: {"ent": bool, "rel": bool}; `device`: where the float64 graph
    runs (a 15K-shape batch gathers 10⁴ matrices).  Returns (loss, {slot: d loss / d raw variable as float64 arrays in
    the shape given})."""
    tv = {k: torch.tensor(np.asarray(v), dtype=torch.float64, device=device, requires_grad=True) for k, v in tabs.items()}
    e_pos = energies(tv, norms, pos, loss_norm)
    e_neg = energies(tv, norms, neg, loss_norm) if neg is not None and np.asarray(neg).shape[1] > 0 else None
    val = loss_value(e_pos, e_neg, loss, margin, neg_margin, balance, scale)
    val.backward()
    grads = {k: (v.grad.cpu().numpy() if v.grad is not None else np.zeros(v.shape)) for k, v in tv.items()}
    return float(val.detach()), grads


def step(state, norms, pos, neg, loss, lr, **kw):
    """One session.run([triple_loss, triple_optimizer]) with dense TF-1 optimiser rules; returns the batch loss."""
    val, grads = fwd_bwd(state.w, norms, pos, neg, loss, **kw)
    state.apply(grads, lr)
    return val
