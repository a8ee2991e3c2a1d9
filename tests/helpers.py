"""Shared test helpers: float64 torch-autograd statement of the triple-scoring graph (an independent
derivation used to check the C oracle's hand-written backward) and seeded batch generators."""
import numpy as np
import torch


def torch_triple_loss(ent, rel, pos, neg, loss, loss_norm, ent_norm, rel_norm, margin=0.0, neg_margin=0.0,
                      balance=1.0, dtype=torch.float64):
    """Formulas of modules/base/losses.py + initializers.py:26 in torch; returns (loss, g_ent, g_rel, scores)."""
    E = torch.tensor(np.asarray(ent), dtype=dtype, requires_grad=True)
    R = torch.tensor(np.asarray(rel), dtype=dtype, requires_grad=True)

    def l2n(x):
        ss = (x * x).sum(1, keepdim=True)
        return x * torch.rsqrt(torch.clamp(ss, min=1e-12))

    Eh = l2n(E) if ent_norm else E
    Rh = l2n(R) if rel_norm else R

    def score(hrt):
        hrt = torch.as_tensor(np.asarray(hrt), dtype=torch.long)
        u = Eh[hrt[0]] + Rh[hrt[1]] - Eh[hrt[2]]
        return u.abs().sum(1) if loss_norm == "L1" else (u * u).sum(1)

    sp = score(pos)
    sn = score(neg) if neg is not None and np.asarray(neg).size else torch.zeros(0, dtype=dtype)
    relu = torch.nn.functional.relu
    if loss == "margin-based":
        val = relu(margin + sp - sn).sum()
    elif loss == "limited":
        val = relu(sp - margin).sum() + balance * relu(neg_margin - sn).sum()
    elif loss == "logistic":
        val = torch.log(1 + torch.exp(sp)).sum() + torch.log(1 + torch.exp(-sn)).sum()
    elif loss == "positive":
        val = sp.sum()
    elif loss == "logsigmoid":
        val = -torch.log(torch.sigmoid(-sp)).sum()
    else:
        raise ValueError(loss)
    val.backward()
    g_e = E.grad if E.grad is not None else torch.zeros_like(E)
    g_r = R.grad if R.grad is not None else torch.zeros_like(R)
    return float(val.detach()), g_e.numpy(), g_r.numpy(), torch.cat([sp, sn]).detach().numpy()


def make_tables(rng, n_ent, n_rel, d, scale=1.0):
    ent = (rng.standard_normal((n_ent, d)) * scale / np.sqrt(d)).astype(np.float32)
    rel = (rng.standard_normal((n_rel, d)) * scale / np.sqrt(d)).astype(np.float32)
    return ent, rel


def make_batch(rng, n_ent, n_rel, n_pos, k, hot=True):
    """Index batch with repeated rows (a few hot entities/relations) as Zipf-like KGs produce."""
    def ents(n):
        e = rng.integers(0, n_ent, size=n)
        if hot and n > 4:
            m = rng.random(n) < 0.3
            e[m] = rng.integers(0, max(1, min(5, n_ent)), size=int(m.sum()))
        return e
    pos = np.stack([ents(n_pos), rng.integers(0, n_rel, size=n_pos), ents(n_pos)]).astype(np.int32)
    if k == 0:
        return pos, None
    neg = np.repeat(pos, k, axis=1)
    side = rng.random(n_pos * k) < 0.5
    repl = ents(n_pos * k)
    neg[0, side] = repl[side]
    neg[2, ~side] = repl[~side]
    return pos, neg.astype(np.int32)


class ReferenceRecording:
    """Results of the reference project's own functions, replayed in call order from tests/golden/<name>.pkl.xz, so that
    a comparison with the reference needs nothing outside this repository.  With OEA_RECORD_REFERENCE=1 (and the
    reference importable through `live`, a zero-argument callable returning {name: function}) the calls go to the
    reference and the file is rewritten.  Objects of the reference's own classes are stored as plain namespaces of
    their attributes.  Every call also stores a signature of its arguments (`_signature`), and a replay whose arguments
    differ from the recorded ones fails as stale instead of comparing against results for other inputs."""

    def __init__(self, name, live):
        import lzma
        import os
        import pickle
        self.path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name + ".pkl.xz")
        self.recording = os.environ.get("OEA_RECORD_REFERENCE") == "1"
        if self.recording:
            self.live, self.calls = live(), []
            assert self.live is not None, "OEA_RECORD_REFERENCE=1 but the reference is not importable"
        else:
            with lzma.open(self.path, "rb") as f:
                self.calls = pickle.load(f)
        self.next = 0

    def __call__(self, fn, *args, **kwargs):
        sig = _signature((args, kwargs))                 # before the call: reference functions may mutate their inputs
        if self.recording:
            out = self.live[fn](*args, **kwargs)
            self.calls.append((fn, sig, _plain(out)))
            return out
        assert self.next < len(self.calls), "the test makes more reference calls than were recorded: re-record"
        name, want_sig, out = self.calls[self.next]
        assert name == fn, "recorded call %d is %s, the test now calls %s: re-record" % (self.next, name, fn)
        assert _same_signature(sig, want_sig), "the inputs of recorded call %d (%s) changed: re-record" % (self.next, fn)
        self.next += 1
        return out

    def save(self):
        import lzma
        import pickle
        if self.recording:
            with lzma.open(self.path, "wb", preset=9 | lzma.PRESET_EXTREME) as f:
                pickle.dump(self.calls, f, protocol=4)
        else:
            assert self.next == len(self.calls), "the test made fewer reference calls than were recorded: re-record"


def _signature(x):
    """(sha256 of everything exact in x, [float64 summaries of its floating-point parts]).  Floats are summarised, not
    hashed, because inputs computed with vectorised reductions (a CPU matmul, a row norm) may differ in the last bit
    between machines.  A directory path stands for the names and bytes of the files under it."""
    import hashlib
    import os
    import numpy as np
    import scipy.sparse as sp
    h, floats = hashlib.sha256(), []

    def exact(*parts):
        for p in parts:
            h.update(repr(p).encode() + b"\0")

    def summary(a):
        a = np.asarray(a, dtype=np.float64).ravel()
        w = np.sin(np.arange(a.size) + 1.0)
        floats.extend([float(a.sum()), float((a * a).sum()), float((a * w).sum())])

    def key(v):                          # order of set / dict members: their exact signature
        return _signature(v)[0]

    def walk(v):
        if v is None or isinstance(v, (bool, int, np.integer, bytes)):
            exact(type(v).__name__, int(v) if isinstance(v, np.integer) else v)
        elif isinstance(v, (float, np.floating)):
            exact("f"); summary([float(v)])
        elif isinstance(v, str):
            if os.path.isdir(v):
                exact("dir")
                for root, _, files in sorted(os.walk(v)):
                    for name in sorted(files):
                        full = os.path.join(root, name)
                        with open(full, "rb") as f:
                            exact(os.path.relpath(full, v), hashlib.sha256(f.read()).hexdigest())
            else:
                exact("s", v)
        elif sp.issparse(v):
            m = sp.coo_matrix(v); m.sum_duplicates()
            exact("sparse", m.shape, m.row.tobytes(), m.col.tobytes()); summary(m.data)
        elif isinstance(v, np.ndarray):
            exact("nd", v.dtype.str, v.shape)
            if np.issubdtype(v.dtype, np.floating):
                summary(v)
            else:
                exact(np.ascontiguousarray(v).tobytes())
        elif hasattr(v, "numpy") and hasattr(v, "detach"):          # torch tensor
            walk(v.detach().cpu().numpy())
        elif isinstance(v, dict):
            exact("dict", len(v))
            for k in sorted(v, key=key):
                walk(k); walk(v[k])
        elif isinstance(v, (set, frozenset)):
            exact("set", len(v))
            for m in sorted(v, key=key):
                walk(m)
        elif isinstance(v, (list, tuple)):
            exact(type(v).__name__, len(v))
            for m in v:
                walk(m)
        elif isinstance(v, type) or hasattr(v, "__dict__"):
            attrs = {k: a for k, a in vars(v).items() if not k.startswith("__") and not callable(a)}
            exact("obj")              # attributes only: a replay hands back namespaces where the reference had its classes
            walk(attrs)
        else:
            exact("other", type(v).__name__)

    walk(x)
    return h.hexdigest(), floats


def _same_signature(a, b):
    import numpy as np
    return a[0] == b[0] and len(a[1]) == len(b[1]) and bool(np.allclose(a[1], b[1], rtol=1e-5, atol=1e-6))


def _plain(x):
    """x with instances of classes defined outside importable modules (the reference's) turned into namespaces."""
    import types
    if isinstance(x, dict):
        return type(x)((k, _plain(v)) for k, v in x.items()) if type(x) is dict else {k: _plain(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)) and type(x) in (list, tuple):
        return type(x)(_plain(v) for v in x)
    mod = getattr(type(x), "__module__", "")
    if hasattr(x, "__dict__") and not isinstance(x, type) and (mod in ("builtins", "__main__", None) or mod.startswith("openea")):
        return types.SimpleNamespace(**{k: _plain(v) for k, v in vars(x).items()})
    return x
