"""Flag patterns for the flagged-row optimiser (rowopt_flagged_body) and a NumPy float32 restatement of its update,
shared by tests/test_emu_rowopt_flags.py (warp emulator, small tables) and tests/test_zz_rowopt_flags_gpu.py (the
device, at the bench's 200 000 + 600 rows).  A pattern flags rows of table A (entities) and table B (relations) and
places a random gradient on exactly those rows, as a scorer leaves them; every other gradient row is zero."""
import zlib

import numpy as np
import torch

LR = 0.01


def _rows(rng, n, p):
    return rng.random(n) < p


def _first_1pct(rng, a, b):
    fa = np.zeros(a, bool)
    head = max(1, (a + b) // 100)
    fa[:head] = _rows(rng, head, 0.6)
    fa[0] = True
    return fa, np.zeros(b, bool)


def _straddle(r):
    # A.rows % 4 = r: the quad at the table boundary holds rows of both tables, all of them flagged
    def flags(rng, a, b):
        fa, fb = _rows(rng, a + r, 0.3), _rows(rng, b, 0.3)
        fa[-r:] = True
        fb[:4 - r] = True
        return fa, fb
    return flags


# name -> flags of table A and table B for a base of `a` rows in A (a multiple of 4) and `b` in B; the lengths of the
# returned arrays are the tables' row counts
PATTERNS = {
    "none": lambda rng, a, b: (np.zeros(a, bool), np.zeros(b, bool)),
    "all": lambda rng, a, b: (np.ones(a, bool), np.ones(b, bool)),
    "first_row": lambda rng, a, b: (np.arange(a) == 0, np.zeros(b, bool)),
    "last_row_of_each_table": lambda rng, a, b: (np.arange(a) == a - 1, np.arange(b) == b - 1),
    "one_row_b": lambda rng, a, b: (_rows(rng, a, 0.3), np.ones(1, bool)),
    "first_1pct": _first_1pct,
    # every row of A: a warp whose quads span several windows holds more than 128 flagged rows
    "dense": lambda rng, a, b: (np.ones(a, bool), _rows(rng, b, 0.5)),
    "straddle_1": _straddle(1),
    "straddle_2": _straddle(2),
    "straddle_3": _straddle(3),
}


def seed_of(*key):
    return zlib.crc32(repr(key).encode())


def place(eng, rng, pattern, dim, opt, device, base_a, base_b):
    """A TripleTrainer whose tables hold random weights, random Adagrad slots and the pattern's flags and gradients;
    returns it with a host copy of that state."""
    fa, fb = PATTERNS[pattern](rng, base_a, base_b)
    ent = rng.standard_normal((len(fa), dim), dtype=np.float32)
    rel = rng.standard_normal((len(fb), dim), dtype=np.float32)
    te, tr = eng.EmbeddingTable(ent, True, opt, device=device), eng.EmbeddingTable(rel, True, opt, device=device)
    state = {}
    for key, tab, f in (("ent", te, fa), ("rel", tr, fb)):
        n = tab.rows
        g = np.zeros((n, tab.pitch), np.float32)
        g[f, :dim] = rng.standard_normal((int(f.sum()), dim), dtype=np.float32)
        tab.grad.copy_(torch.from_numpy(g))
        tab.touched.copy_(torch.from_numpy(f.astype(np.int32)))
        if opt == "Adagrad":
            acc = tab.state1.cpu().numpy()
            acc[:, :dim] = rng.uniform(0.1, 2.0, (n, dim)).astype(np.float32)
            tab.state1.copy_(torch.from_numpy(acc))
        state[key] = snapshot(tab)
    trainer = eng.TripleTrainer(te, tr, eng.loss_cfg("limited", "L2", 0.01, 2.0, 0.2), lr=LR)
    return trainer, state


def snapshot(tab):
    return {"w": tab.weight.cpu().numpy().copy(), "g": tab.grad.cpu().numpy().copy(),
            "acc": None if tab.state1 is None else tab.state1.cpu().numpy().copy(),
            "touched": tab.touched.cpu().numpy().copy(), "dim": tab.dim}


def expect_update(state, opt, lr):
    """TF1 Adagrad (acc += g², x −= lr·g/√acc) or SGD on the flagged rows, in float32; g = 0 and flags cleared there."""
    out = {}
    lr = np.float32(lr)
    for key, s in state.items():
        w, g, acc = s["w"].copy(), s["g"].copy(), None if s["acc"] is None else s["acc"].copy()
        m = s["touched"] != 0
        if opt == "Adagrad":
            acc[m] = acc[m] + g[m] * g[m]
            w[m] = w[m] - lr * g[m] / np.sqrt(acc[m])
        else:
            w[m] = w[m] - lr * g[m]
        g[m] = 0
        out[key] = {"w": w, "g": g, "acc": acc, "flagged": m, "before": s}
    return out


def check_update(trainer, want, rtol=1e-5, atol=1e-7):
    for key, tab in (("ent", trainer.ent), ("rel", trainer.rel)):
        got, e = snapshot(tab), want[key]
        m, s, dim = e["flagged"], e["before"], got["dim"]
        assert not got["touched"].any(), key
        assert not got["g"][m].any(), key
        assert np.array_equal(got["w"][~m], s["w"][~m]), key
        assert np.array_equal(got["g"][~m], s["g"][~m]), key
        assert np.array_equal(got["w"][:, dim:], s["w"][:, dim:]) and not got["g"][:, dim:].any(), key
        np.testing.assert_allclose(got["w"][m], e["w"][m], rtol=rtol, atol=atol, err_msg=key)
        if e["acc"] is not None:
            assert np.array_equal(got["acc"][~m], s["acc"][~m]), key
            assert np.array_equal(got["acc"][:, dim:], s["acc"][:, dim:]), key
            np.testing.assert_allclose(got["acc"][m], e["acc"][m], rtol=rtol, atol=atol, err_msg=key)


def fed_batch(rng, n_ent, n_rel, n_pos, k=3):
    pos = np.stack([rng.integers(0, n_ent, n_pos), rng.integers(0, n_rel, n_pos), rng.integers(0, n_ent, n_pos)]).astype(np.int32)
    neg = np.repeat(pos, k, axis=1)
    neg[0, ::2] = rng.integers(0, n_ent, neg[0, ::2].shape[0])
    neg[2, 1::2] = rng.integers(0, n_ent, neg[2, 1::2].shape[0])
    return pos, np.ascontiguousarray(neg)


def run_fed_step(eng, trainer, pattern, dim, opt, device, base_a, base_b, seed, n_pos, k=3):
    """The one-launch fed step on a placed trainer, checked against the optimiser restatement applied to what the
    two-launch scorer leaves on a second trainer with the same placed state (the scorers' float atomics order their
    sums differently, hence the suite's looser tolerances on the flagged rows)."""
    ref, _ = place(eng, np.random.default_rng(seed), pattern, dim, opt, device, base_a, base_b)
    pos, neg = fed_batch(np.random.default_rng(seed + 1), trainer.ent.rows, trainer.rel.rows, n_pos, k)
    pos_t, neg_t = torch.from_numpy(pos).to(device), torch.from_numpy(neg).to(device)
    ref.score_fed(pos_t, neg_t, grouped=True)
    start = {"ent": snapshot(ref.ent), "rel": snapshot(ref.rel)}
    trainer.step_fed_grouped(pos_t, neg_t)
    check_update(trainer, expect_update(start, opt, LR), rtol=1e-4, atol=1e-6)
