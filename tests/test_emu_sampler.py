"""CPU: the device batch producer (openea_b200/csrc/oea_sampler.cu: k_sample_batch, both reference samplers) on the
warp emulator of tests/emu, checked for the invariants of modules/train/batch.py:36-119 — the same properties
tests/test_zz_triple_ext_gpu.py checks on the GPU."""
import ctypes as C

import numpy as np
import pytest

from openea_b200 import lib as L
from tests.emu import build_emu

M32 = 0xFFFFFFFF
EMPTY = 0xFFFFFFFFFFFFFFFF


def pcg32(x):
    x = (x * 747796405 + 2891336453) & M32
    w = ((((x >> ((x >> 28) + 4)) ^ x) & M32) * 277803737) & M32
    return ((w >> 22) ^ w) & M32


def build_tripleset(triples, ent_bits, rel_bits, capacity=None):
    """Host statement of oea_tripleset_build: open addressing, linear probing, key_hash of oea_common.cuh."""
    cap = capacity or 1 << int(np.ceil(np.log2(max(16, 2 * len(triples)))))
    slots = np.full(cap, EMPTY, dtype=np.uint64)
    for h, r, t in triples.tolist():
        key = (h << (ent_bits + rel_bits)) | (r << ent_bits) | t
        s = pcg32((key & M32) ^ pcg32(((key >> 32) + 0x9E3779B9) & M32)) & (cap - 1)
        while slots[s] != EMPTY and int(slots[s]) != key:
            s = (s + 1) & (cap - 1)
        slots[s] = key
    return slots, cap


@pytest.fixture(scope="module")
def emu():
    return build_emu.load()


def _kgs(rng, n=60, n_rel=5, n_tri=260):
    def kg(lo):
        t = np.stack([rng.integers(lo, lo + n, n_tri), rng.integers(0, n_rel, n_tri), rng.integers(lo, lo + n, n_tri)],
                     axis=1).astype(np.int32)
        return np.ascontiguousarray(np.unique(t, axis=0))
    return kg(0), kg(n), n


@pytest.mark.parametrize("sampler", [0, 1])
@pytest.mark.parametrize("k,with_cand", [(0, False), (1, False), (5, False), (3, True)])
def test_emulated_batch_producer(emu, sampler, k, with_cand):
    rng = np.random.default_rng(31 + 7 * k + sampler)
    t1, t2, n = _kgs(rng)
    ents = [np.arange(0, n, dtype=np.int32), np.arange(n, 2 * n, dtype=np.int32)]
    ent_bits, rel_bits = 7, 3
    slots, cap = build_tripleset(np.concatenate([t1, t2]), ent_bits, rel_bits)
    tset = L.TripleSet(slots.ctypes.data, cap, ent_bits, rel_bits)
    cands = [None, None]
    n_cand = 8
    if with_cand:   # candidate matrix indexed by entity id; rows of the other KG's entities start with −1 (= no list)
        for q in range(2):
            c = np.full((2 * n, n_cand), -1, dtype=np.int32)
            for e in ents[q][::2]:                       # every second entity has a truncated list
                c[e] = rng.choice(ents[q], n_cand, replace=False)
            cands[q] = c
    views = [L.KgView(t.ctypes.data, len(t), e.ctypes.data, len(e), 0 if c is None else c.ctypes.data, 0,
                      0 if c is None else n_cand) for t, e, c in zip((t1, t2), ents, cands)]
    warm_w = np.zeros((2 * n, 8), dtype=np.float32)
    warm = L.Table(warm_w.ctypes.data, 0, 0, 0, 0, 2 * n, 8, 8, 1)
    B = 96
    steps = int(np.ceil((len(t1) + len(t2)) / B))
    b1 = int(len(t1) / (len(t1) + len(t2)) * B)
    known = {tuple(x) for x in np.concatenate([t1, t2]).tolist()}
    seen, n_known, n_neg, dup_rows = [], 0, 0, 0

    def produce(step, seed):
        pos = np.full(3 * B, -7, dtype=np.int32)
        neg = np.full(3 * B * max(k, 1), -7, dtype=np.int32)
        n_pos = C.c_int32(-1)
        smp = L.SampleCfg(B, k, step, 10, seed, 0)
        rc = emu.oea_triple_sample_batch(C.byref(views[0]), C.byref(views[1]), C.byref(tset), C.byref(smp), sampler,
                                         C.byref(warm), pos.ctypes.data, neg.ctypes.data, C.byref(n_pos), None)
        assert rc == 0
        m = n_pos.value
        assert (pos[3 * m:] == -7).all() and (neg[3 * m * k:] == -7).all(), "nothing written past the step's share"
        return pos[:3 * m].reshape(3, m).T.copy(), neg[:3 * m * k].reshape(3, m * k).T.reshape(m, k, 3).copy()

    for step in range(steps):
        p, q = produce(step, 4242)
        want1 = max(0, min((step + 1) * b1, len(t1)) - min(step * b1, len(t1)))
        assert (p[:want1, 0] < n).all() and (p[want1:, 0] >= n).all()
        seen.append(p)
        p2, q2 = produce(step, 4242)
        assert (p2 == p).all() and (q2 == q).all()
        if k == 0:
            continue
        assert (q[:, :, 1] == p[:, None, 1]).all()
        same_h, same_t = q[:, :, 0] == p[:, None, 0], q[:, :, 2] == p[:, None, 2]
        assert (same_h | same_t).all()
        assert ((q[:, :, 0] < n) == (p[:, None, 0] < n)).all() and ((q[:, :, 2] < n) == (p[:, None, 0] < n)).all()
        if with_cand:     # a corrupted end whose original entity has a list must come from that list
            for i in range(len(p)):
                for j in range(k):
                    if not same_h[i, j] and cands[0 if p[i, 0] < n else 1][p[i, 0], 0] >= 0:
                        assert q[i, j, 0] in cands[0 if p[i, 0] < n else 1][p[i, 0]]
                    if not same_t[i, j] and cands[0 if p[i, 0] < n else 1][p[i, 2], 0] >= 0:
                        assert q[i, j, 2] in cands[0 if p[i, 0] < n else 1][p[i, 2]]
        n_known += sum(tuple(x) in known for x in q.reshape(-1, 3).tolist())
        n_neg += q.shape[0] * k
        if sampler == 0 and k > 1 and not with_cand:   # random.sample: distinct inside one try; a re-draw after a
            dup_rows += sum(len({tuple(x) for x in row.tolist()}) < k for row in q)   # rejection may repeat (≈0.5 % here)
    allp = np.concatenate(seen)
    assert len(allp) == len(t1) + len(t2) and {tuple(x) for x in allp.tolist()} == known
    if k:
        assert n_known <= 0.01 * n_neg + 2
        assert dup_rows <= 0.03 * len(allp)


def test_emulated_batch_producer_argument_checks(emu):
    rng = np.random.default_rng(1)
    t1, t2, n = _kgs(rng)
    e1, e2 = np.arange(0, n, dtype=np.int32), np.arange(n, 2 * n, dtype=np.int32)
    slots, cap = build_tripleset(np.concatenate([t1, t2]), 7, 3)
    tset = L.TripleSet(slots.ctypes.data, cap, 7, 3)
    v1 = L.KgView(t1.ctypes.data, len(t1), e1.ctypes.data, len(e1), 0, 0, 0)
    v2 = L.KgView(t2.ctypes.data, len(t2), e2.ctypes.data, len(e2), 0, 0, 0)
    buf = np.zeros(3 * 64 * 4, dtype=np.int32)
    n_pos = C.c_int32(0)
    call = lambda smp, sampler, warm: emu.oea_triple_sample_batch(
        C.byref(v1), C.byref(v2), C.byref(tset), C.byref(smp), sampler, warm, buf.ctypes.data, buf.ctypes.data,
        C.byref(n_pos), None)
    assert call(L.SampleCfg(64, 3, 0, 10, 1, 0), 2, None) == 4        # OEA_ERR_KIND: unknown sampler
    assert call(L.SampleCfg(64, 3, 0, 10, 1, 0), 0, None) == 1        # OEA_ERR_NULL: the fast sampler needs `warm`
    assert call(L.SampleCfg(64, 33, 0, 10, 1, 0), 1, None) == 6       # OEA_ERR_RANGE: more than 32 negatives
    assert call(L.SampleCfg(64, 3, 10 ** 6, 10, 1, 0), 1, None) == 0 and n_pos.value == 0   # past the epoch: empty step
