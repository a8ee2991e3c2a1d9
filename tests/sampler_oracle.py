"""Host restatement of path (i)'s device batch sampler (openea_b200/csrc/oea_sampler.cuh, oea_sampler.cu), integer for
integer, in NumPy and vectorised over positives and lanes: the step's slices (sampler_prepare, batch.py:36-53), the
positive draw (draw_positive), the fast negative sampler (sample_negatives, batch.py:89-119) and the independent one
(k_sample_batch with sampler 1, batch.py:60-86), and the two output formats (the debug dump of the sampled scorers and
the batch producer's index vectors).

Membership comes from a NumPy array of the KGs' (h, r, t), never from the device's triple set or its Bloom filter, so
the model is independent of the hash, the probe and the filter.  The device's RNG is restated from oea_common.cuh:
pcg32 (the one host copy in tests/test_emu_sampler.py), bounded32 = the high word of r·C, and feistel_perm (the host
copy in tests/nce_edge_cases.py).
"""
import numpy as np

from tests.nce_edge_cases import feistel_perm
from tests.test_emu_sampler import pcg32

M32 = 0xFFFFFFFF
M64 = (1 << 64) - 1
KEY_KG1 = 0x0123456789ABCDEF      # draw_positive: seed ^ this keys KG 1's permutation
KEY_KG2 = 0xA5A5A5A5DEADBEEF      # … and this KG 2's
KG2_BIT = 1 << 30                 # dump row[0]: triple index, bit 30 set for KG 2


def _u(x):
    return np.asarray(x, dtype=np.uint64)


def rng_base(seed, step, p):
    """rng_base(seed, step, p) of oea_sampler.cuh: one pcg32 per positive of the step."""
    seed = int(seed) & M64
    inner = int(pcg32(((seed >> 32) ^ ((int(step) * 0x9E3779B9) & M32)) & M32))
    return pcg32(_u(seed & M32) ^ _u(inner) ^ ((_u(p) * np.uint64(0x85EBCA6B)) & np.uint64(M32)))


def rng_draw(base, a, b):
    """rng_draw(base, a, b): pcg32 of the base xor two 32-bit products of the counters."""
    return pcg32(_u(base) ^ ((_u(a) * np.uint64(0xC2B2AE35)) & np.uint64(M32))
                 ^ ((_u(b) * np.uint64(0x27D4EB2F)) & np.uint64(M32)))


def bounded32(r, n):
    """__umulhi(r, n): uniform integer in [0, n) from 32 random bits."""
    return (_u(r) * _u(n)) >> np.uint64(32)


class HostKG:
    """One KG as the device sees it (oea_kg_view): triples [n, 3], the entity list, and optionally the candidate
    matrix, indexed by entity id (`ent2row` None; a row whose first element is −1 has no list) or through `ent2row`
    (−1 = no list)."""

    def __init__(self, triples, entities, cand=None, ent2row=None):
        self.triples = np.ascontiguousarray(np.asarray(triples, dtype=np.int32).reshape(-1, 3))
        self.entities = np.ascontiguousarray(np.asarray(entities, dtype=np.int32))
        self.cand = None if cand is None else np.ascontiguousarray(np.asarray(cand, dtype=np.int32))
        self.ent2row = None if ent2row is None else np.ascontiguousarray(np.asarray(ent2row, dtype=np.int32))
        assert self.ent2row is None or self.cand is not None

    @property
    def n_cand(self):
        return 0 if self.cand is None else self.cand.shape[1]

    def lists(self, corrupted):
        """(row of the candidate matrix or −1 for the entity list, list length C) for each corrupted entity."""
        corrupted = np.asarray(corrupted, dtype=np.int64)
        row = np.full(corrupted.shape, -1, dtype=np.int64)
        if self.cand is not None:
            if self.ent2row is None:
                row = np.where(self.cand[corrupted, 0] >= 0, corrupted, -1)
            else:
                row = self.ent2row[corrupted].astype(np.int64)
        C = np.where(row >= 0, self.n_cand, len(self.entities)).astype(np.uint64)
        return row, C

    def pick(self, row, pos):
        """list[pos] for each (row, position): a candidate-matrix entry, or an entity of the list where row < 0."""
        pos = np.asarray(pos, dtype=np.int64)
        row = np.broadcast_to(row, pos.shape)
        out = np.empty(pos.shape, dtype=np.int64)
        c = row >= 0
        if c.any():
            out[c] = self.cand[row[c], pos[c]]
        out[~c] = self.entities[pos[~c]]
        return out


def triple_keys(h, r, t):
    return (np.asarray(h, dtype=np.int64) << 42) | (np.asarray(r, dtype=np.int64) << 21) | np.asarray(t, dtype=np.int64)


def known_keys(*triple_arrays):
    """The membership set: sorted unique keys of every (h, r, t) of the KGs (ids below 2^21)."""
    allt = np.concatenate([np.asarray(t, dtype=np.int64).reshape(-1, 3) for t in triple_arrays])
    assert allt.size == 0 or allt.max() < 1 << 21
    return np.unique(triple_keys(allt[:, 0], allt[:, 1], allt[:, 2]))


def is_known(known, h, r, t):
    keys = triple_keys(h, r, t)
    i = np.minimum(np.searchsorted(known, keys), max(len(known) - 1, 0))
    return known[i] == keys if len(known) else np.zeros(keys.shape, dtype=bool)


# ---- slices and positives (sampler_prepare, draw_positive) ---------------------------------------------------------
def slice_of(n_triples, batch_kg, step):
    s = step * batch_kg
    e = min(s + batch_kg, n_triples)
    s = min(s, n_triples)
    return s, max(e - s, 0)


def slices(n1, n2, batch_size, step):
    """((start, count) of KG 1, (start, count) of KG 2): b1 = int(n1 / (n1 + n2) · B) in float64, as batch.py:39."""
    b1 = int(n1 / (n1 + n2) * batch_size)
    return slice_of(n1, b1, step), slice_of(n2, batch_size - b1, step)


def positives(kgs, batch_size, step, seed):
    """(q, tri, h, r, t) of every positive p of the step, p in [0, n_pos): the Feistel permutation of start + local
    over the KG's triples, keyed by seed ^ KEY_KG1 / KEY_KG2."""
    sl = slices(len(kgs[0].triples), len(kgs[1].triples), batch_size, step)
    q, tri = [], []
    for j, ((start, count), key) in enumerate(zip(sl, (KEY_KG1, KEY_KG2))):
        n = len(kgs[j].triples)
        idx = np.arange(start, start + count, dtype=np.uint64)
        tri.append(feistel_perm(idx, n, (int(seed) ^ key) & M64).astype(np.int64))
        q.append(np.full(count, j, dtype=np.int64))
    q, tri = np.concatenate(q), np.concatenate(tri)
    hrt = np.zeros((len(q), 3), dtype=np.int64)
    for j in (0, 1):
        m = q == j
        hrt[m] = kgs[j].triples[tri[m]]
    return q, tri, hrt


# ---- negatives -----------------------------------------------------------------------------------------------------
def fast_negatives(kg, known, base, h, r, t, k, max_try):
    """sample_negatives<LANES> for positives of one KG: lane hl < k owns negative hl.  Per round tr < max_try, ONE coin
    for all still-missing negatives; distinct positions among the needing lanes (at iteration `redraw` every unsettled
    lane draws again; the lowest lane of each group of equal positions keeps its draw, the others become unsettled,
    including lanes that had settled); a draw is kept when not a known triple, or always in the last round.
    Returns (e, head, coin of the first round, positions of the first round)."""
    P = len(base)
    e_out = np.zeros((P, k), dtype=np.int64)
    head_out = np.zeros((P, k), dtype=bool)
    coin0 = np.zeros(P, dtype=bool)
    pos0 = np.zeros((P, k), dtype=np.int64)
    if k == 0 or P == 0:
        return e_out, head_out, coin0, pos0
    need = np.ones((P, k), dtype=bool)
    lanes = np.arange(k, dtype=np.uint64)
    lower = np.triu(np.ones((k, k), dtype=bool), 1)          # lower[i, j]: lane i < lane j
    for tr in range(max_try):
        idx = np.nonzero(need.any(1))[0]
        if len(idx) == 0:
            break
        b = base[idx]
        head = (rng_draw(b, 0x51DE, tr) >> np.uint64(31)) != 0
        if tr == 0:
            coin0[:] = head
        row, C = kg.lists(np.where(head, h[idx], t[idx]))
        nd = need[idx]
        pos = np.zeros(nd.shape, dtype=np.uint64)
        uns = nd.copy()
        live = np.arange(len(idx))                          # rows that may still change
        redraw = 0
        while True:
            rr, ll = np.nonzero(uns[live])
            rr = live[rr]
            pos[rr, ll] = bounded32(rng_draw(b[rr], (tr << 8) | lanes[ll], 0xC0FFEE + redraw), C[rr])
            pl, nl = pos[live], nd[live]
            same = (pl[:, :, None] == pl[:, None, :]) & nl[:, :, None] & nl[:, None, :] & lower
            uns[live] = same.any(1)
            live = live[uns[live].any(1)]
            if len(live) == 0:
                break
            redraw += 1
        if tr == 0:
            pos0[:] = pos.astype(np.int64)
        e = kg.pick(row[:, None], pos.astype(np.int64))
        if tr == max_try - 1:
            acc = nd
        else:
            hh, tt = h[idx][:, None], t[idx][:, None]
            kn = is_known(known, np.where(head[:, None], e, hh), r[idx][:, None], np.where(head[:, None], tt, e))
            acc = nd & ~kn
        sub_e, sub_h, sub_n = e_out[idx], head_out[idx], need[idx]
        sub_e[acc] = e[acc]
        sub_h[acc] = np.broadcast_to(head[:, None], acc.shape)[acc]
        sub_n[acc] = False
        e_out[idx], head_out[idx], need[idx] = sub_e, sub_h, sub_n
    return e_out, head_out, coin0, pos0


def independent_negatives(kg, known, base, h, r, t, k, max_try):
    """k_sample_batch, sampler 1: lane j < k flips its own coin per try (counter 0x51DE + 64·j), draws one position
    with replacement, keeps the first draw that is not a known triple; after max_try rejections the negative is
    (h, r, entities[bounded32(rng_draw(base, 0xFA11, j), n_entities)]).
    Returns (e, head, the first try's coins [P, k], fallback flags [P, k])."""
    P = len(base)
    e_out = np.zeros((P, k), dtype=np.int64)
    head_out = np.zeros((P, k), dtype=bool)
    coin0 = np.zeros((P, k), dtype=bool)
    done = np.zeros((P, k), dtype=bool)
    if k == 0 or P == 0:
        return e_out, head_out, coin0, ~done
    lanes = np.arange(k, dtype=np.uint64)
    b = base[:, None]
    for tr in range(max_try):
        head = (rng_draw(b, 0x51DE + 64 * lanes, tr) >> np.uint64(31)) != 0
        if tr == 0:
            coin0 = head.copy()
        row, C = kg.lists(np.where(head, h[:, None], t[:, None]))
        e = kg.pick(row, bounded32(rng_draw(b, (tr << 8) | lanes, 0xC0FFEE), C).astype(np.int64))
        kn = is_known(known, np.where(head, e, h[:, None]), r[:, None], np.where(head, t[:, None], e))
        acc = ~done & ~kn
        e_out[acc], head_out[acc] = e[acc], head[acc]
        done |= acc
    fb = ~done
    pos = bounded32(rng_draw(b, 0xFA11, lanes), len(kg.entities)).astype(np.int64)
    e_fb = kg.entities[np.broadcast_to(pos, (P, k))]
    e_out[fb], head_out[fb] = e_fb[fb], False
    return e_out, head_out, coin0, fb


class Draws:
    """One step's batch: per positive its KG q, triple index, (h, r, t), and per negative the corrupted entity e and
    whether the head was corrupted; plus the first round's coins and positions (fast sampler) or the first try's
    coins and the fallback flags (independent sampler)."""

    def __init__(self, q, tri, hrt, e, head, coin0, extra):
        self.q, self.tri, self.hrt, self.e, self.head, self.coin0, self.extra = q, tri, hrt, e, head, coin0, extra

    @property
    def n_pos(self):
        return len(self.q)

    def dump(self):
        """The sampled scorers' debug dump: row p = [tri | q << 30, head mask, e_0 … e_{k−1}]."""
        k = self.e.shape[1]
        out = np.zeros((self.n_pos, 2 + k), dtype=np.int64)
        out[:, 0] = self.tri + self.q * KG2_BIT
        out[:, 1] = (self.head.astype(np.int64) << np.arange(k, dtype=np.int64)).sum(1) if k else 0
        out[:, 2:] = self.e
        return out.astype(np.uint32).view(np.int32)

    def batch(self):
        """The batch producer's index vectors: pos [3, n_pos] (h | r | t) and neg [3, n_pos·k]."""
        k = self.e.shape[1]
        pos = self.hrt.T.astype(np.int32)
        h, r, t = (np.repeat(self.hrt[:, c], k) for c in range(3))
        e, hd = self.e.ravel(), self.head.ravel()
        neg = np.stack([np.where(hd, e, h), r, np.where(hd, t, e)]).astype(np.int32)
        return pos, neg


def sample(kgs, known, batch_size, k, step, max_try, epoch_seed, dev_seed=None, sampler=0):
    """The whole step as the device draws it (dev_seed: the device scalar xor-ed into the epoch seed)."""
    seed = (int(epoch_seed) ^ (0 if dev_seed is None else int(dev_seed))) & M64
    q, tri, hrt = positives(kgs, batch_size, step, seed)
    base = rng_base(seed, step, np.arange(len(q)))
    P = len(q)
    e = np.zeros((P, k), dtype=np.int64)
    head = np.zeros((P, k), dtype=bool)
    coin0 = np.zeros(P if sampler == 0 else (P, k), dtype=bool)
    extra = np.zeros((P, k), dtype=np.int64 if sampler == 0 else bool)
    fn = fast_negatives if sampler == 0 else independent_negatives
    for j in (0, 1):
        m = q == j
        if m.any():
            e[m], head[m], coin0[m], extra[m] = fn(kgs[j], known, base[m], hrt[m, 0], hrt[m, 1], hrt[m, 2], k, max_try)
    return Draws(q, tri, hrt, e, head, coin0, extra)
