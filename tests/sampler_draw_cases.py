"""The edge cases of path (i)'s device batch sampler, shared by tests/test_emu_sampler_draws.py (warp emulator) and
tests/test_zz_sampler_draws_gpu.py (H100): each case builds two KGs, candidate lists and a seed, runs the device's
sampling entry points through the raw C-ABI — the debug dump of oea_triple_score_sampled in every kernel it dispatches
to, the batch producer oea_triple_sample_batch with both samplers, and the one-launch step oea_triple_step_sampled —
and compares what they drew with tests/sampler_oracle.py, integer for integer.

The kernel a sampled call reaches follows from its shape: L1 → one warp per positive (k_score_sampled, VEC bucket from
the pitch); squared L2 with pitch ≤ 128 → the duo (k ≤ 16, two positives per warp, a half-warp each) or the octet
(k > 16); squared L2 with pitch > 128 → one warp per positive.
"""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

from openea_b200 import engine as eng
from openea_b200 import lib as L
from tests import sampler_oracle as so

DUO_MAX_K = 16
# (name, score, dim): every kernel oea_triple_score_sampled dispatches to
KERNELS = [("warp-l1-vec1", "L1", 8), ("warp-l1-vec2", "L1", 132), ("warp-l1-vec3", "L1", 260),
           ("warp-l1-vec4", "L1", 388), ("octet-layout-l2", "L2", 8), ("warp-l2", "L2", 132)]


def case(name, **kw):
    spec = dict(name=name, n=48, n_rel=5, n_tri=(150, 170), k=5, B=40, cand="none", n_cand=0, repeat=False, dense=0,
                dense_cand=0, max_try=10, step=1, seed=4242, dev_seed=None, shard=None, no_list_every=3)
    spec.update(kw)
    return spec


# One table of edges, run on the emulator and on the GPU.  k covers 0, 1, 2, 15, 16 (a full half-warp), 17 (past the
# duo), 31 and 32 (a full warp); B covers 1, 2, 3 and odd counts (the duo's idle half); the candidate layouts cover
# none, by entity id with rows starting with −1, through ent2row with −1 entries, n_cand = k, n_cand = k + 1, repeated
# ids and n_cand ≥ 1 000; `dense` makes KG 1 the complete graph of relation 0 on its first m entities, with candidate
# lists inside it, so every corruption is a known triple and every round rejects; seeds set bit 31 and bit 63.
CASES = [
    case("k0", k=0, B=33),
    case("k1-B1", k=1, B=1),
    case("k2-B2", k=2, B=2),
    case("k15-B3", k=15, B=3, n=60),
    case("k16-B7", k=16, B=7, n=60),
    case("k17-B5", k=17, B=5, n=60),
    case("k31-B9", k=31, B=9, n=70),
    case("k32-B37", k=32, B=37, n=70),
    case("cand-id", k=6, B=41, cand="id", n_cand=9),
    case("cand-ent2row", k=6, B=41, cand="e2r", n_cand=9),
    case("cand-id-n-equals-k16", k=16, B=23, cand="id", n_cand=16, n=60, no_list_every=0),
    case("cand-e2r-n-equals-k32", k=32, B=11, cand="e2r", n_cand=32, n=70, no_list_every=0),
    case("cand-id-n-k-plus-1", k=12, B=25, cand="id", n_cand=13),
    case("cand-e2r-n-k-plus-1-k17", k=17, B=13, cand="e2r", n_cand=18, n=60),
    case("cand-repeated-ids", k=8, B=29, cand="e2r", n_cand=10, repeat=True),
    case("cand-1000", k=20, B=15, cand="id", n_cand=1000, n=1100, n_tri=(300, 300)),
    case("duo-collisions", k=16, B=31, cand="e2r", n_cand=16, n=40, no_list_every=0),
    case("duo-collisions-k9", k=9, B=27, cand="id", n_cand=10, n=40, no_list_every=0),
    case("duo-cross-half", k=8, B=31, cand="e2r", n_cand=17, n=40, no_list_every=0),
    case("dense-try1", k=6, B=30, dense=12, dense_cand=8, cand="e2r", n_cand=8, max_try=1, no_list_every=0),
    case("dense-try2", k=6, B=30, dense=12, dense_cand=8, cand="e2r", n_cand=8, max_try=2, no_list_every=0),
    case("dense-try10", k=20, B=30, dense=12, dense_cand=24, cand="id", n_cand=24, max_try=10, n=60, no_list_every=0),
    case("dense-half-known", k=4, B=31, dense=10, dense_cand=10, cand="e2r", n_cand=20, max_try=2, no_list_every=0),
    case("seed-bits-31-63", k=7, B=21, seed=(1 << 63) | (1 << 31) | 77),
    case("dev-seed", k=7, B=21, seed=5, dev_seed=(1 << 63) | 0x80000000F00D),
    case("step0", k=4, B=25, step=0),
    case("feistel-1-and-2", k=2, B=3, n_tri=(1, 2), step=0),
    case("feistel-64-and-65", k=3, B=129, n_tri=(64, 65), step=0),
    case("feistel-256-and-257", k=3, B=100, n_tri=(256, 257), step=2, n=80),
    case("b1-zero", k=3, B=20, n_tri=(1, 200), step=0),
    case("kg2-past-its-slices", k=3, B=7, n_tri=(10, 10), step=3),
    case("past-the-epoch", k=3, B=40, step=1000),
    case("shard-2", k=5, B=33, shard=(1, 2)),
    case("shard-3-empty-rank", k=5, B=2, shard=(2, 3)),
    case("shard-3-duo", k=5, B=17, shard=(0, 3)),
]
CASE_IDS = [c["name"] for c in CASES]


# ---- building a case ---------------------------------------------------------------------------------------------------
def build(spec, rng=None):
    """(HostKG 1, HostKG 2, n_rel, entity rows): KG 1 over entities [0, n), KG 2 over [n, 2n)."""
    rng = np.random.default_rng(zlib.crc32(spec["name"].encode())) if rng is None else rng
    n, n_rel = spec["n"], spec["n_rel"]

    def triples(lo, count):
        t = np.stack([rng.integers(lo, lo + n, 4 * count + 8), rng.integers(0, n_rel, 4 * count + 8),
                      rng.integers(lo, lo + n, 4 * count + 8)], 1)
        t = np.unique(t, axis=0)
        return t[rng.permutation(len(t))[:count]]

    t1 = triples(0, spec["n_tri"][0])
    if spec["dense"]:
        m = spec["dense"]
        a, b = np.meshgrid(np.arange(m), np.arange(m), indexing="ij")
        t1 = np.stack([a.ravel(), np.zeros(m * m, dtype=np.int64), b.ravel()], 1)
    t2 = triples(n, spec["n_tri"][1])
    kgs = []
    for q, t in enumerate((t1, t2)):
        ents = np.arange(q * n, (q + 1) * n)
        cand, e2r = make_candidates(spec, rng, ents, 2 * n)
        kgs.append(so.HostKG(t, ents, cand, e2r))
    return kgs[0], kgs[1], n_rel, 2 * n


def make_candidates(spec, rng, ents, rows):
    """The candidate matrix of one KG (None for cand = 'none').  Rows list entities of the KG (inside the dense block
    for a dense case: its first m entities, then outsiders, so that a draw is known with probability m / n_cand).
    Every `no_list_every`-th entity has no list: by id, its row starts with −1 and the rest of the row is valid ids (the
    device reads only the first element); through ent2row, its entry is −1.  ent2row maps entities to shuffled rows."""
    layout, nc = spec["cand"], spec["n_cand"]
    if layout == "none":
        return None, None
    dense = spec["dense"] and ents[0] == 0
    block, outside = ents[:spec["dense"]], ents[spec["dense"]:]
    lists = []
    for _ in ents:
        if dense and spec["dense_cand"] >= nc:       # every entry inside the block (repeated when the block is short)
            row = rng.choice(block, nc, replace=nc > len(block))
        elif dense:                                  # dense_cand entries inside the block, the rest outside
            row = rng.permutation(np.concatenate([rng.choice(block, spec["dense_cand"], replace=False),
                                                  rng.choice(outside, nc - spec["dense_cand"], replace=False)]))
        else:
            row = rng.choice(ents, nc, replace=bool(spec["repeat"]) or nc > len(ents))
        lists.append(row)
    lists = np.asarray(lists, dtype=np.int64)
    no_list = np.zeros(len(ents), dtype=bool)
    if spec["no_list_every"]:
        no_list[::spec["no_list_every"]] = True
    if layout == "id":
        cand = np.full((rows, nc), -1, dtype=np.int64)
        cand[ents] = lists
        cand[ents[no_list], 0] = -1                 # only the first element marks "no list"
        return cand, None
    perm = rng.permutation(len(ents))
    cand = np.full((len(ents) + 3, nc), -1, dtype=np.int64)       # three spare rows nobody maps to
    cand[perm] = lists
    e2r = np.full(rows, -1, dtype=np.int64)
    e2r[ents] = perm
    e2r[ents[no_list]] = -1
    return cand, e2r


def model(spec, kgs, sampler=0, step=None, seed=None):
    known = so.known_keys(kgs[0].triples, kgs[1].triples)
    return so.sample(kgs, known, spec["B"], spec["k"], spec["step"] if step is None else step, spec["max_try"],
                     spec["seed"] if seed is None else seed, spec["dev_seed"], sampler)


# ---- device side -------------------------------------------------------------------------------------------------------
class DeviceCase:
    """The case's KGs, triple set and tables on `dev` (CPU tensors for the emulator, whose device pointers are host
    pointers).  `filt`: 'built' (the triple set's Bloom filter), 'none' (no filter) or 'saturated' (every bit set)."""

    def __init__(self, spec, kgs, n_rel, rows, dev, filt="built"):
        self.spec, self.kgs, self.dev = spec, kgs, torch.device(dev)
        self.keep = []
        self.views = [self._view(kg) for kg in kgs]
        tri = [torch.as_tensor(kg.triples, device=self.dev) for kg in kgs]
        ts = eng.DeviceTripleSet(tri, rows, n_rel, device=self.dev)
        self.tset_obj = ts
        if filt == "built":
            self.tset = ts.view()
        elif filt == "none":
            self.tset = L.TripleSet(ts.slots.data_ptr(), ts.capacity, ts.ent_bits, ts.rel_bits, 0, 0)
        else:
            self.sat = torch.full_like(ts.filter, -1)
            self.tset = L.TripleSet(ts.slots.data_ptr(), ts.capacity, ts.ent_bits, ts.rel_bits, self.sat.data_ptr(),
                                    self.sat.numel())
        self.rows, self.n_rel = rows, n_rel
        self.dev_seed = None
        if spec["dev_seed"] is not None:
            self.dev_seed = torch.tensor([spec["dev_seed"] - (1 << 64) if spec["dev_seed"] >> 63 else spec["dev_seed"]],
                                         dtype=torch.int64, device=self.dev)

    def _t(self, a):
        if a is None:
            return 0
        t = torch.as_tensor(np.ascontiguousarray(a, dtype=np.int32), device=self.dev)
        self.keep.append(t)
        return t.data_ptr()

    def _view(self, kg):
        return L.KgView(self._t(kg.triples) if len(kg.triples) else 0, len(kg.triples), self._t(kg.entities),
                        len(kg.entities), self._t(kg.cand), self._t(kg.ent2row), kg.n_cand)

    def cfg(self, step=None, seed=None, shard=None, max_try=None):
        s = self.spec
        sr, sw = (0, 0) if shard is None else shard
        return L.SampleCfg(s["B"], s["k"], s["step"] if step is None else step,
                           s["max_try"] if max_try is None else max_try,
                           (s["seed"] if seed is None else seed) & so.M64,
                           0 if self.dev_seed is None else self.dev_seed.data_ptr(), sr, sw)

    def tables(self, d, opt="Adagrad", seed=0):
        rng = np.random.default_rng(seed)
        ent = rng.standard_normal((self.rows, d)).astype(np.float32)
        rel = rng.standard_normal((self.n_rel, d)).astype(np.float32)
        return eng.EmbeddingTable(ent, True, opt, device=self.dev), eng.EmbeddingTable(rel, True, opt, device=self.dev)

    def dump(self, score, d, shard=None, **cfg_kw):
        """oea_triple_score_sampled's debug dump (rows nobody wrote stay −7) and n_pos."""
        s = self.spec
        k = s["k"]
        te, tr = self.tables(d)
        loss = eng.loss_cfg("positive" if k == 0 else "limited", score, 0.01, 2.0, 0.2)
        dbg = torch.full((s["B"] + 1, 2 + k), -7, dtype=torch.int32, device=self.dev)
        n_pos = torch.full((1,), -1, dtype=torch.int32, device=self.dev)
        loss_out = torch.zeros(1, dtype=torch.float64, device=self.dev)
        smp = self.cfg(shard=shard, **cfg_kw)
        lib = L.load()
        rc = lib.oea_triple_score_sampled(C.byref(te.c_struct()), C.byref(tr.c_struct()), C.byref(self.views[0]),
                                          C.byref(self.views[1]), C.byref(self.tset), C.byref(smp), C.byref(loss),
                                          eng._ptr(loss_out), eng._ptr(n_pos), eng._ptr(dbg), eng._stream_ptr())
        assert rc == 0, rc
        return dbg.cpu().numpy(), int(n_pos.cpu()[0])

    def batch(self, sampler, **cfg_kw):
        """oea_triple_sample_batch: (pos [3, n], neg [3, n·k]) and n; nothing written past the step's share."""
        s = self.spec
        B, k = s["B"], s["k"]
        warm = torch.zeros((self.rows, 4), dtype=torch.float32, device=self.dev)
        wt = L.Table(warm.data_ptr(), 0, 0, 0, 0, self.rows, 4, 4, 0)
        pos = torch.full((3 * B + 8,), -7, dtype=torch.int32, device=self.dev)
        neg = torch.full((3 * B * max(k, 1) + 8,), -7, dtype=torch.int32, device=self.dev)
        n = C.c_int32(-1)
        smp = self.cfg(**cfg_kw)
        rc = L.load().oea_triple_sample_batch(C.byref(self.views[0]), C.byref(self.views[1]), C.byref(self.tset),
                                              C.byref(smp), sampler, C.byref(wt), eng._ptr(pos), eng._ptr(neg),
                                              C.byref(n), eng._stream_ptr())
        assert rc == 0, rc
        m = n.value
        p, q = pos.cpu().numpy(), neg.cpu().numpy()
        assert (p[3 * m:] == -7).all() and (q[3 * m * k:] == -7).all(), "written past the step's share"
        return p[:3 * m].reshape(3, m), q[:3 * m * k].reshape(3, m * k), m


# ---- comparisons -------------------------------------------------------------------------------------------------------
def _first_diff(got, want):
    bad = np.argwhere(got != want)
    i = tuple(bad[0])
    return "%d of %d entries differ, first at %s: device %s, model %s" % (len(bad), got.size, i, got[i], want[i])


def check_dump(dc, draws, score, d, shard=None, what=""):
    got, n_pos = dc.dump(score, d, shard=shard)
    want = draws.dump()
    assert n_pos == draws.n_pos, (what, n_pos, draws.n_pos)
    mine = np.zeros(len(got), dtype=bool)
    sr, sw = (0, 1) if shard is None else shard
    mine[sr:draws.n_pos:sw] = True
    assert (got[~mine] == -7).all(), "%s: the dump has rows outside this launch's positives" % what
    g = got[:draws.n_pos][mine[:draws.n_pos]]
    w = want[mine[:draws.n_pos]]
    assert g.shape == w.shape and np.array_equal(g, w), "%s: %s" % (what, _first_diff(g, w))


def check_batch(dc, draws, sampler, what=""):
    pos, neg, m = dc.batch(sampler)
    wp, wn = draws.batch()
    assert m == draws.n_pos, (what, m, draws.n_pos)
    assert np.array_equal(pos, wp), "%s positives: %s" % (what, _first_diff(pos, wp))
    assert np.array_equal(neg, wn), "%s negatives: %s" % (what, _first_diff(neg, wn))


def kernels_for(k):
    """The kernels of KERNELS with the name of the octet-layout kernel this k reaches."""
    out = []
    for name, score, d in KERNELS:
        if name == "octet-layout-l2":
            name = "duo" if k <= DUO_MAX_K else "octet"
        out.append((name, score, d))
    return out


def check_case(spec, dev, kernels=None, filt="built", samplers=(0, 1), built=None):
    """Every sampled kernel's dump and the batch producer's vectors equal the model's draws, for one case (`built`:
    the case's (KG 1, KG 2, n_rel, entity rows) when not build(spec)).  Returns the KGs and the model's draws of
    both samplers."""
    kg1, kg2, n_rel, rows = build(spec) if built is None else built
    kgs = (kg1, kg2)
    dc = DeviceCase(spec, kgs, n_rel, rows, dev, filt)
    fast = model(spec, kgs, 0)
    indep = None
    for name, score, d in kernels_for(spec["k"]) if kernels is None else kernels:
        check_dump(dc, fast, score, d, spec["shard"], "%s %s" % (spec["name"], name))
    if spec["shard"] is None and spec["dev_seed"] is None:      # the batch producer takes neither
        for sampler in samplers:
            draws = fast if sampler == 0 else model(spec, kgs, 1)
            indep = draws if sampler == 1 else indep
            check_batch(dc, draws, sampler, "%s batch producer sampler %d" % (spec["name"], sampler))
    return kgs, fast, indep


def check_case_properties(spec, kgs, draws):
    """What the model's own draws must show for a case, independent of the device."""
    k = spec["k"]
    if draws.n_pos == 0 or k == 0:
        return
    if spec["cand"] != "none" and spec["n_cand"] == k and spec["no_list_every"] == 0:
        # every list has exactly k entries: the first round draws every position once
        assert (np.sort(draws.extra, 1) == np.arange(k)).all()
    if spec["dense"] and spec["dense_cand"] >= spec["n_cand"]:
        in_kg1 = draws.q == 0
        hrt = draws.hrt[in_kg1]
        known = so.known_keys(kgs[0].triples, kgs[1].triples)
        e, hd = draws.e[in_kg1], draws.head[in_kg1]
        h, r, t = hrt[:, 0:1], hrt[:, 1:2], hrt[:, 2:3]
        kn = so.is_known(known, np.where(hd, e, h), r, np.where(hd, t, e))
        assert kn.all(), "a dense case leaves only known corruptions: the last round keeps them"


# ---- the one-launch step ------------------------------------------------------------------------------------------------
def check_step(spec, dev, opt="Adagrad", d=8, lr=0.05):
    """oea_triple_step_sampled (the duo or the octet one-launch step, with dev_seed) against score_fed + apply on the
    model's batch: the referenced rows within the suite's tolerance, every other row bit-identical."""
    kg1, kg2, n_rel, rows = build(spec)
    kgs = (kg1, kg2)
    dc = DeviceCase(spec, kgs, n_rel, rows, dev)
    draws = model(spec, kgs, 0)
    pos, neg = draws.batch()
    cfg = eng.loss_cfg("logistic", "L2")
    a_ent, a_rel = dc.tables(d, opt, seed=3)
    b_ent, b_rel = dc.tables(d, opt, seed=3)
    w0 = [a_ent.raw().cpu().numpy().copy(), a_rel.raw().cpu().numpy().copy()]
    a = eng.TripleTrainer(a_ent, a_rel, cfg, lr)
    smp = dc.cfg()
    n_pos = torch.full((1,), -1, dtype=torch.int32, device=dc.dev)
    ocfg = eng.opt_cfg(a_ent, lr)
    rc = L.load().oea_triple_step_sampled(C.byref(a_ent.c_struct()), C.byref(a_rel.c_struct()), C.byref(dc.views[0]),
                                          C.byref(dc.views[1]), C.byref(dc.tset), C.byref(smp), C.byref(cfg),
                                          C.byref(ocfg), eng._ptr(a.loss_dev), eng._ptr(n_pos), eng._stream_ptr())
    assert rc == 0, rc
    assert int(n_pos.cpu()[0]) == draws.n_pos
    b = eng.TripleTrainer(b_ent, b_rel, cfg, lr)
    t = lambda x: torch.as_tensor(np.ascontiguousarray(x), device=dc.dev)
    if draws.n_pos:
        b.score_fed(t(pos), t(neg) if spec["k"] else None)
        b.apply()
    assert a.read_loss() == pytest.approx(b.read_loss(), rel=1e-4, abs=1e-6)
    used_e = np.zeros(rows, dtype=bool)
    used_r = np.zeros(n_rel, dtype=bool)
    for x in (pos, neg):
        used_e[x[0]] = True
        used_e[x[2]] = True
        used_r[x[1]] = True
    for got_t, want_t, before, used, what in ((a_ent, b_ent, w0[0], used_e, "entity"), (a_rel, b_rel, w0[1], used_r, "relation")):
        got, want = got_t.raw().cpu().numpy(), want_t.raw().cpu().numpy()
        assert np.array_equal(got[~used], before[~used]), \
            "%s %s rows the model's batch does not reference moved: %s" % (spec["name"], what, np.nonzero((got != before).any(1) & ~used)[0][:8])
        np.testing.assert_allclose(got[used], want[used], rtol=1e-4, atol=1e-6, err_msg="%s %s" % (spec["name"], what))
        assert not np.array_equal(got[used], before[used]) or not used.any(), "the step moved nothing"
    return draws
