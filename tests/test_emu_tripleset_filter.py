"""CPU: the blocked Bloom filter in front of the triple membership set (tset_filter_hash / tset_filter_bits /
tset_contains of openea_b200/csrc/oea_common.cuh, built in torch by engine.tripleset_filter).  The filter built in
torch equals one built with the C hash, no key of a set is ever reported absent, the filter lets at most 2 % of
absent keys through to the slot probe, and every sampled kernel draws exactly the same batch with and without it."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from openea_b200 import engine as eng
from openea_b200 import lib as L
from tests.emu import build_emu

CSRC = os.path.join(build_emu.ROOT, "openea_b200", "csrc")
EMPTY = -1

# The product's header compiled for the host: the C statement of the filter (build, query) and a sequential
# restatement of k_tripleset_build, so that 100K-sized sets are built in milliseconds.
HELPER = r"""
#include "cuda_host_emu.h"
#include "%s/oea_common.cuh"
using namespace oea;
extern "C" void filter_build(const uint64_t* keys, int64_t n, uint64_t* words, uint32_t n_words) {
    for (int64_t i = 0; i < n; ++i) {
        const uint32_t fh = tset_filter_hash(keys[i]);
        words[fh & (n_words - 1u)] |= tset_filter_bits(fh);
    }
}
extern "C" void slots_build(const uint64_t* keys, int64_t n, uint64_t* slots, uint32_t capacity) {
    for (uint32_t i = 0; i < capacity; ++i) slots[i] = 0xFFFFFFFFFFFFFFFFull;
    for (int64_t i = 0; i < n; ++i) {
        uint32_t slot = key_hash(keys[i]) & (capacity - 1u);
        while (slots[slot] != 0xFFFFFFFFFFFFFFFFull && slots[slot] != keys[i]) slot = (slot + 1u) & (capacity - 1u);
        slots[slot] = keys[i];
    }
}
extern "C" void contains(const oea_tripleset* s, const uint64_t* keys, int64_t n, uint8_t* out) {
    for (int64_t i = 0; i < n; ++i) out[i] = tset_contains(*s, keys[i]);
}
extern "C" void filter_passes(const uint64_t* words, uint32_t n_words, const uint64_t* keys, int64_t n, uint8_t* out) {
    for (int64_t i = 0; i < n; ++i) {
        const uint32_t fh = tset_filter_hash(keys[i]);
        const uint64_t bits = tset_filter_bits(fh);
        out[i] = (words[fh & (n_words - 1u)] & bits) == bits;
    }
}
"""


@pytest.fixture(scope="module")
def chelp(tmp_path_factory):
    if build_emu.cuda_include() is None:
        pytest.skip("no CUDA headers for the emulator build")
    d = tmp_path_factory.mktemp("filter_helper")
    src = d / "filter_helper.cpp"
    src.write_text(HELPER % CSRC)
    lib = C.CDLL(build_emu.compile(str(src), str(d / "libfilter_helper.so")))
    P = C.c_void_p
    lib.filter_build.argtypes = [P, C.c_int64, P, C.c_uint32]
    lib.slots_build.argtypes = [P, C.c_int64, P, C.c_uint32]
    lib.contains.argtypes = [C.POINTER(L.TripleSet), P, C.c_int64, P]
    lib.filter_passes.argtypes = [P, C.c_uint32, P, C.c_int64, P]
    return lib


def _keys(rng, n, ent_bits=18, rel_bits=10):
    """n distinct packed (h, r, t) keys of the 100K shape's widths, in random order."""
    h = rng.integers(0, 1 << ent_bits, 2 * n, dtype=np.int64)
    r = rng.integers(0, 1 << rel_bits, 2 * n, dtype=np.int64)
    t = rng.integers(0, 1 << ent_bits, 2 * n, dtype=np.int64)
    keys = np.unique((h << (ent_bits + rel_bits)) | (r << ent_bits) | t)
    return rng.permutation(keys)[:n]


def _built(chelp, keys):
    cap = 1 << int(np.ceil(np.log2(max(16, 2 * len(keys)))))
    slots = np.empty(cap, dtype=np.int64)
    chelp.slots_build(keys.ctypes.data, len(keys), slots.ctypes.data, cap)
    return slots


# 126 296 and 826 528 keys: the membership sets of the bench's 15K and 100K shapes
SIZES = [1, 37, 5000, 126296, 826528]


@pytest.mark.parametrize("n", SIZES)
def test_torch_filter_equals_the_c_statement(chelp, n):
    keys = _keys(np.random.default_rng(n), n)
    slots = _built(chelp, keys)
    got = eng.tripleset_filter(torch.from_numpy(slots)).numpy()
    n_words = len(got)
    assert n_words & (n_words - 1) == 0 and 64 * n_words >= 16 * n
    assert n_words * 8 <= max(8, 4 * n)                       # < 32 bits per key: 2 MB at the 100K shape
    want = np.zeros(n_words, dtype=np.uint64)
    chelp.filter_build(keys.ctypes.data, n, want.ctypes.data, n_words)
    assert np.array_equal(got.view(np.uint64), want)


@pytest.mark.parametrize("n", SIZES)
def test_every_key_is_present_and_few_absent_keys_pass_the_filter(chelp, n):
    rng = np.random.default_rng(100 + n)
    keys = _keys(rng, n)
    slots = _built(chelp, keys)
    filt = eng.tripleset_filter(torch.from_numpy(slots)).numpy()
    with_f = L.TripleSet(slots.ctypes.data, len(slots), 18, 10, filt.ctypes.data, len(filt))
    without = L.TripleSet(slots.ctypes.data, len(slots), 18, 10)
    out = np.zeros(n, dtype=np.uint8)
    chelp.contains(C.byref(with_f), keys.ctypes.data, n, out.ctypes.data)
    assert out.all(), "a key of the set reported absent"
    probe = _keys(rng, 200000)
    probe = probe[~np.isin(probe, keys)]
    for view in (with_f, without):
        out = np.ones(len(probe), dtype=np.uint8)
        chelp.contains(C.byref(view), probe.ctypes.data, len(probe), out.ctypes.data)
        assert not out.any()
    passed = np.zeros(len(probe), dtype=np.uint8)
    chelp.filter_passes(filt.ctypes.data, len(filt), probe.ctypes.data, len(probe), passed.ctypes.data)
    assert passed.mean() <= 0.02, passed.mean()


def test_malformed_filter_is_rejected(chelp, monkeypatch):
    build_emu.patch_engine(monkeypatch, build_emu.load())
    rng = np.random.default_rng(3)
    t1, t2, kg1, kg2, tset = _dense_kgs(rng)
    tr = _trainer(rng)
    bad = L.TripleSet(tset.slots.data_ptr(), tset.capacity, tset.ent_bits, tset.rel_bits, tset.filter.data_ptr(), 3)
    with pytest.raises(L.OeaError, match="rc=6"):
        tr.score_sampled(kg1, kg2, _View(bad), 16, 3, 0, 1)


class _View:
    def __init__(self, ts):
        self.ts = ts

    def view(self):
        return self.ts


N, N_REL, D = 24, 2, 12


def _dense_kgs(rng):
    """Two KGs over 24 entities and 2 relations each with ≈ 60 % of all (h, r, t) present, so that a good share of the
    drawn corruptions are known triples and the membership test decides draws."""
    def kg(lo):
        t = np.stack([rng.integers(lo, lo + N, 800), rng.integers(0, N_REL, 800), rng.integers(lo, lo + N, 800)], 1)
        return np.unique(t.astype(np.int32), axis=0)
    t1, t2 = kg(0), kg(N)
    kg1 = eng.DeviceKG(t1, np.arange(0, N), 2 * N, device="cpu")
    kg2 = eng.DeviceKG(t2, np.arange(N, 2 * N), 2 * N, device="cpu")
    return t1, t2, kg1, kg2, eng.DeviceTripleSet([kg1.triples, kg2.triples], 2 * N, N_REL, device="cpu")


def _trainer(rng, loss_norm="L2"):
    ent = rng.standard_normal((2 * N, D)).astype(np.float32)
    rel = rng.standard_normal((N_REL, D)).astype(np.float32)
    return eng.TripleTrainer(eng.EmbeddingTable(ent, True, device="cpu"), eng.EmbeddingTable(rel, True, device="cpu"),
                             eng.loss_cfg("limited", loss_norm, 0.1, 2.0, 0.2), 0.01)


@pytest.mark.parametrize("kernel,loss_norm,k", [("duo", "L2", 6), ("octet", "L2", 20), ("warp", "L1", 6)])
def test_sampled_scorers_draw_the_same_batch_with_and_without_the_filter(chelp, monkeypatch, kernel, loss_norm, k):
    """The duo (k <= 16), octet (k = 17 … 32) and warp-per-positive (L1) scorers: the debug dumps (positives, coins,
    negatives) are identical with and without the filter; with an empty set they are not, so the set decided draws."""
    build_emu.patch_engine(monkeypatch, build_emu.load())
    rng = np.random.default_rng(7 + k)
    t1, t2, kg1, kg2, tset = _dense_kgs(rng)
    assert tset.filter.any()
    empty = torch.full_like(tset.slots, EMPTY)
    views = {"filter": tset,
             "no_filter": _View(L.TripleSet(tset.slots.data_ptr(), tset.capacity, tset.ent_bits, tset.rel_bits)),
             "empty": _View(L.TripleSet(empty.data_ptr(), tset.capacity, tset.ent_bits, tset.rel_bits))}
    B = 48
    dumps = {}
    for name, ts in views.items():
        dumps[name] = []
        for step in range(2):
            dbg = torch.zeros(B, 2 + k, dtype=torch.int32)
            _trainer(np.random.default_rng(0), loss_norm).score_sampled(kg1, kg2, ts, B, k, step, 99, dbg=dbg)
            dumps[name].append(dbg.numpy().copy())
    assert all(np.array_equal(a, b) for a, b in zip(dumps["filter"], dumps["no_filter"]))
    assert not all(np.array_equal(a, b) for a, b in zip(dumps["filter"], dumps["empty"]))


@pytest.mark.parametrize("sampler", [0, 1])
def test_batch_producer_draws_the_same_batch_with_and_without_the_filter(chelp, monkeypatch, sampler):
    """oea_triple_sample_batch, both samplers (sample_negatives<32> and the per-negative sampler of batch.py:60-86)."""
    emu = build_emu.load()
    build_emu.patch_engine(monkeypatch, emu)
    rng = np.random.default_rng(40 + sampler)
    t1, t2, kg1, kg2, tset = _dense_kgs(rng)
    empty = torch.full_like(tset.slots, EMPTY)
    views = {"filter": tset.view(), "no_filter": L.TripleSet(tset.slots.data_ptr(), tset.capacity, tset.ent_bits, tset.rel_bits),
             "empty": L.TripleSet(empty.data_ptr(), tset.capacity, tset.ent_bits, tset.rel_bits)}
    warm_w = np.zeros((2 * N, 12), dtype=np.float32)
    warm = L.Table(warm_w.ctypes.data, 0, 0, 0, 0, 2 * N, 12, 12, 1)
    k1, k2 = kg1.view(), kg2.view()
    B, k = 64, 5
    out = {}
    for name, ts in views.items():
        out[name] = []
        for step in range(2):
            pos = np.zeros(3 * B, dtype=np.int32)
            neg = np.zeros(3 * B * k, dtype=np.int32)
            n_pos = C.c_int32(0)
            smp = L.SampleCfg(B, k, step, 10, 4242, 0)
            assert emu.oea_triple_sample_batch(C.byref(k1), C.byref(k2), C.byref(ts), C.byref(smp), sampler, C.byref(warm),
                                               pos.ctypes.data, neg.ctypes.data, C.byref(n_pos), None) == 0
            out[name].append(np.concatenate([pos, neg]))
    assert all(np.array_equal(a, b) for a, b in zip(out["filter"], out["no_filter"]))
    assert not all(np.array_equal(a, b) for a, b in zip(out["filter"], out["empty"]))
