"""CPU: the seed-row exchange kernels' SOURCES (csrc/oea_p2p.cu) on the warp emulator.  G "ranks" live in one process — every
rank's exchange window is a host buffer and the peers' window pointers are plain pointers — so the protocol can be checked
without GPUs: slot layout, the double buffer by epoch parity, release / acquire flags, owner rows untouched, the bounded
wait's status word, and the pack / unpack pair of the NCCL transport."""
import ctypes as C

import numpy as np
import pytest

from openea_b200 import lib as L
from tests.emu import build_emu


@pytest.fixture(scope="module")
def emu():
    return build_emu.load()


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _setup(emu, world, rows, pitch, seeds):
    owner = seeds % world
    per_owner = [seeds[owner == g] for g in range(world)]
    max_rows = max(1, max(len(p) for p in per_owner))
    slot = np.full((world, max_rows), -1, dtype=np.int32)
    for g, p in enumerate(per_owner):
        slot[g, :len(p)] = p
    nbytes = emu.oea_seed_xchg_window_bytes(world, max_rows, pitch)
    windows = [np.zeros(nbytes // 8 + 1, dtype=np.int64) for _ in range(world)]
    xs, keep = [], []
    for g in range(world):
        own = np.ascontiguousarray(per_owner[g].astype(np.int32))
        ticket = np.zeros(1, dtype=np.int32)
        win = (C.c_void_p * 16)(*[w.ctypes.data for w in windows])
        xs.append(L.SeedXchg(g, world, pitch, max_rows, win, own.ctypes.data, len(own), slot.ctypes.data, ticket.ctypes.data))
        keep.append((own, ticket))
    return xs, windows, slot, per_owner, keep


@pytest.mark.parametrize("world,pitch", [(2, 8), (3, 100), (8, 12)])
def test_emulated_push_pull_protocol(emu, world, pitch):
    rng = np.random.default_rng(world)
    rows = 97
    seeds = np.unique(rng.integers(0, rows, 40)).astype(np.int64)
    xs, windows, slot, per_owner, keep = _setup(emu, world, rows, pitch, seeds)
    tables = [np.zeros((rows, pitch), dtype=np.float32) for _ in range(world)]
    for epoch in range(1, 6):                                   # five epochs: both parities reused
        for g in range(world):
            tables[g][:] = 1000.0 * epoch + 10.0 * g + np.arange(rows, dtype=np.float32)[:, None] / 128.0
        for g in range(world):                                  # every rank publishes …
            assert emu.oea_seed_push(C.byref(xs[g]), _p(tables[g]), epoch, None) == 0
        for g in range(world):
            tables[g] += 0.5                                    # … trains a step …
        for g in range(world):                                  # … and applies what the peers published
            assert emu.oea_seed_pull(C.byref(xs[g]), _p(tables[g]), epoch, 10 ** 9, None) == 0
        for g in range(world):
            for r in range(rows):
                o = r % world
                base = 1000.0 * epoch + np.float32(r) / 128.0
                if r in set(seeds.tolist()) and o != g:
                    assert np.all(tables[g][r] == np.float32(base + 10.0 * o)), (epoch, g, r)     # the owner's PUBLISHED row
                else:
                    assert np.all(tables[g][r] == np.float32(base + 10.0 * g) + np.float32(0.5)), (epoch, g, r)
            st = C.c_int32(7)
            assert emu.oea_seed_xchg_status(C.byref(xs[g]), C.byref(st)) == 0 and st.value == 0


def test_emulated_pull_times_out_instead_of_hanging(emu):
    world, rows, pitch = 2, 20, 8
    xs, windows, slot, per_owner, keep = _setup(emu, world, rows, pitch, np.arange(rows, dtype=np.int64))
    t = np.ones((rows, pitch), dtype=np.float32)
    before = t.copy()
    # rank 0 pulls epoch 1 although rank 1 never published it: the bounded wait gives up, sets the status word
    assert emu.oea_seed_pull(C.byref(xs[0]), _p(t), 1, 2 * 10 ** 6, None) == 0
    st = C.c_int32(0)
    assert emu.oea_seed_xchg_status(C.byref(xs[0]), C.byref(st)) == 0 and st.value == 1
    assert np.array_equal(t[0::2], before[0::2])               # own rows are never written by a pull
    assert emu.oea_seed_push(C.byref(xs[0]), _p(t), 0, None) == 6          # OEA_ERR_RANGE: epochs start at 1


def test_emulated_pack_unpack_pair(emu):
    world, rows, pitch, rank = 3, 50, 12, 1
    rng = np.random.default_rng(1)
    seeds = np.arange(0, rows, 2)
    owner = seeds % world
    per_owner = [seeds[owner == g] for g in range(world)]
    max_rows = max(len(p) for p in per_owner)
    slot = np.full((world, max_rows), -1, dtype=np.int32)
    for g, p in enumerate(per_owner):
        slot[g, :len(p)] = p
    w = rng.standard_normal((rows, pitch)).astype(np.float32)
    own = np.ascontiguousarray(per_owner[rank].astype(np.int32))
    send = np.zeros((max_rows, pitch), dtype=np.float32)
    assert emu.oea_seed_pack(_p(w), pitch, _p(own), len(own), _p(send), None) == 0
    assert np.array_equal(send[:len(own)], w[own])
    recv = rng.standard_normal((world, max_rows, pitch)).astype(np.float32)
    before = w.copy()
    assert emu.oea_seed_unpack(_p(w), pitch, _p(recv), _p(slot), world, max_rows, rank, None) == 0
    for g in range(world):
        for i, r in enumerate(per_owner[g]):
            assert np.array_equal(w[r], before[r] if g == rank else recv[g, i])
    untouched = np.setdiff1d(np.arange(rows), seeds)
    assert np.array_equal(w[untouched], before[untouched])
