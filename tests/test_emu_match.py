"""CPU: the f-4 kernels' SOURCES (csrc/oea_match.cu: Gale–Shapley rounds, gather-sort of preference lists) on the warp
emulator against the host restatement of modules/finding/alignment.py:171-224 fed with full argsort lists."""
import ctypes as C

import numpy as np
import pytest

from tests.emu import build_emu


@pytest.fixture(scope="module")
def emu():
    return build_emu.load()


def _host_matching(s, cut):
    from openea_b200.modules.finding.alignment import arg_sort, galeshapley
    n1, n2 = s.shape
    m = galeshapley(arg_sort(list(range(n1)), s, "x_", "y_"), arg_sort(list(range(n2)), s.T, "y_", "x_"), cut)
    out = -np.ones(n1, dtype=np.int64)
    for x, y in m.items():
        out[int(x[2:])] = int(y[2:])
    return out


def _p(a):
    return C.c_void_p(a.ctypes.data)


@pytest.mark.parametrize("n1,n2,cut", [(60, 60, 20), (45, 70, 70), (70, 45, 8), (33, 40, 3), (50, 50, 100)])
def test_emulated_gale_shapley_equals_host(emu, n1, n2, cut):
    rng = np.random.default_rng(n1 * 7 + cut)
    s = rng.integers(-6, 7, (n1, n2)).astype(np.float32)          # many exact ties: the tie rules are exercised
    kk = min(cut, n2)
    order = np.argsort(-s, axis=1, kind="stable")[:, :kk]          # what K3's sorted top-k hands over
    idx = np.ascontiguousarray(order.astype(np.int32))
    val = np.ascontiguousarray(np.take_along_axis(s, order, 1).astype(np.float32))
    match = np.full(n1, -7, dtype=np.int32)
    nbytes = emu.oea_gale_shapley_workspace_bytes(n1, n2)
    ws = np.zeros(nbytes // 8 + 1, dtype=np.int64)
    rounds = C.c_int32(0)
    rc = emu.oea_gale_shapley(_p(idx), _p(val), n1, n2, kk, cut, _p(match), _p(ws), ws.nbytes, C.byref(rounds), None)
    assert rc == 0 and 1 <= rounds.value <= cut
    want = _host_matching(s, cut)
    assert np.array_equal(match.astype(np.int64), want), int((match != want).sum())
    held = match[match >= 0]
    assert len(np.unique(held)) == len(held)


def test_emulated_gather_sort_orders_unordered_sets(emu):
    rng = np.random.default_rng(4)
    n, m, k = 37, 210, 100
    mat = rng.integers(-20, 21, (n, m)).astype(np.float32)
    ld = (m + 3) // 4 * 4
    store = np.zeros((n, ld), dtype=np.float32); store[:, :m] = mat
    want = np.argsort(-mat, axis=1, kind="stable")[:, :k]
    idx = np.ascontiguousarray(np.stack([rng.permutation(row) for row in want]).astype(np.int32))     # the set, shuffled
    # ties at the k-th value: any member of the tie class is a legal top-k set; use the exact stable prefix here
    val = np.zeros((n, k), dtype=np.float32)
    assert emu.oea_rows_gather_sort(_p(store), ld, n, k, _p(idx), _p(val), None) == 0
    assert np.array_equal(idx, want.astype(np.int32))
    assert np.array_equal(val, np.take_along_axis(mat, want, 1))
    assert emu.oea_rows_gather_sort(_p(store), ld, n, 129, _p(idx), _p(val), None) == 6      # OEA_ERR_RANGE: k > 128


def test_gale_shapley_argument_checks(emu):
    assert emu.oea_gale_shapley(None, None, 4, 4, 2, 2, None, None, 0, None, None) == 1       # OEA_ERR_NULL
    a = np.zeros(8, dtype=np.int32); v = np.zeros(8, dtype=np.float32); m = np.zeros(4, dtype=np.int32); ws = np.zeros(64, dtype=np.int64)
    assert emu.oea_gale_shapley(_p(a), _p(v), 4, 1, 2, 2, _p(m), _p(ws), ws.nbytes, None, None) == 6     # cut > n2
    assert emu.oea_gale_shapley(_p(a), _p(v), 4, 4, 2, 2, _p(m), _p(ws), 8, None, None) == 7             # workspace too small
