"""CPU: the path-(iii) kernels at their edges — every contraction length class, row / column tile and split boundary, every
kcap bucket, exact tie classes across threads, tiles and splits, the stored-matrix CSLS kernels' scalar path and row
splits, the radix selection's tie rule and the row normaliser's degenerate rows — executed from the product's kernel
source on the warp emulator (tests/emu) through the product's own host layer and the raw C-ABI, against the float64
references of tests/sim_edge_cases.py.  tests/test_zz_sim_edges_gpu.py runs the same cases on the GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

from openea_b200 import lib as L
from oracle import finding as orf
from tests import sim_edge_cases as sc
from tests.emu import build_emu

SHAPES = [(1, 127), (127, 128), (128, 129), (129, 255), (255, 257), (257, 1)]


@pytest.fixture()
def F(monkeypatch):
    so = build_emu.build()
    if so is None:
        pytest.skip("no CUDA headers for the emulator build")
    lib = C.CDLL(so)
    for name, (res, args) in L.SIGNATURES.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    from openea_b200 import engine as eng
    from openea_b200 import finding
    monkeypatch.setattr(L, "load", lambda: lib)
    monkeypatch.setattr(finding, "_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(finding, "_stream_ptr", lambda: C.c_void_p(0))
    monkeypatch.setattr(eng, "_stream_ptr", lambda: C.c_void_p(0))
    monkeypatch.delenv("OEA_SIM_TC", raising=False)
    monkeypatch.delenv("OEA_SIM_NO_SHORTK", raising=False)
    dev = C.c_int(0)
    assert lib.cudaGetDevice(C.byref(dev)) != 0, "a CUDA device is visible: the emulator's split counts are not the fallback's"
    return finding


@pytest.mark.parametrize("i,pitch", list(enumerate(sc.PITCHES)))
def test_emulated_tile_kernels_exact_at_every_pitch(F, monkeypatch, i, pitch):
    """The three epilogues, the short-K store kernel and the streaming store kernel: inner with CSLS, manhattan, euclidean,
    bit for bit, at a contraction length of each class and on the row / column tile edges."""
    n1, n2 = SHAPES[i % len(SHAPES)]
    d = pitch - (i % 2)                          # odd widths run on a zero-padded pitch
    rng = np.random.default_rng(pitch)
    e1, e2 = sc.ints(rng, n1, d), sc.ints(rng, n2, d)
    e1[0] = 0                                    # a zero row: every inner product ties at 0
    k = min(sc.KS[i % len(sc.KS)], n2)
    sc.check_exact(F, e1, e2, "inner", k, csls_k=min(10, n1, n2), monkeypatch=monkeypatch, wants=i < 2)
    sc.check_exact(F, e1, e2, "manhattan", k, monkeypatch=monkeypatch, wants=False)
    sc.check_exact(F, e1, e2, "euclidean", k, monkeypatch=monkeypatch, wants=False)


@pytest.mark.parametrize("k", sc.KS)
def test_emulated_topk_at_every_kcap_edge_with_spread_tie_classes(F, monkeypatch, k):
    """Duplicated columns spread over every tile (and split) of the row, rows equal to them (the tie class is the top),
    zero rows: the top-k order is (value descending, column ascending) across the 16 threads of a row, the column
    tiles and the split merge."""
    rng = np.random.default_rng(100 + k)
    e2, cols = sc.tie_rows(rng, 300, 20, 40, spread=True)
    e2[cols] = 3.0
    e1 = sc.ints(rng, 130, 20)
    e1[::3] = 3.0                                # the tie class holds these rows' maximum
    e1[1::7] = 0.0
    gold = np.arange(130) % 300
    gold[::3] = cols[len(cols) // 2]             # gold inside the tie class
    for metric in ("inner", "manhattan"):
        sc.check_exact(F, e1, e2, metric, k, gold=gold, shortk=(False,), monkeypatch=monkeypatch, wants=k == 9)


def test_emulated_topk_with_k_equal_to_n2(F):
    rng = np.random.default_rng(5)
    for n2 in (1, 7, 32):
        e1, e2 = sc.ints(rng, 129, 12), sc.ints(rng, n2, 12)
        e1[:40] = 0
        sc.check_exact(F, e1, e2, "inner", n2, shortk=(False,))
        sc.check_exact(F, e1, e2, "manhattan", n2, shortk=(False,), wants=False)


def test_emulated_column_splits_from_one_to_fifty_with_a_ragged_last_split(F):
    """Split counts read from the ABI.  A tie class at the maximum spans the first and the last split (the packed
    atomicMax must keep the lowest column), gold sits in another split than the arg-max, and the last split holds fewer
    valid columns than k."""
    rng = np.random.default_rng(11)
    seen = {}
    for n1, n2, k in ((5, 100, 8), (5, 129, 8), (3, 1000, 16), (2, 50 * 128 + 3, 8)):
        d = 8
        e2 = sc.ints(rng, n2, d)
        hot = np.unique([0, 1, 64, 65, n2 // 2, n2 - 2, n2 - 1])
        e2[hot] = 3.0
        e1 = sc.ints(rng, n1, d)
        e1[0] = 3.0
        gold = np.array([n2 - 1] + [n2 - 1 - 7 * i for i in range(1, n1)])
        t1, t2 = sc.dev_rows(F, e1), sc.dev_rows(F, e2)
        picked, eff, per = sc.splits_of(F, t1, t2, d)
        # pick_splits takes the smallest split count for each tile count per split, so no split is ever empty
        assert eff <= picked
        seen[(n1, n2)] = (picked, eff, per)
        sc.check_exact(F, e1, e2, "inner", k, gold=gold, shortk=(False,), wants=n2 == 129)
    counts = [v[1] for v in seen.values()]
    assert 1 in counts and 2 in counts and max(counts) >= 50
    last = 50 * 128 + 3 - (seen[(2, 50 * 128 + 3)][1] - 1) * seen[(2, 50 * 128 + 3)][2] * sc.TILE
    assert last < 8, "the last split must hold fewer valid columns than k"


def test_emulated_rank_gold_positions_and_permuted_gold(F):
    """Gold at column 0, at the last column, in the ragged last tile, in a tie class and in another split than the
    arg-max; a permuted gold vector."""
    rng = np.random.default_rng(12)
    n1, n2, d = 200, 389, 16
    e2 = sc.ints(rng, n2, d)
    e2[[3, 130, 388]] = 3.0
    e1 = sc.ints(rng, n1, d)
    e1[:50] = 3.0
    gold = rng.permutation(np.arange(n1) % n2)
    gold[:8] = [0, n2 - 1, 384, 385, 3, 130, 388, 129]
    for metric in ("inner", "manhattan", "euclidean"):
        sc.check_exact(F, e1, e2, metric, 9, gold=gold, shortk=(False,), wants=False)
    sc.check_exact(F, e1, e2, "inner", 9, csls_k=10, gold=gold, shortk=(False,), wants=False)


@pytest.mark.parametrize("metric,csls_k", [("inner", 10), ("inner", 1), ("manhattan", 10), ("manhattan", 32)])
def test_emulated_streaming_and_materialised_csls_agree_bit_for_bit(F, metric, csls_k):
    rng = np.random.default_rng(csls_k)
    e1, e2 = sc.ints(rng, 140, 36), sc.ints(rng, 260, 36)
    e2[100:140] = e1[:40]
    e1[60:70] = 0
    gold = rng.permutation(260)[:140]
    sc.check_eval_both_strategies(F, e1, e2, metric, csls_k, gold)


@pytest.mark.parametrize("metric,kind,csls_k,normalize,n1,n2,d", [
    ("inner", "random", 10, False, 129, 257, 100), ("inner", "near", 10, False, 130, 131, 300),
    ("cosine", "random", 10, False, 130, 131, 300), ("inner", "random", 5, True, 129, 257, 100),
    ("euclidean", "random", 10, False, 129, 257, 100), ("euclidean", "near", 0, False, 130, 131, 300),
    ("manhattan", "near", 10, False, 129, 257, 100), ("inner", "unit", 0, False, 130, 131, 300)])
def test_emulated_real_valued_within_the_fp32_bound(F, metric, kind, csls_k, normalize, n1, n2, d):
    rng = np.random.default_rng(len(metric) + csls_k)
    base = sc.real_rows(rng, n2, d, "random")
    e2 = base if kind != "unit" else sc.real_rows(rng, n2, d, "unit")
    e1 = sc.real_rows(rng, n1, d, kind, base=e2)
    sc.check_bound(F, e1, e2, metric, 10, csls_k=csls_k, normalize=normalize, gold=np.arange(n1) % n2)


@pytest.mark.parametrize("ld_extra,col_shift", [(0, 0), (1, 0), (2, 1), (3, 3), (0, 1)])
def test_emulated_stored_matrix_rank_scalar_and_vector_paths(F, ld_extra, col_shift):
    """ld % 4 != 0 or an unaligned col_off take the scalar loop; gold at every position of a float4 group."""
    for n_cols in (37, 260):
        ld = (n_cols + 3) // 4 * 4 + ld_extra
        for csls_on in (False, True):
            sc.check_matrix_rank("cpu", 90, n_cols, ld, col_shift, csls_on, seed=n_cols + ld_extra)


@pytest.mark.parametrize("n_rows,n_cols,k", [(100, 70, 10), (40, 50, 8), (13, 9, 1), (200, 33, 32), (77, 130, 17), (9, 260, 5)])
def test_emulated_stored_matrix_row_and_column_means(F, n_rows, n_cols, k):
    """Column means over row splits whose length is not a multiple of the 8-row unroll, and with fewer rows than 8·kcap."""
    rps = sc.check_matrix_means("cpu", n_rows, n_cols, k, seed=n_rows + k)
    assert rps % 8 or n_rows < 64


@pytest.mark.parametrize("n_cols,k", [(1, 1), (31, 1), (31, 31), (512, 32), (512, 33), (513, 128), (513, 33), (513, 513),
                                      (2000, 1500), (2000, 10), (9000, 1500)])
def test_emulated_selection_takes_the_lowest_index_ties(F, n_cols, k):
    rng = np.random.default_rng(n_cols + k)
    s = sc.selection_matrix(rng, 7, n_cols, k)
    sc.check_select("cpu", s, k)
    sc.check_select("cpu", s, k, ld_extra=1)
    ids = (rng.permutation(n_cols) * 3 + 1).astype(np.int32)
    sc.check_select("cpu", s, k, col_ids=ids)


def test_emulated_selection_tie_examples_and_more_rows_than_the_grid(F):
    """The all-zero row must give columns 0 … 9, the row with 5.0 at columns 0–4 and 1500–1999 columns 0 … 4 and
    1500 … 1504; and a grid-stride pass over more rows than 4 CTAs per SM."""
    s = np.zeros((2, 2000), dtype=np.float32)
    s[1, :5] = 5.0
    s[1, 1500:] = 5.0
    sc.check_select("cpu", s, 10)
    rng = np.random.default_rng(3)
    sc.check_select("cpu", rng.integers(-2, 3, (4 * 132 + 5, 40)).astype(np.float32), 33)


@pytest.mark.parametrize("cut", [40, 100])
def test_emulated_stable_matching_on_selected_lists_equals_host(F, cut):
    from tests.test_emu_match import _host_matching
    rng = np.random.default_rng(cut)
    e2 = sc.ints(rng, 130, 8)
    e1 = (e2[rng.integers(0, 130, 110)] + rng.integers(-1, 2, (110, 8))).astype(np.float32)
    s = sc.exact_sim(e1, e2, "inner")
    match, rounds = F.stable_matching(e1, e2, "inner", False, 0, cut)
    assert 1 <= rounds <= cut
    assert np.array_equal(match.numpy().astype(np.int64), _host_matching(s, cut))


@pytest.mark.parametrize("dim", [1, 3, 31, 32, 33, 100, 300])
def test_emulated_normalise_follows_sklearn(F, dim):
    sk = pytest.importorskip("sklearn.preprocessing")
    rng = np.random.default_rng(dim)
    x = sc.normalize_inputs(rng, dim)
    want = sk.normalize(x)
    assert np.array_equal(orf.normalize_rows(x)[:6], want[:6])              # degenerate rows: the same bits
    # the norms are summed in different orders: each entry within γ_dim/2 of the sum, plus sqrt and the scaling
    rtol = sc.gamma(dim) / 2 + 3 * sc.U
    np.testing.assert_allclose(orf.normalize_rows(x), want, rtol=rtol, atol=0)
    for in_pitch, out_pitch in ((dim, (dim + 3) // 4 * 4), (dim + 5, dim + 9)):
        got = sc.normalize_rows_device("cpu", x, in_pitch, out_pitch)
        assert np.array_equal(got[:5], x[:5]), "rows with a norm below 10·eps stay unchanged"
        np.testing.assert_allclose(got, want, rtol=rtol, atol=0)
