"""GPU: the edge cases of tests/test_emu_sim_edges.py on the device — every contraction length class, tile and split edge,
kcap bucket, exact tie classes, the stored-matrix kernels' scalar path, the selection's tie rule, the normaliser's
degenerate rows — plus evaluations of more than three resident waves of the H100 (40 000², d = 100) checked by the
interval rule against a float64 reference run on the device in row blocks, and the tensor-core kernel bit for bit in
exact mode."""
import numpy as np
import pytest
import torch

from oracle import finding as orf
from tests import sim_edge_cases as sc
from tests.test_emu_sim_edges import SHAPES

pytestmark = pytest.mark.gpu


@pytest.fixture()
def F(cuda_device, monkeypatch):
    monkeypatch.delenv("OEA_SIM_TC", raising=False)
    monkeypatch.delenv("OEA_SIM_NO_SHORTK", raising=False)
    from openea_b200 import finding
    return finding


def _slots(dev="cuda:0"):
    """Resident CTAs of the tile kernel: 2 per SM."""
    return 2 * torch.cuda.get_device_properties(dev).multi_processor_count


@pytest.mark.parametrize("i,pitch", list(enumerate(sc.PITCHES)))
def test_tile_kernels_exact_at_every_pitch(F, monkeypatch, i, pitch):
    n1, n2 = SHAPES[i % len(SHAPES)]
    d = pitch - (i % 2)
    rng = np.random.default_rng(pitch)
    e1, e2 = sc.ints(rng, n1, d), sc.ints(rng, n2, d)
    e1[0] = 0
    k = min(sc.KS[i % len(sc.KS)], n2)
    sc.check_exact(F, e1, e2, "inner", k, csls_k=min(10, n1, n2), monkeypatch=monkeypatch)
    sc.check_exact(F, e1, e2, "manhattan", k, monkeypatch=monkeypatch)
    sc.check_exact(F, e1, e2, "euclidean", k, monkeypatch=monkeypatch)


@pytest.mark.parametrize("k", sc.KS)
def test_topk_at_every_kcap_edge_with_spread_tie_classes(F, monkeypatch, k):
    rng = np.random.default_rng(100 + k)
    e2, cols = sc.tie_rows(rng, 3000, 20, 300, spread=True)
    e2[cols] = 3.0
    e1 = sc.ints(rng, 700, 20)
    e1[::3] = 3.0
    e1[1::7] = 0.0
    gold = np.arange(700) % 3000
    gold[::3] = cols[len(cols) // 2]
    for metric in ("inner", "manhattan"):
        sc.check_exact(F, e1, e2, metric, k, gold=gold, monkeypatch=monkeypatch)


def test_topk_with_k_equal_to_n2(F):
    rng = np.random.default_rng(5)
    for n2 in (1, 7, 32):
        e1, e2 = sc.ints(rng, 129, 12), sc.ints(rng, n2, 12)
        e1[:40] = 0
        sc.check_exact(F, e1, e2, "inner", n2, shortk=(False,))
        sc.check_exact(F, e1, e2, "manhattan", n2, shortk=(False,))


def test_column_splits_from_one_to_fifty_with_a_ragged_last_split(F):
    rng = np.random.default_rng(11)
    seen = {}
    for n1, n2, k in ((5, 100, 8), (5, 129, 8), (3, 1000, 16), (2, 50 * 128 + 3, 8), (3000, 6403, 8)):
        d = 8
        e2 = sc.ints(rng, n2, d)
        hot = np.unique([0, 1, 64, 65, n2 // 2, n2 - 2, n2 - 1])
        e2[hot] = 3.0
        e1 = sc.ints(rng, n1, d)
        e1[0] = 3.0
        gold = (n2 - 1 - 7 * np.arange(n1)) % n2
        t1, t2 = sc.dev_rows(F, e1), sc.dev_rows(F, e2)
        picked, eff, per = sc.splits_of(F, t1, t2, d)
        assert eff <= picked
        seen[(n1, n2)] = (picked, eff, per)
        sc.check_exact(F, e1, e2, "inner", k, gold=gold, shortk=(False,))
    counts = [v[1] for v in seen.values()]
    assert 1 in counts and 2 in counts and max(counts) >= 50
    picked, eff, per = seen[(2, 50 * 128 + 3)]
    assert 50 * 128 + 3 - (eff - 1) * per * sc.TILE < 8


def test_rank_gold_positions_and_permuted_gold(F):
    rng = np.random.default_rng(12)
    n1, n2, d = 200, 389, 16
    e2 = sc.ints(rng, n2, d)
    e2[[3, 130, 388]] = 3.0
    e1 = sc.ints(rng, n1, d)
    e1[:50] = 3.0
    gold = rng.permutation(np.arange(n1) % n2)
    gold[:8] = [0, n2 - 1, 384, 385, 3, 130, 388, 129]
    for metric in ("inner", "manhattan", "euclidean"):
        sc.check_exact(F, e1, e2, metric, 9, gold=gold, shortk=(False,))
    sc.check_exact(F, e1, e2, "inner", 9, csls_k=10, gold=gold, shortk=(False,))


@pytest.mark.parametrize("metric,csls_k", [("inner", 10), ("inner", 1), ("manhattan", 10), ("manhattan", 32)])
def test_streaming_and_materialised_csls_agree_bit_for_bit(F, metric, csls_k):
    rng = np.random.default_rng(csls_k)
    e1, e2 = sc.ints(rng, 1400, 36), sc.ints(rng, 2600, 36)
    e2[1000:1400] = e1[:400]
    e1[600:700] = 0
    gold = rng.permutation(2600)[:1400]
    sc.check_eval_both_strategies(F, e1, e2, metric, csls_k, gold)


@pytest.mark.parametrize("metric,kind,csls_k,normalize", [
    ("inner", "random", 10, False), ("inner", "near", 10, False), ("cosine", "random", 10, False),
    ("inner", "random", 5, True), ("euclidean", "random", 10, False), ("euclidean", "near", 0, False),
    ("manhattan", "near", 10, False), ("inner", "unit", 0, False)])
def test_real_valued_within_the_fp32_bound(F, metric, kind, csls_k, normalize):
    rng = np.random.default_rng(len(metric) + csls_k)
    for (n1, n2), d in (((129, 257), 100), ((1300, 1310), 300), ((700, 3001), 75)):
        base = sc.real_rows(rng, n2, d, "random")
        e2 = base if kind != "unit" else sc.real_rows(rng, n2, d, "unit")
        e1 = sc.real_rows(rng, n1, d, kind, base=e2)
        sc.check_bound(F, e1, e2, metric, 10, csls_k=csls_k, normalize=normalize, gold=np.arange(n1) % n2)


@pytest.mark.parametrize("ld_extra,col_shift", [(0, 0), (1, 0), (2, 1), (3, 3), (0, 1)])
def test_stored_matrix_rank_scalar_and_vector_paths(F, ld_extra, col_shift):
    for n_cols in (37, 260, 3001):
        ld = (n_cols + 3) // 4 * 4 + ld_extra
        for csls_on in (False, True):
            sc.check_matrix_rank("cuda:0", 900, n_cols, ld, col_shift, csls_on, seed=n_cols + ld_extra)


@pytest.mark.parametrize("n_rows,n_cols,k", [(100, 70, 10), (40, 50, 8), (13, 9, 1), (200, 33, 32), (77, 130, 17), (9, 260, 5),
                                             (3001, 2000, 10), (1100, 5000, 32)])
def test_stored_matrix_row_and_column_means(F, n_rows, n_cols, k):
    rps = sc.check_matrix_means("cuda:0", n_rows, n_cols, k, seed=n_rows + k)
    assert rps % 8 or n_rows < 64


@pytest.mark.parametrize("n_cols,k", [(1, 1), (31, 1), (31, 31), (512, 32), (512, 33), (513, 128), (513, 33), (513, 513),
                                      (2000, 1500), (2000, 10), (15000, 1500)])
def test_selection_takes_the_lowest_index_ties(F, n_cols, k):
    rng = np.random.default_rng(n_cols + k)
    s = sc.selection_matrix(rng, 7, n_cols, k)
    sc.check_select("cuda:0", s, k)
    sc.check_select("cuda:0", s, k, ld_extra=1)
    ids = (rng.permutation(n_cols) * 3 + 1).astype(np.int32)
    sc.check_select("cuda:0", s, k, col_ids=ids)


def test_selection_tie_examples_and_more_rows_than_the_grid(F):
    s = np.zeros((2, 2000), dtype=np.float32)
    s[1, :5] = 5.0
    s[1, 1500:] = 5.0
    sc.check_select("cuda:0", s, 10)
    rng = np.random.default_rng(3)
    n_rows = 4 * torch.cuda.get_device_properties(0).multi_processor_count + 5
    sc.check_select("cuda:0", rng.integers(-2, 3, (n_rows, 2000)).astype(np.float32), 1500)
    sc.check_select("cuda:0", rng.integers(-2, 3, (n_rows, 40)).astype(np.float32), 33)


@pytest.mark.parametrize("cut", [40, 100])
def test_stable_matching_on_selected_lists_equals_host(F, cut):
    from tests.test_stable_matching_gpu import _host_matching
    rng = np.random.default_rng(cut)
    e2 = sc.ints(rng, 330, 8)
    e1 = (e2[rng.integers(0, 330, 300)] + rng.integers(-1, 2, (300, 8))).astype(np.float32)
    s = sc.exact_sim(e1, e2, "inner")
    match, rounds = F.stable_matching(e1, e2, "inner", False, 0, cut)
    assert 1 <= rounds <= cut
    assert np.array_equal(match.cpu().numpy().astype(np.int64), _host_matching(s, cut))


@pytest.mark.parametrize("dim", [1, 3, 31, 32, 33, 100, 300])
def test_normalise_follows_the_oracle(F, dim):
    rng = np.random.default_rng(dim)
    x = sc.normalize_inputs(rng, dim)
    want = orf.normalize_rows(x)
    rtol = sc.gamma(dim) / 2 + 3 * sc.U
    for in_pitch, out_pitch in ((dim, (dim + 3) // 4 * 4), (dim + 5, dim + 9)):
        got = sc.normalize_rows_device("cuda:0", x, in_pitch, out_pitch)
        assert np.array_equal(got[:6], want[:6])
        np.testing.assert_allclose(got, want, rtol=rtol, atol=0)


# the shapes of tests/test_sim_tc_gpu.py
TC_SHAPES = [(128, 256, 32), (1000, 777, 100), (300, 1300, 75), (513, 511, 300), (257, 300, 8), (64, 40, 36), (2000, 3000, 100),
             (1, 1, 4), (129, 127, 16), (127, 129, 20), (256, 128, 12), (100, 5, 128), (5, 100, 132), (40000, 300, 64)]


@pytest.mark.parametrize("n1,n2,d", TC_SHAPES)
def test_tensor_core_matrix_is_exact_on_small_integers(F, n1, n2, d):
    """3xTF32 splits each operand into a TF32 head and a remainder; a small integer is its own head, so every product and
    every partial sum is an exact integer: bit-identical to the reference, with and without (quarter-integer) offsets."""
    rng = np.random.default_rng(n1 + n2 + d)
    e1, e2 = sc.ints(rng, n1, d), sc.ints(rng, n2, d)
    t1, t2 = sc.dev_rows(F, e1), sc.dev_rows(F, e2)
    s = sc.exact_sim(e1, e2, "inner")
    got = F.sim_matrix_tc(t1, t2, d, "inner")[:, :n2].cpu().numpy()
    assert np.array_equal(got, s), int((got != s).sum())
    r = (rng.integers(-40, 41, n1) / 4).astype(np.float32)
    c = (rng.integers(-40, 41, n2) / 4).astype(np.float32)
    got = F.sim_matrix_tc(t1, t2, d, "inner", torch.as_tensor(r, device=t1.device), torch.as_tensor(c, device=t1.device))
    want = sc.csls(s, r, c)
    assert np.array_equal(got[:, :n2].cpu().numpy(), want)


@pytest.mark.parametrize("csls_k,materialize", [(0, False), (10, False), (10, True)])
def test_evaluation_past_three_resident_waves(F, csls_k, materialize):
    """40 000² at d = 100, inner: grids of more than three resident waves.  About 1 000 rows, the first and last row blocks
    included, are checked by the interval rule against float64 computed on the device."""
    blocks, eff = sc.check_waves(F, 40000, 100, csls_k, materialize, seed=40000 + csls_k)
    assert blocks * eff > 3 * _slots()
