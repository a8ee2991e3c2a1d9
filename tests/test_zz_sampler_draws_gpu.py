"""GPU: path (i)'s device sampler draw for draw against tests/sampler_oracle.py — every case of
tests/sampler_draw_cases.py, batches of more than three resident waves, a 10⁶-triple KG, three builds of the triple
set's filter and the one-launch steps — and, with fixed seeds, the distribution the reference's batch.py prescribes:
fair coins, uniform candidate positions, positives and steps that draw independently, and rejection rates q^max_try.

Each statistical threshold sits at a p-value near 10⁻⁶: 5σ for a normal approximation (two-sided p = 5.7·10⁻⁷), and
scipy's chi-square quantile at 10⁻⁶ for the chi-square statistics.  Under the rule the tests pass for their fixed
seeds; a rule that drifts from it (an unfair coin, a biased or non-mixing position draw) moves the statistic by far
more than these margins at these sample sizes.  The draws are first checked bit for bit against the model, so the
statistics pin the device and the model at once."""
import numpy as np
import pytest
import torch
from scipy import stats

from tests import sampler_draw_cases as dc
from tests import sampler_oracle as so

pytestmark = pytest.mark.gpu
CASES = {c["name"]: c for c in dc.CASES}
P_MIN = 1e-6
SIGMAS = 5.0


def _wave(dev):
    """Warps in one resident wave: 64 per SM."""
    return torch.cuda.get_device_properties(dev).multi_processor_count * 64


def _within(count, n, p, what):
    sd = np.sqrt(n * p * (1 - p))
    assert abs(count - n * p) <= SIGMAS * sd, "%s: %d of %d, expected %.1f ± %.1f" % (what, count, n, n * p, sd)


def _chi2_uniform(values, bins, what):
    counts = np.bincount(values, minlength=bins)
    assert len(counts) == bins, what
    exp = len(values) / bins
    chi = ((counts - exp) ** 2 / exp).sum()
    limit = stats.chi2.isf(P_MIN, bins - 1)
    assert chi <= limit, "%s: chi-square %.1f over %d bins, limit %.1f" % (what, chi, bins, limit)
    return counts


def _independent(a, b, what):
    table = np.zeros((16, 16), dtype=np.int64)
    np.add.at(table, (a, b), 1)
    p = stats.chi2_contingency(table)[1]
    assert p >= P_MIN, "%s: contingency p = %.3g" % (what, p)


def _small_kg2(n, k):
    """A KG 2 of one triple and k + 1 entities past KG 1's, so that nearly the whole batch comes from KG 1."""
    return so.HostKG(np.array([[n, 0, n + 1]]), np.arange(n, n + k + 1))


# ---- the edge table --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("spec", dc.CASES, ids=dc.CASE_IDS)
def test_sampler_draws_equal_the_model(cuda_device, spec):
    kgs, draws, _ = dc.check_case(spec, cuda_device)
    dc.check_case_properties(spec, kgs, draws)


@pytest.mark.parametrize("filt", ["none", "saturated"])
@pytest.mark.parametrize("name", ["dense-half-known", "cand-id", "dense-try10"])
def test_filter_builds_draw_the_same(cuda_device, name, filt):
    dc.check_case(CASES[name], cuda_device, filt=filt)


@pytest.mark.parametrize("name", ["dev-seed", "k17-B5", "k1-B1", "duo-collisions", "dense-try2", "cand-1000",
                                  "k32-B37", "k16-B7"])
def test_one_launch_step_draws_the_model_batch(cuda_device, name):
    dc.check_step(CASES[name], cuda_device)


# ---- past three resident waves, and a 10⁶-triple permutation ---------------------------------------------------------
@pytest.mark.parametrize("k,cand", [(16, "e2r"), (32, "id"), (5, "none")])
def test_sampler_draws_past_three_waves(cuda_device, k, cand):
    spec = dc.case("multi-wave-k%d" % k, k=k, B=50001, n=20000, n_tri=(30000, 30000), cand=cand,
                   n_cand=0 if cand == "none" else 40, seed=(1 << 63) | 31, dev_seed=None)
    assert spec["B"] > 3 * _wave(cuda_device)
    dc.check_case(spec, cuda_device)
    dc.check_step(dict(spec, dev_seed=0x1234_5678_9ABC_DEF0), cuda_device)


def test_sampler_draws_over_a_million_triples(cuda_device):
    """KG 1 of 1 000 003 triples (not a power of two: the Feistel permutation walks cycles), at a step in the middle
    of the epoch."""
    rng = np.random.default_rng(5)
    n, n_tri = 100000, 1_000_003
    i = np.arange(n_tri)
    t1 = np.stack([i % n, i // n, rng.integers(0, n, n_tri)], 1)            # (h, r) distinct for every i
    kg1 = so.HostKG(t1, np.arange(n))
    kg2 = so.HostKG(np.stack([n + i[:5000] % 700, i[:5000] // 700, n + rng.integers(0, 700, 5000)], 1),
                    np.arange(n, n + 700))
    spec = dc.case("million", k=16, B=60000, step=7, n=n, n_rel=11)
    dc.check_case(spec, cuda_device, kernels=[("duo", "L2", 8), ("warp-l1-vec1", "L1", 8)], built=(kg1, kg2, 11, n + 700))


# ---- the distribution ---------------------------------------------------------------------------------------------------
def test_coins_and_candidate_positions_are_uniform(cuda_device):
    """1 000-entry candidate rows of distinct entities (row x lists x + (j + 1)·s mod n for j < 1 000, never x itself,
    which would give back the positive):
    the position of every negative inside its row, recovered from the device's draws, over ≥ 10⁶ draws — a
    chi-square over the 1 000 positions, and the last position at its rate.  The fast sampler's first-round coin per
    positive (one coin covers a round's k negatives) and the independent sampler's first coin per lane: 1/2 ± 5σ."""
    n, nc, s, k = 20000, 1000, 7919, 32
    rng = np.random.default_rng(11)
    t1 = np.unique(np.stack([rng.integers(0, n, 70000), rng.integers(0, 5, 70000), rng.integers(0, n, 70000)], 1), axis=0)
    j = np.arange(nc)
    cand = np.full((n + k + 1, nc), -1, dtype=np.int64)
    cand[:n] = (np.arange(n)[:, None] + (j[None, :] + 1) * s) % n
    kg1 = so.HostKG(t1, np.arange(n), cand)
    kg2 = _small_kg2(n, k)
    spec = dc.case("positions", k=k, B=50000, step=0, seed=0xC0FFEE_0000_0001 | (1 << 63), n=n)
    _, fast, indep = dc.check_case(spec, cuda_device, kernels=[("octet", "L2", 8)], built=(kg1, kg2, 5, n + k + 1))
    one = fast.q == 0
    x = np.where(fast.head, fast.hrt[:, 0:1], fast.hrt[:, 2:3])[one]
    pos = ((fast.e[one] - x) * pow(s, -1, n) - 1) % n
    assert pos.max() < nc and pos.size >= 10 ** 6
    _chi2_uniform(pos.ravel(), nc, "candidate positions")
    _within(int((pos == nc - 1).sum()), pos.size, 1 / nc, "the last position")
    _within(int(fast.coin0[one].sum()), int(one.sum()), 0.5, "fast sampler: first-round coin per positive")
    _within(int(indep.coin0[indep.q == 0].sum()), int(indep.coin0[indep.q == 0].size), 0.5,
            "independent sampler: first coin per lane")


def test_entity_list_draws_are_uniform_and_independent(cuda_device):
    """No candidate lists over a 100 000-entity KG: the draws over the entity list in 1 000 bins; a 16 × 16
    contingency of lane 0's draws of positives p and p + 1, and of the same p at steps s and s + 1 (an rng_base that
    stopped mixing p or the step would make these tables diagonal)."""
    n, k = 100000, 8
    rng = np.random.default_rng(12)
    t1 = np.unique(np.stack([rng.integers(0, n, 130000), rng.integers(0, 5, 130000), rng.integers(0, n, 130000)], 1), axis=0)
    kg1, kg2 = so.HostKG(t1, np.arange(n)), _small_kg2(n, k)
    built = (kg1, kg2, 5, n + k + 1)
    lane0 = []
    for step in (0, 1):
        spec = dc.case("entity-list-step%d" % step, k=k, B=50000, step=step, seed=(1 << 31) | 3, n=n)
        _, fast, _ = dc.check_case(spec, cuda_device, kernels=[("duo", "L2", 8)], samplers=(0,), built=built)
        one = np.nonzero(fast.q == 0)[0]
        if step == 0:
            _chi2_uniform((fast.e[one].ravel() * 1000) // n, 1000, "entity-list positions")
        lane0.append(fast.e[one[:49000], 0] * 16 // n)
    _independent(lane0[0][0::2], lane0[0][1::2], "positives p and p + 1")
    _independent(lane0[0], lane0[1], "the same p at steps s and s + 1")


@pytest.mark.parametrize("max_try", [1, 2, 3])
def test_rejection_rates_are_q_to_the_max_try(cuda_device, max_try):
    """KG 1 is the complete graph of relation 0 on m = 64 entities; every block entity's list holds the 64 block
    entities and 64 others, so each draw is a known triple with probability q = 1/2.  The fast sampler keeps a known
    triple only when every round drew one: a fraction q^max_try of its negatives.  The independent sampler falls back
    to (h, r, uniform entity) after max_try known draws: the same fraction."""
    m, nc, n, k = 64, 128, 400, 16
    rng = np.random.default_rng(13)
    a, b = np.meshgrid(np.arange(m), np.arange(m), indexing="ij")
    t1 = np.stack([a.ravel(), np.zeros(m * m, dtype=np.int64), b.ravel()], 1)
    cand = np.full((n + k + 1, nc), -1, dtype=np.int64)
    for x in range(n):
        cand[x] = rng.permutation(np.concatenate([np.arange(m), rng.choice(np.arange(m, n), nc - m, replace=False)]))
    kg1 = so.HostKG(t1, np.arange(n), cand)
    kg2 = _small_kg2(n, k)
    spec = dc.case("rejections-%d" % max_try, k=k, B=m * m + 1, step=0, max_try=max_try, seed=77 + max_try, n=n)
    _, fast, indep = dc.check_case(spec, cuda_device, kernels=[("duo", "L2", 8)], built=(kg1, kg2, 1, n + k + 1))
    q = m / nc
    one = fast.q == 0
    h, r, t = (fast.hrt[one, c:c + 1] for c in range(3))
    known = so.known_keys(kg1.triples, kg2.triples)
    e, hd = fast.e[one], fast.head[one]
    kn = so.is_known(known, np.where(hd, e, h), r, np.where(hd, t, e))
    _within(int(kn.sum()), kn.size, q ** max_try, "fast sampler: known negatives at max_try %d" % max_try)
    fb = indep.extra[indep.q == 0]
    _within(int(fb.sum()), fb.size, q ** max_try, "independent sampler: fallbacks at max_try %d" % max_try)
