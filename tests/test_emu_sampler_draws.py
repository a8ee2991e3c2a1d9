"""CPU: path (i)'s device sampler (openea_b200/csrc/oea_sampler.cuh, oea_sampler.cu) on the warp emulator (tests/emu),
draw for draw against the host restatement tests/sampler_oracle.py, at the edges of tests/sampler_draw_cases.py: every
kernel oea_triple_score_sampled dispatches to (its debug dump), the batch producer with both samplers, the one-launch
duo and octet steps (through the tables they leave), three builds of the triple set's filter, and eight mutants of the
sampler source, each of which some case must catch.  tests/test_zz_sampler_draws_gpu.py runs the same cases on the GPU,
with the multi-wave, 10⁶-triple and statistical checks."""
import ctypes as C
import os
import shutil

import numpy as np
import pytest

from tests import sampler_draw_cases as dc
from tests import sampler_oracle as so
from tests.emu import build_emu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {c["name"]: c for c in dc.CASES}


@pytest.fixture()
def emu(monkeypatch):
    lib = build_emu.load()
    build_emu.patch_engine(monkeypatch, lib)
    d = C.c_int(0)
    assert lib.cudaGetDevice(C.byref(d)) != 0, "a CUDA device is visible: the grids would not be the emulator's"
    return lib


@pytest.mark.parametrize("spec", dc.CASES, ids=dc.CASE_IDS)
def test_emulated_sampler_draws_equal_the_model(emu, spec):
    kgs, draws, _ = dc.check_case(spec, "cpu")
    dc.check_case_properties(spec, kgs, draws)


@pytest.mark.parametrize("filt", ["none", "saturated"])
@pytest.mark.parametrize("name", ["dense-half-known", "cand-id", "dense-try10"])
def test_emulated_filter_builds_draw_the_same(emu, name, filt):
    """No filter, or a filter with every bit set (every query goes to the slots): the same draws as the model, whose
    membership test knows neither."""
    dc.check_case(CASES[name], "cpu", kernels=[("duo-or-octet", "L2", 8)], filt=filt)


@pytest.mark.parametrize("name", ["dev-seed", "k17-B5", "k1-B1", "duo-collisions", "dense-try2", "cand-1000"])
def test_emulated_one_launch_step_draws_the_model_batch(emu, name):
    """oea_triple_step_sampled (duo at k ≤ 16, octet above) with the case's dev_seed: the tables after one step equal
    score_fed + apply on the model's batch, and every row that batch does not reference is bit-identical."""
    dc.check_step(CASES[name], "cpu")


def test_emulated_steps_epochs_and_dev_seeds_draw_what_the_model_says(emu):
    """Two steps, two epoch seeds, and a device seed xor-ed into the epoch seed: each dump equals the model's, and the
    model's draws differ between them where they must."""
    spec = dict(CASES["cand-ent2row"], B=40, n_tri=(400, 420))
    kg1, kg2, n_rel, rows = dc.build(spec)
    dcase = dc.DeviceCase(spec, (kg1, kg2), n_rel, rows, "cpu")
    seen = []
    for step, seed in ((1, 4242), (2, 4242), (1, 4243), (1, (1 << 63) | 4242)):
        draws = dc.model(spec, (kg1, kg2), 0, step=step, seed=seed)
        got, n = dcase.dump("L2", 8, step=step, seed=seed)
        assert np.array_equal(got[:n], draws.dump()), (step, seed)
        seen.append(draws)
    for a in range(len(seen)):
        for b in range(a):
            assert not np.array_equal(seen[a].e, seen[b].e)
            assert seen[a].tri.tolist() != seen[b].tri.tolist()
    # seed = epoch ^ dev_seed: the same draws from (epoch ^ x) with dev_seed 0 as from epoch with dev_seed x
    spec2 = dict(spec, seed=4242 ^ 0x5A5A, dev_seed=0x5A5A)
    dc2 = dc.DeviceCase(spec2, (kg1, kg2), n_rel, rows, "cpu")
    got, n = dc2.dump("L1", 8)
    assert np.array_equal(got[:n], dc.model(dict(spec, dev_seed=None), (kg1, kg2), 0).dump())


# ---- the model on its own -------------------------------------------------------------------------------------------
def test_model_slices_follow_batch_py():
    assert so.slices(10, 10, 7, 0) == ((0, 3), (0, 4))           # b1 = int(0.5 · 7) = 3
    assert so.slices(10, 10, 7, 3) == ((9, 1), (10, 0))          # KG 2 past its slices, KG 1 not
    assert so.slices(1, 200, 20, 0) == ((0, 0), (0, 20))         # b1 = int(1/201 · 20) = 0
    assert so.slices(5, 5, 4, 1000) == ((5, 0), (5, 0))          # past the epoch
    # float64 division then multiplication then truncation, not integer arithmetic: 1/3·3 is exactly 1.0 here
    assert so.slices(1, 2, 3, 0)[0] == (0, int(1 / 3 * 3))


def test_model_rng_restates_the_device_formulas():
    """Spot values of rng_base / rng_draw composed with Python integers from the host pcg32, and bounded32 as a
    multiply-high: for C = 3 the draw 0xFFFFFFFF maps to 2, where r % C gives 0."""
    pcg = so.pcg32
    seed, step, p = (1 << 63) | (1 << 31) | 12345, 7, 99
    base = pcg((seed % 2 ** 32) ^ pcg(((seed >> 32) ^ (step * 0x9E3779B9)) % 2 ** 32) ^ ((p * 0x85EBCA6B) % 2 ** 32))
    assert int(so.rng_base(seed, step, np.array([p]))[0]) == base
    want = pcg(base ^ ((0x51DE * 0xC2B2AE35) % 2 ** 32) ^ ((3 * 0x27D4EB2F) % 2 ** 32))
    assert int(so.rng_draw(np.array([base]), 0x51DE, 3)[0]) == want
    assert int(so.bounded32(np.array([0xFFFFFFFF]), 3)[0]) == 2 and int(so.bounded32(np.array([0]), 3)[0]) == 0


def test_model_feistel_positives_are_a_permutation():
    for n in (1, 2, 3, 64, 65, 256, 257, 1000):
        kg = so.HostKG(np.stack([np.arange(n), np.zeros(n, int), np.arange(n)], 1), np.arange(max(n, 4)))
        empty = so.HostKG(np.zeros((0, 3), int), np.arange(4))
        q, tri, hrt = so.positives((kg, empty), n, 0, 99)
        assert sorted(tri.tolist()) == list(range(n)) and (hrt[:, 0] == tri).all()


def test_model_duo_halves_and_warps_draw_the_same():
    """Lane hl owns negative hl and the distinct-position test stays inside a group: the model has no notion of the
    group, so the rule is restated once for a warp and a half-warp.  Its redraw loop re-unsettles a settled lane when
    a lower lane redraws onto its position: with C = k every round is a permutation of the positions."""
    spec = CASES["cand-id-n-equals-k16"]
    kgs = dc.build(spec)[:2]
    draws = dc.model(spec, kgs)
    assert (np.sort(draws.extra, 1) == np.arange(16)).all()


# ---- mutants of the sampler ------------------------------------------------------------------------------------------
MUTANTS = {
    # 1. the highest lane of a group of equal positions keeps its draw
    "highest-lane-keeps": ("oea_sampler.cuh", "unsettled = need && ((same & ((1u << lane) - 1u)) != 0u);",
                           "unsettled = need && ((same & ~((2u << lane) - 1u)) != 0u);"),
    # 2. the duo's two halves share one distinct-position test
    "no-group-bit": ("oea_sampler.cuh", "same = __match_any_sync(active, pos | group_bit);",
                     "same = __match_any_sync(active, pos);"),
    # 3. ent2row ignored: every corrupted entity falls back to the KG's entity list
    "skip-ent2row": ("oea_sampler.cuh", "const int row = __ldg(kg.ent2row + corrupted);",
                     "const int row = -1 + 0 * __ldg(kg.ent2row + corrupted);"),
    # 4. the last round rejects like any other
    "last-round-rejects": ("oea_sampler.cuh", "bool accept = tr == P.max_try - 1;", "bool accept = false;"),
    # 5. one coin per lane in the fast sampler
    "coin-per-lane": ("oea_sampler.cuh", "(rng_draw(base, 0x51DEu, tr) >> 31) != 0;",
                      "(rng_draw(base, 0x51DEu + (uint32_t)hl * 64u, tr) >> 31) != 0;"),
    # 6. r % C in place of the multiply-high
    "modulo-position": ("oea_sampler.cuh", "pos = bounded32(rng_draw(base, (tr << 8) | hl, 0xC0FFEEu + redraw), C);",
                        "pos = rng_draw(base, (tr << 8) | hl, 0xC0FFEEu + redraw) % C;"),
    # 7. KG 2's permutation keyed with KG 1's constant
    "kg2-key-of-kg1": ("oea_sampler.cuh", "seed ^ (q ? 0xA5A5A5A5DEADBEEFull : 0x0123456789ABCDEFull)",
                       "seed ^ 0x0123456789ABCDEFull"),
    # 8. the independent sampler's fallback replaces the head instead of the tail
    "fallback-replaces-head": ("oea_sampler.cu", "                neg_head = false;\n",
                               "                neg_head = true;\n"),
}
# the cases every mutant runs, with the duo / octet kernel and the batch producer
MUTANT_CASES = ["k16-B7", "k32-B37", "cand-ent2row", "cand-id-n-k-plus-1", "duo-collisions", "duo-collisions-k9",
                "duo-cross-half", "dense-try2", "dense-try10", "b1-zero", "feistel-64-and-65"]


def _runs_without_group_bit(spec):
    """Without group_bit, the 2·k lanes of a duo warp need 2·k distinct positions: a list shorter than that never
    settles.  Such cases are left out of that mutant's run."""
    return spec["k"] > dc.DUO_MAX_K or spec["cand"] == "none" or spec["n_cand"] >= 2 * spec["k"]


def _mutant_lib(tmp_path, mutant):
    fname, old, new = MUTANTS[mutant]
    csrc = tmp_path / "openea_b200" / "csrc"
    shutil.copytree(os.path.join(ROOT, "openea_b200", "csrc"), csrc)
    shutil.copytree(os.path.join(ROOT, "include"), tmp_path / "include")
    src = (csrc / fname).read_text()
    assert src.count(old) == 1, "the mutated statement is not in the sampler source any more"
    (csrc / fname).write_text(src.replace(old, new))
    main = tmp_path / "mutant.cpp"
    main.write_text('#include "cuda_host_emu.h"\n#include "openea_b200/csrc/oea_triple.cu"\n'
                    '#include "openea_b200/csrc/oea_sampler.cu"\n#include "openea_b200/csrc/oea_optim_ext.cu"\n')
    return build_emu.load(build_emu.compile(str(main), str(tmp_path / "libmutant.so")),
                          ["oea_triple_score_sampled", "oea_triple_sample_batch", "oea_tripleset_build"])


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_emulated_sampler_mutants_are_caught(tmp_path, monkeypatch, mutant):
    if build_emu.cuda_include() is None:
        pytest.skip("no CUDA headers for the emulator build")
    lib = _mutant_lib(tmp_path, mutant)
    build_emu.patch_engine(monkeypatch, lib)
    caught = []
    for name in MUTANT_CASES:
        if mutant == "no-group-bit" and not _runs_without_group_bit(CASES[name]):
            continue
        try:
            dc.check_case(CASES[name], "cpu", kernels=[("duo-or-octet", "L2", 8)])
        except AssertionError as e:
            caught.append((name, str(e).splitlines()[0][:160]))
    assert caught, "no case catches the mutant " + mutant
    print(mutant, "caught by", caught)
