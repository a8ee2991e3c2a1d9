"""CPU: the sampled-NCE head, ProjE's batch norms and the device samplers (openea_b200/csrc/oea_proje.cu) at their edges
on the warp emulator (tests/emu), through the raw C-ABI, against the float64 references of tests/nce_edge_cases.py:
every row width, S % 4 != 0 and S % 16 != 0, S = every class, n = 1, contention on one label / one input, accidental
hits, saturated logits, the expected-count shortcut, NaN-poisoned workspaces, on raw and l2-normalised tables; and three
mutants of the head's kernel source, each of which some case must catch.  tests/test_zz_nce_edges_gpu.py runs the same
cases on the GPU at the H100's sizes and splits."""
import ctypes as C
import os
import shutil

import numpy as np
import pytest
import torch

from openea_b200 import lib as L
from tests import attr2vec_oracle as ao
from tests import nce_edge_cases as nc
from tests.emu import build_emu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture()
def dev(monkeypatch):
    lib = build_emu.load()
    build_emu.patch_engine(monkeypatch, lib)
    d = C.c_int(0)
    assert lib.cudaGetDevice(C.byref(d)) != 0, "a CUDA device is visible: the grids would not be the emulator's"
    return torch.device("cpu")


def _nce_params(cases):
    out = []
    for c in cases:
        out.append(pytest.param(c, nc.RAW, id=c[0] + "-raw"))
        if not c[4].get("raw_only"):
            out.append(pytest.param(c, nc.NORMED, id=c[0] + "-normalised"))
    return out


@pytest.mark.parametrize("case,norms", _nce_params(nc.NCE_EMU_CASES))
def test_emulated_nce_step_at_its_edges(dev, case, norms):
    _, d, S, n, extra = case
    nc.case_nce(dev, d, S, n, extra, norms)


@pytest.mark.parametrize("norms", [nc.RAW, nc.NORMED, {"in": True, "w": False}], ids=["raw", "normalised", "mixed"])
def test_closed_form_reference_is_the_autograd_oracle(norms):
    """The closed-form float64 step of nce_edge_cases equals tests/attr2vec_oracle.py (torch autograd through
    jape.nce_loss) on edge data with repeats, hits and zero rows."""
    tabs, inputs, labels, sampled, tries, scale = nc.nce_case(9, 37, 40, {"kind": "hits"}, 3)
    ref = nc.nce_reference(tabs, norms, inputs, labels, sampled, tries, scale, torch.device("cpu"))
    want_loss, want = ao.fwd_bwd(tabs, norms, inputs, labels, sampled, tries, scale)
    assert ref["loss"] == pytest.approx(want_loss, rel=1e-12)
    for k in ("in", "w", "b"):
        np.testing.assert_allclose(ref[k], want[k].reshape(ref[k].shape), rtol=1e-10, atol=1e-12, err_msg=k)


@pytest.mark.parametrize("case", nc.PROJE_EMU_CASES, ids=[c[0] for c in nc.PROJE_EMU_CASES])
def test_emulated_proje_step_at_its_edges(dev, case):
    _, d, n, S, extra = case
    nc.case_proje(dev, d, n, S, extra)


@pytest.mark.parametrize("n_classes", [1, 2, 3, 40])
def test_emulated_sampler_at_its_edges(dev, n_classes):
    for S in sorted({1, 2, n_classes - 1, n_classes} & set(range(1, n_classes + 1))):
        nc.check_sampler(dev, n_classes, S, 11 + S)
    nc.check_sampler(dev, n_classes, n_classes, (1 << 63) | 12345)              # a seed with bit 63 set


def test_emulated_sampler_at_the_round_edges(dev):
    """The S-th distinct class drawn at the last draw of the first 4 096-draw round and at the first of the next."""
    for seed in range(1, 200):
        last, first = nc.round_edge_sizes(100000, seed)
        if last and first:
            break
    _, tries = nc.check_sampler(dev, 100000, last, seed)
    assert tries == nc.KROUND
    _, tries = nc.check_sampler(dev, 100000, first, seed)
    assert tries == nc.KROUND + 1


def test_emulated_sampler_reuses_one_workspace_across_ranges(dev):
    ws, _ = nc.check_sampler(dev, 4097, 300, 5)
    nc.check_sampler(dev, 3, 3, 6, ws)
    nc.check_sampler(dev, 4097, 4000, 7, ws)


@pytest.mark.parametrize("n", [1, 2, 3, 255, 256, 257, 4097])
def test_emulated_pair_draw_is_the_keyed_permutation(dev, n):
    nc.check_pairs_permutation(dev, n, (1 << 63) | 99, 3, 17)


# ---- mutants of the head -----------------------------------------------------------------------------------------
MUTANTS = {
    # a split that ends at S on a partial slice loses its last S % 16 classes in dX
    "dx-drops-ragged-slice": ("for (int k0 = s0; k0 < s1; k0 += kTk) {", "for (int k0 = s0; k0 + kTk <= s1; k0 += kTk) {"),
    # dW loses the last partial float4 of the sampled columns
    "dw-drops-partial-float4": ("min(kTile, T.ldg - m0)", "(min(kTile, T.num_sampled - m0) & ~3)"),
    # G's padding columns S … ldg − 1 left unwritten: only the poisoned workspace shows it
    "logits-skip-g-padding": ("if (m >= n || s >= T.ldg) continue;", "if (m >= n || s >= S) continue;"),
}
MUTANT_CASES = [c for c in nc.NCE_EMU_CASES if c[0] in ("d17-S17-n31", "d33-S33-n17", "d4-S3-n33")]


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_emulated_head_mutants_are_caught(tmp_path, monkeypatch, mutant):
    if build_emu.cuda_include() is None:
        pytest.skip("no CUDA headers for the emulator build")
    old, new = MUTANTS[mutant]
    csrc = tmp_path / "openea_b200" / "csrc"
    shutil.copytree(os.path.join(ROOT, "openea_b200", "csrc"), csrc)
    shutil.copytree(os.path.join(ROOT, "include"), tmp_path / "include")
    src = (csrc / "oea_proje.cu").read_text()
    assert src.count(old) == 1, "the mutated statement is not in the kernel source any more"
    (csrc / "oea_proje.cu").write_text(src.replace(old, new))
    main = tmp_path / "mutant.cpp"
    main.write_text('#include "cuda_host_emu.h"\n#include "openea_b200/csrc/oea_proje.cu"\n')
    lib = build_emu.load(build_emu.compile(str(main), str(tmp_path / "libmutant.so")),
                         ["oea_nce_score_fed", "oea_nce_workspace_bytes"])
    build_emu.patch_engine(monkeypatch, lib)
    caught = []
    for name, d, S, n, extra in MUTANT_CASES:
        try:
            nc.case_nce(torch.device("cpu"), d, S, n, extra, nc.RAW)
        except AssertionError as e:
            caught.append((name, str(e).splitlines()[0][:200]))
    assert caught, "no case catches the mutant " + mutant
    print(mutant, "caught by", caught)
