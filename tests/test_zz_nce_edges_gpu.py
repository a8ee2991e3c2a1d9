"""GPU: the edge cases of tests/test_emu_nce_edges.py on the device at the H100's sizes, with the splits head_grids
computes from the SM count (the emulator fixes them at 32): every row width 1-128, sampled sets that end a split on a
partial slice (S % 16 != 0) and a partial float4 (S % 4 != 0), a batch past (2·SM − 1)·128 rows (the whole sampled set
one dX split) and a sampled set past it (the whole batch one dW split), S = every class and E = 200 000, contention,
saturated logits against __expf's documented error, NaN-poisoned workspaces; ProjE's batch norms on their degenerate
columns; the unique sampler at the edges of its 4 096-draw rounds; and the pair draw's permutation."""
import numpy as np
import pytest
import torch

from tests import nce_edge_cases as nc

pytestmark = pytest.mark.gpu


@pytest.fixture()
def dev(cuda_device):
    return cuda_device


def _sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def _nce_params(cases):
    out = []
    for c in cases:
        out.append(pytest.param(c, nc.RAW, id=c[0] + "-raw"))
        if not c[4].get("raw_only"):
            out.append(pytest.param(c, nc.NORMED, id=c[0] + "-normalised"))
    return out


@pytest.mark.parametrize("case,norms", _nce_params(nc.NCE_GPU_CASES))
def test_nce_step_at_its_edges(dev, case, norms):
    _, d, S, n, extra = case
    nc.case_nce(dev, d, S, n, extra, norms, sms=_sms(dev))


@pytest.mark.parametrize("which", [0, 1], ids=["rows-past-2SM-tiles", "classes-past-2SM-tiles"])
@pytest.mark.parametrize("norms", [nc.RAW, nc.NORMED], ids=["raw", "normalised"])
def test_nce_step_at_the_split_extremes(dev, which, norms):
    sms = _sms(dev)
    _, d, S, n, extra = nc.split_extreme_cases(sms)[which]
    nc.case_nce(dev, d, S, n, extra, norms, sms=sms)


def test_nce_cases_cover_every_split_structure(dev):
    """On this device's SM count, the case list has, for dX (split of the sampled set) and for dW (split of the batch):
    several splits per tile with a ragged last one, and exactly one split; and sampled sets with S % 4 != 0 and
    S % 16 != 0."""
    sms = _sms(dev)
    cases = nc.NCE_GPU_CASES + nc.split_extreme_cases(sms)
    dx, dw = set(), set()
    for _, d, S, n, _ in cases:
        split_s, split_b = nc.head_splits(n, S, sms)
        dx.add(nc.split_kind(S, split_s))
        dw.add(nc.split_kind(n, split_b))
    print("SMs %d: dX splits %s, dW splits %s" % (sms, sorted(dx), sorted(dw)))
    assert {"ragged", "one"} <= dx and {"ragged", "one"} <= dw, (dx, dw)
    assert any(c[2] % 4 for c in cases) and any(c[2] % 16 for c in cases)


@pytest.mark.parametrize("case", nc.PROJE_GPU_CASES, ids=[c[0] for c in nc.PROJE_GPU_CASES])
def test_proje_step_at_its_edges(dev, case):
    _, d, n, S, extra = case
    nc.case_proje(dev, d, n, S, extra, sms=_sms(dev))


def test_proje_step_past_2sm_row_tiles(dev):
    sms = _sms(dev)
    nc.case_proje(dev, 128, (2 * sms - 1) * nc.KTILE + 1, 17, {}, sms=sms)


@pytest.mark.parametrize("n_classes", [1, 2, 3, 4095, 4096, 4097])
def test_sampler_at_its_edges(dev, n_classes):
    for S in sorted({1, 2, n_classes - 1, n_classes} & set(range(1, n_classes + 1))):
        nc.check_sampler(dev, n_classes, S, 1000 + S)
    nc.check_sampler(dev, n_classes, n_classes, (1 << 63) | 12345)             # a seed with bit 63 set


def test_sampler_at_the_round_edges(dev):
    """The S-th distinct class drawn at the last draw of the first 4 096-draw round and at the first of the next."""
    for seed in range(1, 200):
        last, first = nc.round_edge_sizes(100000, seed)
        if last and first:
            break
    _, tries = nc.check_sampler(dev, 100000, last, seed)
    assert tries == nc.KROUND
    _, tries = nc.check_sampler(dev, 100000, first, seed)
    assert tries == nc.KROUND + 1


def test_sampler_reuses_one_workspace_across_ranges(dev):
    ws, _ = nc.check_sampler(dev, 200000, 4096, 5)
    nc.check_sampler(dev, 3, 3, 6, ws)
    nc.check_sampler(dev, 4097, 4097, 7, ws)


@pytest.mark.parametrize("n", [1, 2, 3, 255, 256, 257, 65535, 65536, 65537, 1000003])
def test_pair_draw_is_the_keyed_permutation(dev, n):
    nc.check_pairs_permutation(dev, n, (1 << 63) | 99, 3, 17)
    nc.check_pairs_permutation(dev, n, 7, 0, 0)
