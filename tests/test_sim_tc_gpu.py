"""GPU: the tensor-core similarity kernel (oea_sim_matrix_tc: 3xTF32 wgmma, register accumulators) against the FP32 FFMA
kernel (oea_sim_matrix) — values to fp32 round-off on ragged shapes, every K-chunk count, with and without the CSLS offsets;
and the materialised CSLS evaluation with OEA_SIM_TC=1 against the default path (modules/finding/similarity.py:11-77)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


# 128 x 128 output tiles, 16-wide K chunks: shapes on, just past and just short of each boundary, one and many chunks,
# a grid of more tiles than resident CTAs (persistent loop), and a single row / column
@pytest.mark.parametrize("n1,n2,d", [(128, 256, 32), (1000, 777, 100), (300, 1300, 75), (513, 511, 300), (257, 300, 8), (64, 40, 36),
                                     (2000, 3000, 100), (1, 1, 4), (129, 127, 16), (127, 129, 20), (256, 128, 12), (100, 5, 128),
                                     (5, 100, 132), (40000, 300, 64)])
@pytest.mark.parametrize("csls", [False, True])
def test_tc_matrix_equals_fp32_matrix(cuda_device, n1, n2, d, csls):
    from openea_b200 import finding as F
    rng = np.random.default_rng(n1 + d)
    e1, _ = F.to_device_rows(rng.standard_normal((n1, d)).astype(np.float32), False)
    e2, _ = F.to_device_rows(rng.standard_normal((n2, d)).astype(np.float32), False)
    r = c = None
    if csls:
        r = torch.as_tensor(rng.standard_normal(n1).astype(np.float32), device=e1.device)
        c = torch.as_tensor(rng.standard_normal(n2).astype(np.float32), device=e1.device)
    want = F.sim_matrix(e1, e2, d, "inner", r, c)
    got = F.sim_matrix_tc(e1, e2, d, "inner", r, c)[:, :n2]
    torch.cuda.synchronize()
    scale = float(want.abs().max())
    err = float((got - want).abs().max())
    assert err <= 4e-6 * max(1.0, scale) * np.sqrt(d / 32.0), (err, scale)


def test_materialised_csls_evaluation_with_tensor_cores(cuda_device, monkeypatch):
    from openea_b200 import finding as F
    rng = np.random.default_rng(9)
    e2 = rng.standard_normal((3000, 100)).astype(np.float32)
    e1 = (e2 + 0.7 * rng.standard_normal((3000, 100))).astype(np.float32)
    monkeypatch.setenv("OEA_SIM_TC", "0")
    top1, rk, hits, mr, mrr = F.eval_alignment(e1, e2, [1, 5, 10], "inner", False, 10, materialize=True)
    monkeypatch.setenv("OEA_SIM_TC", "1")
    top1t, rkt, hitst, mrt, mrrt = F.eval_alignment(e1, e2, [1, 5, 10], "inner", False, 10, materialize=True)
    # ranks may differ only where two CSLS values tie to fp32 round-off
    assert int((top1 != top1t).sum()) <= 3 and int((rk != rkt).sum()) <= 6
    assert abs(hits[0] - hitst[0]) <= 0.1 and abs(mrr - mrrt) <= 1e-3
