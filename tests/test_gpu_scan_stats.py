"""The forward scan's x LayerNorm statistics: every CTA computes them itself from the x rows it receives, and the one
CTA that saves them (to the workspace, for the backward) must have normalised with exactly those values, as must every
other CTA.  Checked on the kernels' own outputs: every row of `x_act` is SiLU(LayerNorm(`x_pre`)) recomputed from the
saved (mean, rstd), and two runs of the fused forward and backward are bitwise identical (statistics included)."""
import pytest
import torch

from tests.test_gpu_rssm_scan import CASES, EPS, make_problem, pre_products, run_bwd, run_fwd

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from sheeprl_b200.lib import CudaOps

    return CudaOps()


def saved_x_stats(ops, ws, T, B, S, D, Dx, R, Dr):
    """(mean, rstd) [T*B][2] of the x LayerNorm as the forward saved them: the workspace ends with the [3][T*B][2]
    statistics block and 256 bytes of slack"""
    n = ops.lib.b200rl_rssm_scan_workspace_bytes(T, B, S, D, Dx, R, Dr)
    off = (n - 256 - 4 * 3 * T * B * 2) // 4
    return ws[off: off + T * B * 2].view(torch.float32).reshape(T * B, 2).clone()


# production S (fix), partial groups everywhere, two x groups per CTA at the Dx limit
@pytest.mark.parametrize("key", ["01", "08", "09b"])
def test_x_act_uses_saved_statistics_and_runs_are_bitwise_identical(ops, key):
    T, B, S, D, R, Dx, Dr, A = CASES[key]
    runs, q = [], None
    for _ in range(2):                                # fresh inputs, workspace and outputs for each run
        dims, t, gr = make_problem(CASES[key], seed=500 + list(CASES).index(key))
        ws = ops.rssm_scan_workspace(T, B, S, D, Dx, R, Dr)
        fwd = run_fwd(ops, dims, 0.01, t, ws)
        stats = saved_x_stats(ops, ws, T, B, S, D, Dx, R, Dr)
        # the second backward takes the first run's q_r / q_g / q_x: the GEMM that makes them may split K with atomics
        if q is None:
            pre_products(ops, dims, t, gr)
            q = {k: gr[k].clone() for k in ("q_r", "q_g", "q_x")}
        else:
            gr.update({k: v.clone() for k, v in q.items()})
        bwd = run_bwd(ops, dims, 0.01, t, gr, ws)
        runs.append((fwd, stats, bwd, t))
    (f1, s1, b1, t1), (f2, s2, b2, _) = runs
    for k in f1:                                      # (the latent padding columns stay NaN)
        v1, v2 = (x[:, : S * D + R] if k == "latent" else x for x in (f1[k], f2[k]))
        assert torch.equal(v1, v2), (k, "second forward differs")
    assert torch.equal(s1, s2), "saved x statistics differ between runs"
    for k in b1:
        assert torch.equal(b1[k], b2[k]), (k, "second backward differs")

    x_pre, x_act = f1["x_pre"].double().cpu(), f1["x_act"].double().cpu()
    mean, rstd = s1[:, 0:1].double().cpu(), s1[:, 1:2].double().cpu()
    # the saved statistics are the rows' own (float64 over the kernel's x_pre, to fp32 rounding)
    m64 = x_pre.mean(1, keepdim=True)
    r64 = (x_pre.var(1, unbiased=False, keepdim=True) + EPS).rsqrt()
    assert float((mean - m64).abs().max()) <= 1e-6 * max(1.0, float(x_pre.abs().max()))
    assert float(((rstd - r64) / r64).abs().max()) <= 1e-5
    # every column, whichever CTA produced it, was normalised with exactly the saved values: recomputed from them the
    # rows agree to the rounding of the fp32 arithmetic and the fast SiLU (~1e-6 of the largest value); statistics off
    # by a relative 1e-4 in one CTA would show as ~1e-4 of the normalised values in its columns
    y = (x_pre - mean) * rstd * t1["lnx_g"].double().cpu() + t1["lnx_b"].double().cpu()
    want = y * torch.sigmoid(y)
    err = float((x_act - want).abs().max()) / float(want.abs().max())
    assert err <= 4e-6, err
