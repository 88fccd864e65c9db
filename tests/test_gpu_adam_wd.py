"""`b200rl_adam_step_wd` on the GPU: clip + torch.optim.Adam with L2 weight decay against torch.optim.Adam in float64
and against its torch specification (oracle/ops_emul_dv2.py), and weight_decay = 0 bit-identical to `b200rl_adam_step`."""
import pytest
import torch

from oracle.ops_emul_dv2 import DV2EmulOps
from tests.test_adam_weight_decay_cpu import BETAS, EPS, LR, torch_adam_run

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cu():
    from sheeprl_b200.lib import CudaOps

    return CudaOps()


def run(cu, p0, grads, max_norm, wd, offset=0, plain_entry=False):
    """three fused steps on buffers `offset` floats into their allocation (offset 1: the scalar path)"""
    n = p0.numel()

    def buf():
        return torch.zeros(n + offset + 64, device="cuda")[offset:offset + n]

    p, g, m, v = buf(), buf(), buf(), buf()
    p.copy_(p0)
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    normsq, out = torch.zeros((), dtype=torch.float64, device="cuda"), torch.zeros(1, device="cuda")
    for gs in grads:
        g.copy_(gs)
        cu.increment(step)
        if offset == 0:
            cu.sumsq(g, normsq)
        else:                                              # sumsq reads 16-byte aligned buffers only
            normsq.fill_(float((gs.double() ** 2).sum()))
        if plain_entry:
            cu._ck(cu.lib.b200rl_adam_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), normsq.data_ptr(),
                                           step.data_ptr(), out.data_ptr(), n, max_norm, LR, *BETAS, EPS, cu._st()))
        else:
            cu.adam_step(p, g, m, v, normsq, max_norm, LR, *BETAS, EPS, step, out, weight_decay=wd)
    torch.cuda.synchronize()
    return p, m, v, float(out)


CASES = [(4096, 0), (1003, 0), (1003, 1), (1 << 20, 0)]


@pytest.mark.parametrize("wd", [1e-6, 1e-2, 0.5])
@pytest.mark.parametrize("max_norm", [0.0, 0.5, 100.0])
@pytest.mark.parametrize("n,offset", CASES)
def test_adam_weight_decay_matches_torch(cu, wd, max_norm, n, offset):
    gen = torch.Generator().manual_seed(n + offset)
    p0 = torch.randn(n, generator=gen)
    grads = [torch.randn(n, generator=gen) * (0.1 * (s + 1)) for s in range(3)]
    p, m, v, norm = run(cu, p0, grads, max_norm, wd, offset)
    want, st = torch_adam_run(p0, grads, max_norm, wd)
    check(p, m, v, p0, want, st["exp_avg"], st["exp_avg_sq"])
    assert abs(norm - float(grads[-1].double().norm())) <= 1e-5 * float(grads[-1].norm())
    # and against the emulator's specification in fp32
    sp, sm, sv = p0.clone(), torch.zeros(n), torch.zeros(n)
    step, normsq, out = torch.zeros(1, dtype=torch.int32), torch.zeros((), dtype=torch.float64), torch.zeros(1)
    em = DV2EmulOps()
    for gs in grads:
        step += 1
        em.sumsq(gs, normsq)
        em.adam_step(sp, gs, sm, sv, normsq, max_norm, LR, *BETAS, EPS, step, out, weight_decay=wd)
    check(p, m, v, p0, sp, sm, sv)


def check(p, m, v, p0, want_p, want_m, want_v):
    """Norm-wise against the parameter update and the moments: fp32 rounding of a gradient that the decay nearly
    cancels is amplified by up to lr / eps in that one element (a 1M-element case has elements off by 3e-5 in plain
    fp32 torch too), so the element-wise bound is 1 % of lr and the tight bounds are on the norms."""
    p, m, v = (t.cpu().double() for t in (p, m, v))
    want_p, want_m, want_v = (t.double() for t in (want_p, want_m, want_v))
    assert float((p - want_p).norm() / (want_p - p0.double()).norm()) <= 2e-5
    assert float((p - want_p).abs().max()) <= 1e-2 * LR
    assert float((m - want_m).norm() / want_m.norm()) <= 1e-6
    # the kernel forms 1 - b2 from b2 in fp32: 1 - 0.999f is 1.3e-5 off 0.001, in every element of v
    assert float((v - want_v).norm() / want_v.norm()) <= 2e-5


@pytest.mark.parametrize("n,offset", CASES)
def test_zero_weight_decay_is_bit_identical_to_adam_step(cu, n, offset):
    gen = torch.Generator().manual_seed(7 * n + offset)
    p0 = torch.randn(n, generator=gen)
    grads = [torch.randn(n, generator=gen) for _ in range(3)]
    a = run(cu, p0, grads, 0.5, 0.0, offset)
    b = run(cu, p0, grads, 0.5, 0.0, offset, plain_entry=True)
    for x, y in zip(a[:3], b[:3]):
        assert torch.equal(x, y)
    assert a[3] == b[3]
    c = run(cu, p0, grads, 0.5, 1e-6, offset)             # a nonzero decay does change the result
    assert not torch.equal(a[0], c[0])


def test_adam_weight_decay_writes_only_its_range_and_refuses_a_negative_decay(cu):
    from sheeprl_b200.lib import B200RLError

    n = 1003
    base = [torch.full((n + 64,), 7.0, device="cuda") for _ in range(4)]
    p, g, m, v = (t[:n] for t in base)
    m.zero_(), v.zero_(), g.normal_()
    step = torch.ones(1, dtype=torch.int32, device="cuda")
    normsq, out = torch.ones((), dtype=torch.float64, device="cuda"), torch.zeros(1, device="cuda")
    cu.adam_step(p, g, m, v, normsq, 0.0, LR, *BETAS, EPS, step, out, weight_decay=1e-2)
    torch.cuda.synchronize()
    for t in base:
        assert bool((t[n:] == 7.0).all())
    before = p.clone()
    with pytest.raises(B200RLError, match="weight_decay"):
        cu.adam_step(p, g, m, v, normsq, 0.0, LR, *BETAS, EPS, step, out, weight_decay=-1e-6)
    torch.cuda.synchronize()
    assert torch.equal(p, before)
