"""A2C on the GPU through the C-ABI: the whole one-pass train() against the executed reference (tests/golden/a2c_*.pt),
the A2C objective against its torch specification, and one user-sized pixel rollout against the oracle run on the same
GPU.  The fused clip+RMSprop kernels are held to a float64 reference in tests/test_gpu_optim_precision.py."""
import pytest
import torch

from oracle import a2c_oracle as AO
from oracle.ops_emul_a2c import A2CEmulOps
from tests.test_a2c_cpu import NAMES, build, check_engine, engine_grads

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cu():
    from sheeprl_b200.lib import CudaOps

    return CudaOps()


def close(a, b, rtol=1e-4, atol=1e-5, what=""):
    a, b = a.detach().cpu(), b.detach().cpu()
    err = (a - b).abs()
    assert bool((err <= atol + rtol * b.abs()).all()), (what, float(err.max()))


@pytest.mark.parametrize("name", NAMES)
def test_engine_matches_reference(cu, name):
    check_engine(name, device="cuda", ops=cu, uint8_image=True)


# ---------------------------------------------------------------------------------------------------------
# a2c_loss against its specification
# ---------------------------------------------------------------------------------------------------------
def _loss_case(N, mode, seed):
    g = torch.Generator().manual_seed(seed)
    dims = [4, 3] if mode == 0 else [3]
    width = sum(dims) if mode == 0 else 2 * sum(dims)
    head = torch.randn(N, width, generator=g)
    if mode == 0:
        actions = torch.cat([torch.nn.functional.one_hot(torch.randint(0, n, (N,), generator=g), n).float() for n in dims], -1)
    else:
        head[:, sum(dims):] *= 0.3                       # log-std around 0
        actions = torch.randn(N, sum(dims), generator=g)
        if mode == 2:
            actions = torch.tanh(actions).clamp(-0.999, 0.999)
    adv, values, returns = (torch.randn(N, generator=g) for _ in range(3))
    return dims, head, actions, adv, values, returns


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("reduce_sum", [False, True])
@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("N,seg", [(1, 1), (5, 1), (20, 5), (20, 6), (300, 64), (2048, 64), (1000, 1000),
                                   (65536, 512), (65536, 65536)])
def test_a2c_loss_kernel(cu, mode, reduce_sum, normalize, N, seg):
    if normalize and (seg == 1 or N % seg == 1):
        pytest.skip("normalisation needs at least two rows per minibatch (refused: see the next test)")
    dims, head, actions, adv, values, returns = _loss_case(N, mode, seed=N + seg + 7 * mode)
    n_seg = (N + seg - 1) // seg
    want = [torch.full_like(head, 7.0), torch.full((N,), 7.0), torch.zeros(n_seg, 3)]
    got = [t.cuda() for t in want]
    args = (seg, dims, mode, normalize, reduce_sum, 0.5, 0.01)
    A2CEmulOps().a2c_loss(head, actions, adv, values, returns, *want, *args)
    cu.a2c_loss(head.cuda(), actions.cuda(), adv.cuda(), values.cuda(), returns.cuda(), *got, *args)
    torch.cuda.synchronize()
    close(got[0], want[0], rtol=2e-4, atol=2e-6, what="dhead")
    close(got[1], want[1], rtol=2e-4, atol=2e-6, what="dvalues")
    # a sum over up to 65536 rows: fp32 accumulation-order error grows like sqrt(rows)
    scale = max(1.0, (seg if reduce_sum else 1) ** 0.5)
    close(got[2], want[2], rtol=2e-4 * scale, atol=1e-5 * scale, what="losses")


def test_a2c_loss_kernel_refuses_a_one_row_minibatch_with_normalisation(cu):
    from sheeprl_b200.lib import B200RLError

    dims, head, actions, adv, values, returns = (t.cuda() if torch.is_tensor(t) else t for t in _loss_case(9, 0, 1))
    out = [torch.zeros_like(head), torch.zeros_like(adv), torch.zeros(3, 3, device="cuda")]
    with pytest.raises(B200RLError, match="two rows"):
        cu.a2c_loss(head, actions, adv, values, returns, *out, 4, dims, 0, True, False, 0.5, 0.0)


# ---------------------------------------------------------------------------------------------------------
# a user-sized rollout without a fixture: 16 envs x 128 steps of 64x64x3 + a vector key, minibatch 64
# ---------------------------------------------------------------------------------------------------------
def test_user_sized_pixel_rollout_matches_the_oracle_on_the_gpu(cu):
    """every gradient tensor against the float64 oracle on the same GPU, to 1e-4 or, where a fp32 computation cannot
    get that close, within twice the error of torch's own fp32 run; the parameters after the RMSprop step"""
    from oracle import ppo_oracle as PO
    from oracle.make_golden_a2c import RMSPROP

    spec = dict(cnn_channels=3, screen=64, mlp_dim=8, dense=64, layers=2, cnn_features=512, mlp_features=64,
                actions_dim=(6,), is_continuous=False, act="tanh")
    hp = dict(vf_coef=0.5, ent_coef=0.01, normalize_advantages=True, max_grad_norm=0.5, loss_reduction="mean")
    N, B = 16 * 128, 64
    init = AO.init_params(spec, 41)
    data = PO.make_rollout(spec, N, 42)
    plan = torch.randperm(N, generator=torch.Generator().manual_seed(43)).view(-1, B).tolist()
    r = {"spec": spec, "hp": hp, "opt": RMSPROP, "init": init, "calls": [{"batch": B}]}
    agent, _, _ = build(r, device="cuda", ops=cu)
    eng = agent._b200_engine
    gdata = {k: v.cuda() for k, v in data.items()}
    gdata["rgb"] = gdata["rgb"].to(torch.uint8)
    eng.train(gdata, plan)
    mine = {k: v.cpu().double() for k, v in engine_grads(eng).items()}

    def oracle(dtype):
        p = {k: v.cuda().to(dtype) for k, v in init.items()}
        opt = AO.make_optimizer(p, RMSPROP)
        grads = {}
        AO.a2c_train(p, opt, spec, {k: v.cuda().to(dtype) for k, v in data.items()}, plan, hp, grads_out=grads)
        return {k: v.detach().cpu().double() for k, v in p.items()}, {k: v.cpu().double() for k, v in grads.items()}

    # float64 is the reference; torch's own fp32 on the same GPU (TF32 off) shows the rounding a fp32 computation of
    # these sums has: the first conv's weight gradient reduces over 2048 x 15 x 15 rows with heavy cancellation
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        p64, g64 = oracle(torch.float64)
        _, g32 = oracle(torch.float32)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    gnorm = float(torch.sqrt(sum((v ** 2).sum() for v in g64.values())))

    def rel(a, k):
        return float((a[k] - g64[k]).norm()) / (float(g64[k].norm()) + 1e-6 * gnorm)

    for k in g64:
        assert rel(mine, k) <= max(1e-4, 2.0 * rel(g32, k)), (k, rel(mine, k), rel(g32, k))
    after = agent.state_dict()
    lr_step = 1e-3 / 0.1
    for k, v in p64.items():
        err = (after[k].cpu().double() - v).abs()
        bad = err > 2e-5 + 1e-4 * v.abs()
        # an element whose accumulated gradient is ~0 can take either sign in RMSprop's first step
        assert float(bad.float().mean()) < 5e-3 and float(err.max()) <= 2.2 * lr_step, (k, int(bad.sum()), float(err.max()))
