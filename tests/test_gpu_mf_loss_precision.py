"""Every model-free objective and sampling kernel (csrc/ppo.cu, csrc/sac.cu and the GAE scan of csrc/replay.cu) against
the float64 reference of oracle/mf_loss_ref.py, across each launch's warp, block and grid edges.

Each case runs the kernel twice and checks:
  - error <= bound element by element (not relative to the largest entry, so one wrong row fails);
  - the two runs bit-identical: none of these kernels uses float atomics;
  - NaN guard bands around every input and output view untouched, including the padding of a strided SAC action
    view (ld_action > A) and between the critics of a padded [nets, stride_net] layout;
  - the inputs not written.
ppo_act's discrete actions must equal fp32 torch's argmax of p / q exactly; only its log-prob has a bound.
`gae` has no caller in the engines today (PPO and A2C take the reference's host `gae`); it is held to the same
standard because the C-ABI exports it.
Cases, input families and the emulators' margins are in tests/test_mf_loss_ref_cpu.py, which also shows the bounds
reject a gradient through the clipped branch, a biased std, eps inside the root, a strict value-clip mask, the entropy
gradient without + H, one logsumexp over every head, the tanh correction at atanh(a), SAC's correction without its
1e-6, a log-std clamp that passes the gradient, DroQ's dq = -1 / B, a shifted A2C minibatch and GAE's dones[t + 1].
"""
import json
import math
import os

import pytest
import torch

from oracle import mf_loss_ref as R
from tests.test_gpu_ln_precision import Guarded
from tests.test_loss_ref_cpu import gen, worst
from tests.test_mf_loss_ref_cpu import (A2C_CASES, ACT_BS, CLIP, CRITIC_BS, CRITIC_NETS, DISTS, DONE_PATTERNS, ENT,
                                        GAE_ES, GAE_TS, MASKED_CASES, PPO_CASES, SAC_NETS, SAC_SHAPES, VF, a2c_inputs,
                                        act_inputs, critic_inputs, gae_inputs, make_mask, ppo_inputs, sac_inputs)

pytestmark = pytest.mark.gpu

MARGINS = {}                     # case id -> worst error / bound per output, kept for reporting


@pytest.fixture(scope="module")
def cu():
    from sheeprl_b200.lib import CudaOps

    yield CudaOps("cuda")
    path = os.environ.get("MF_LOSS_PRECISION_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(MARGINS, f, indent=1, sort_keys=True)


class NanGuarded(Guarded):
    """Guarded with NaN in every element outside the view: a stray read shows in the outputs, a stray write here"""

    def __init__(self, M, C, ld=None, fill=None):
        super().__init__(M, C, ld or C, fill=fill if fill is not None else torch.full((M, C), math.nan, device="cuda"))
        self.buf[~self.mask] = math.nan

    def outside_untouched(self):
        return bool(self.buf[~self.mask].isnan().all())


def vec(n, fill=None):
    return NanGuarded(1, n, fill=None if fill is None else fill.reshape(1, n))


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def twice(run):
    first, again = run(), run()
    for k in first:
        assert same_bits(first[k], again[k]), f"{k}: rerun is not bit-identical"
    return first


def checked(outs, ins, pristine):
    for b in outs + ins:
        assert b.outside_untouched(), "write outside a view"
    for b, p in zip(ins, pristine):
        assert torch.equal(b.view.reshape(p.shape), p), "an input was written"


def record(case, m):
    MARGINS[case] = m
    assert max(m.values()) <= 1.0, m


def guard_inputs(*ts):
    """inputs copied into NaN-guarded buffers: (guarded buffers, their views, pristine copies)"""
    gs = [NanGuarded(t.shape[0], t[0].numel(), fill=t.reshape(t.shape[0], -1)) if t.dim() > 1 else vec(t.numel(), t)
          for t in ts]
    views = [g.view if t.dim() > 1 else g.view[0] for g, t in zip(gs, ts)]
    return gs, views, [t.clone() for t in ts]


# ------------------------------------------------------------------------------------------------------------ PPO
def run_ppo(cu, inp, dims, mode, clip_v, norm, mask=None):
    B, W = inp[0].shape
    t_in = list(inp) + ([mask] if mask is not None else [])
    gs, v, pristine = guard_inputs(*t_in)

    def run():
        dh, dv, ls = NanGuarded(B, W), vec(B), vec(3)
        args = (dh.view, dv.view[0], ls.view[0], dims, mode, clip_v, norm, R.f32(CLIP), R.f32(VF), R.f32(ENT))
        if mask is None:
            cu.ppo_loss(*v, *args)
        else:
            cu.ppo_loss_masked(*v[:7], v[7], *args)
        checked([dh, dv, ls], gs, pristine)
        return {"dhead": dh.view.clone(), "dvalues": dv.view[0].clone(), "losses": ls.view[0].clone()}

    return twice(run)


@pytest.mark.parametrize("case", list(PPO_CASES))
def test_ppo_loss_precision(cu, case):
    B, dist, afam, clip_v, norm = PPO_CASES[case]
    mode, dims = DISTS[dist]
    inp = ppo_inputs(B, dist, afam, seed=len(case) + B, device="cuda")
    out = run_ppo(cu, inp, dims, mode, clip_v, norm)
    ref, bd = R.ppo_loss(*inp, dims, mode, clip_v, norm, CLIP, VF, ENT)
    ref.pop("ambiguous")
    record(f"ppo_{case}", worst(out, ref, bd))


@pytest.mark.parametrize("case", list(MASKED_CASES))
def test_ppo_loss_masked_precision(cu, case):
    """normalisation over the kept rows when more than one is kept; no kept row: zero losses and gradients"""
    B, mk, dist, clip_v, afam = MASKED_CASES[case]
    mode, dims = DISTS[dist]
    inp = ppo_inputs(B, dist, afam, seed=len(case) + B, device="cuda")
    mask = make_mask(B, mk, gen(B, "cuda"), "cuda")
    out = run_ppo(cu, inp, dims, mode, clip_v, True, mask)
    if mk == "none":
        assert all(bool((o == 0).all()) for o in out.values()), out
    ref, bd = R.ppo_loss(*inp, dims, mode, clip_v, True, CLIP, VF, ENT, mask=mask)
    ref.pop("ambiguous")
    record(f"ppo_masked_{case}", worst(out, ref, bd))


# ------------------------------------------------------------------------------------------------------------ A2C
@pytest.mark.parametrize("case", list(A2C_CASES))
def test_a2c_loss_precision(cu, case):
    N, seg, dist, norm, red_sum = A2C_CASES[case]
    mode, dims = DISTS[dist]
    inp = a2c_inputs(N, dist, seed=len(case), device="cuda")
    W = inp[0].shape[1]
    n_seg = (N + seg - 1) // seg
    gs, v, pristine = guard_inputs(*inp)

    def run():
        dh, dv, ls = NanGuarded(N, W), vec(N), NanGuarded(n_seg, 3)
        cu.a2c_loss(*v, dh.view, dv.view[0], ls.view, seg, dims, mode, norm, red_sum, R.f32(VF), R.f32(ENT))
        checked([dh, dv, ls], gs, pristine)
        return {"dhead": dh.view.clone(), "dvalues": dv.view[0].clone(), "losses": ls.view.clone()}

    out = twice(run)
    ref, bd = R.a2c_loss(*inp, seg, dims, mode, norm, red_sum, VF, ENT)
    record(f"a2c_{case}", worst(out, ref, bd))


# ------------------------------------------------------------------------------------------------------------ ppo_act
ACT_DISTS = (("cat3x3x2", 0), ("cat8heads", 0), ("cat128", 0), ("normal6", 1), ("tanh6", 2), ("tanh33", 3))


@pytest.mark.parametrize("greedy", [False, True], ids=["sample", "greedy"])
@pytest.mark.parametrize("dist,mode", ACT_DISTS)
@pytest.mark.parametrize("B", ACT_BS)
def test_ppo_act_precision(cu, B, dist, mode, greedy):
    dims = DISTS[dist][1]
    head, noise = act_inputs(B, dist, seed=B + mode, device="cuda")
    W = sum(dims)
    gs, v, pristine = guard_inputs(head, noise)

    def run():
        a, lp = NanGuarded(B, W), vec(B)
        cu.ppo_act(v[0], v[1], a.view, lp.view[0], dims, mode, greedy)
        checked([a, lp], gs, pristine)
        return {"actions": a.view.clone(), "logp": lp.view[0].clone()}

    out = twice(run)
    ref, bd = R.ppo_act(head, noise, dims, mode, greedy)
    if mode == 0:
        bad = (out["actions"] != ref["actions"].float()).any(-1)
        assert not bool(bad.any()), f"{int(bad.sum())} rows differ from fp32 torch's argmax, first {bad.nonzero()[:4]}"
        out.pop("actions")
        ref.pop("actions")
    record(f"act_B{B}_{dist}_m{mode}_{'greedy' if greedy else 'sample'}", worst(out, ref, bd))


# ------------------------------------------------------------------------------------------------------------ SAC
def _sac_case_list():
    return [(A, B, SAC_NETS[i % 3]) for i, (A, B) in enumerate(SAC_SHAPES)]


@pytest.mark.parametrize("A,B,nets", _sac_case_list(), ids=lambda v: str(v))
def test_sac_sample_precision(cu, A, B, nets):
    """sac_sample_fwd into an action view with ld_action = A + 3 (the critics' input columns), then sac_sample_bwd
    from dact [nets, stride_net] with stride_net = B A + 5 (NaN between the critics), on the forward's own tanh"""
    head, eps, scale, bias, dact = sac_inputs(B, A, nets, seed=A * 7 + B + nets, device="cuda")
    la = torch.tensor([-1.3], device="cuda")
    stride = B * A + 5
    dg = NanGuarded(nets, B * A, stride, fill=dact.reshape(nets, B * A))
    gs, v, pristine = guard_inputs(head, eps, scale, bias, la)
    from sheeprl_b200.lib import _p

    def run():
        act, lp, y, dh = NanGuarded(B, A, A + 3), vec(B), NanGuarded(B, A), NanGuarded(B, 2 * A)
        cu.sac_sample_fwd(v[0], v[1], v[2], v[3], act.view, lp.view[0], y.view)
        cu._ck(cu.lib.b200rl_sac_sample_bwd(_p(v[0]), _p(v[1]), _p(y.view), _p(v[2]), _p(dg.view), stride, nets,
                                            _p(v[4]), _p(dh.view), B, A, cu._st()))
        checked([act, lp, y, dh, dg], gs, pristine)
        return {"action": act.view.clone(), "logp": lp.view[0].clone(), "tanh": y.view.clone(),
                "dhead": dh.view.clone()}

    out = twice(run)
    m = {}
    for a, b in [(a, min(B, a + (1 << 20) // A)) for a in range(0, B, (1 << 20) // A)]:
        ref, bd = R.sac_sample_fwd(head[a:b], eps[a:b], scale, bias)
        r2, b2 = R.sac_sample_bwd(head[a:b], eps[a:b], scale, dact[:, a:b], la, batch=B)
        ref.update(r2)
        bd.update(b2)
        for k, val in worst({k: o[a:b] for k, o in out.items()}, ref, bd).items():
            m[k] = max(m.get(k, 0.0), val)
    if B >= 4096:
        raw = head[:, A:]
        assert bool((raw < -5).any() and (raw > 2).any() and (raw == -5).any()), "log-std families missing"
    record(f"sac_sample_A{A}_B{B}_n{nets}", m)


def _critic_case_list():
    return [(B, nets, (-10.0, 0.0, 2.0)[i % 3]) for i, (B, nets) in enumerate((B, n) for B in CRITIC_BS
                                                                             for n in CRITIC_NETS)]


@pytest.mark.parametrize("B,nets,log_alpha", _critic_case_list(), ids=lambda v: str(v))
def test_sac_losses_precision(cu, B, nets, log_alpha):
    """sac_target, sac_critic_loss, sac_actor_loss and droq_actor_loss on [nets, stride_net] with stride_net = B + 3"""
    q, logp, rew, term = critic_inputs(B, nets, seed=B + nets, device="cuda")
    la = torch.tensor([log_alpha], device="cuda")
    stride = B + 3
    qg = NanGuarded(nets, B, stride, fill=q)
    gs, v, pristine = guard_inputs(logp, rew, term, la)
    pristine_q = q.clone()
    from sheeprl_b200.lib import _p

    def run():
        y = vec(B)
        cu._ck(cu.lib.b200rl_sac_target(_p(qg.view), stride, nets, _p(v[0]), _p(v[1]), _p(v[2]), _p(v[3]),
                                        R.f32(0.99), _p(y.view[0]), B, cu._st()))
        dqc, lc = NanGuarded(nets, B, stride), vec(1)
        cu._ck(cu.lib.b200rl_sac_critic_loss(_p(qg.view), stride, nets, _p(y.view[0]), _p(dqc.view), _p(lc.view[0]),
                                             B, cu._st()))
        res = {"y": y.view[0].clone(), "critic_loss": lc.view[0].clone(), "dq_critic": dqc.view.clone()}
        outs = [y, dqc, lc]
        for tag, fn in (("sac", cu.lib.b200rl_sac_actor_loss), ("droq", cu.lib.b200rl_droq_actor_loss)):
            dq, al, alp, dla = NanGuarded(nets, B, stride), vec(1), vec(1), vec(1)
            cu._ck(fn(_p(qg.view), stride, nets, _p(v[0]), _p(v[3]), R.f32(-3.0), _p(dq.view), _p(al.view[0]),
                      _p(alp.view[0]), _p(dla.view[0]), B, cu._st()))
            outs += [dq, al, alp, dla]
            res.update({f"{tag}_dq": dq.view.clone(), f"{tag}_actor_loss": al.view[0].clone(),
                        f"{tag}_alpha_loss": alp.view[0].clone(), f"{tag}_dlog_alpha": dla.view[0].clone()})
        checked(outs + [qg], gs, pristine)
        assert torch.equal(qg.view, pristine_q), "q was written"
        return res

    out = twice(run)
    ref, bd = R.sac_target(q, logp, rew, term, la, 0.99)
    m = worst({"y": out["y"]}, ref, bd)
    ref, bd = R.sac_critic_loss(q, out["y"])
    m.update(worst({"loss": out["critic_loss"], "dq": out["dq_critic"]}, ref, bd))
    for tag, mean_over in (("sac", False), ("droq", True)):
        ref, bd = R.sac_actor_loss(q, logp, la, -3.0, mean_over)
        got = {k: out[f"{tag}_{k}"] for k in ("actor_loss", "alpha_loss", "dlog_alpha", "dq")}
        m.update({f"{tag}_{k}": val for k, val in worst(got, ref, bd).items()})
    record(f"critics_B{B}_n{nets}_la{log_alpha}", m)


# ------------------------------------------------------------------------------------------------------------ GAE
@pytest.mark.parametrize("T,E,pattern", [(T, E, DONE_PATTERNS[i % 4]) for i, (T, E) in
                                         enumerate((T, E) for T in GAE_TS for E in GAE_ES)], ids=lambda v: str(v))
def test_gae_precision(cu, T, E, pattern):
    r, v_, d, nv = gae_inputs(T, E, pattern, seed=T + E, device="cuda")
    gs, v, pristine = guard_inputs(r, v_, d, nv)

    def run():
        ret, adv = NanGuarded(T, E), NanGuarded(T, E)
        cu.gae(v[0], v[1], v[2], v[3], R.f32(0.99), R.f32(0.95), ret.view, adv.view)
        checked([ret, adv], gs, pristine)
        return {"returns": ret.view.clone(), "advantages": adv.view.clone()}

    out = twice(run)
    ref, bd = R.gae(r, v_, d, nv, 0.99, 0.95)
    record(f"gae_T{T}_E{E}_{pattern}", worst(out, ref, bd))
