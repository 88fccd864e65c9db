"""The float64 reference of the model-free objective and sampling kernels (oracle/mf_loss_ref.py) and its error bounds,
on the CPU.

  - the reference is the reference's semantics: it reproduces a fixture made by running the reference's own
    policy_loss / value_loss / entropy_loss / normalize_tensor, PPOAgent's distribution code, SACActor, the SAC losses
    and `gae` in float64 with autograd (oracle/make_golden_mf_loss_ref.py -> tests/golden/mf_loss_ref.pt), and re-runs
    the comparison live when the reference package is importable;
  - the fp32 emulators (the kernels' executable specification, used by the engine tests) stay within half of every
    bound on the GPU cases that fit on the CPU (the cases of tests/test_gpu_mf_loss_precision.py are defined here);
  - fp32 implementations with one plausible defect each exceed the bound by at least 4x.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import mf_loss_ref as R
from oracle.ops_emul import EmulOps
from oracle.ops_emul_a2c import A2CEmulOps
from oracle.ops_emul_droq import DroQEmulOps
from oracle.ops_emul_recurrent import RecurrentEmulOps
from tests.test_loss_ref_cpu import gen, worst

GOLDEN = "tests/golden/mf_loss_ref.pt"
CLIP, VF, ENT = 0.2, 0.5, 0.01

# ------------------------------------------------------------------------------------------------------------ inputs
DISTS = {"cat2": (0, (2,)), "cat18": (0, (18,)), "cat3x3x2": (0, (3, 3, 2)), "cat8heads": (0, (2, 3, 4, 5, 2, 3, 4, 5)),
         "cat128": (0, (128,)), "normal1": (1, (1,)), "normal6": (1, (6,)), "normal32": (1, (32,)),
         "normal33": (1, (33,)), "tanh1": (2, (1,)), "tanh6": (2, (6,)), "tanh32": (2, (32,)), "tanh33": (2, (33,))}
ADV_FAMILIES = ("normal", "offset", "near_const", "heavy")


def adv_inputs(n, fam, g, device="cpu"):
    """N(0, 1); offset 1e3 + N(0, 1); near-constant 0.5 + 1e-4 N(0, 1) (its std is comparable to sqrt(eps) = 1e-4);
    heavy-tailed N(0, 1) exp(1.5 N(0, 1))"""
    z = torch.randn(n, generator=g, device=device)
    if fam == "normal":
        return z
    if fam == "offset":
        return 1e3 + z
    if fam == "near_const":
        return 0.5 + 1e-4 * z
    assert fam == "heavy", fam
    return z * torch.exp(1.5 * torch.randn(n, generator=g, device=device))


def head_actions(B, mode, dims, g, device="cpu"):
    """discrete: logits N(0, 2) and one-hot actions drawn from them; Normal: mean N(0, 1), log-std U(-20, 5), the
    action an fp32 draw mean + std e; tanh_normal: log-std U(-5, 2) (atanh of an fp32 tanh is conditioned by
    |x| u / std), the stored action fp32 tanh of a draw, with a tenth of the entries at exactly +-1 and a tenth in the
    clamp band (1 - 1e-6, 1), their means drawn so that the clamped atanh is a draw of the head.  An action a thousand
    std from its mean has a log-prob of -5e5 whose fp32 rounding alone moves the ratio by tens of percent: no fp32
    kernel, and no first-order bound, says anything useful there."""
    if mode == 0:
        head = 2 * torch.randn(B, sum(dims), generator=g, device=device)
        acts, o = [], 0
        for K in dims:
            idx = torch.multinomial(torch.softmax(head[:, o:o + K], -1), 1, generator=g).reshape(-1)
            acts.append(F.one_hot(idx, K).float())
            o += K
        return head, torch.cat(acts, -1)
    A = dims[0]
    mu = torch.randn(B, A, generator=g, device=device)
    lo, hi = (-20.0, 5.0) if mode == 1 else (-5.0, 2.0)
    ls = lo + (hi - lo) * torch.rand(B, A, generator=g, device=device)
    x = (mu.double() + ls.double().exp() * torch.randn(B, A, generator=g, device=device, dtype=torch.float64))
    if mode == 1:
        return torch.cat((mu, ls), -1), x.float()
    a = x.tanh().float()
    pick = torch.rand(B, A, generator=g, device=device)
    sgn = torch.where(torch.rand(B, A, generator=g, device=device) < 0.5, -1.0, 1.0)
    band = 1.0 - 1e-6 * torch.rand(B, A, generator=g, device=device)
    a = torch.where(pick < 0.1, sgn, torch.where(pick < 0.2, sgn * band, a))
    # the saturated entries are draws of their own head: the mean sits a few std inside the clamped atanh
    xs = a.double().clamp(-R.SAFE_LIM, R.SAFE_LIM).atanh()
    mu_s = (xs - ls.double().exp() * torch.randn(B, A, generator=g, device=device, dtype=torch.float64)).float()
    mu = torch.where(pick < 0.2, mu_s, mu)
    return torch.cat((mu, ls), -1), a


def ratio_targets(B, clip, g, device="cpu"):
    """per row: near 1 (half the rows), far outside the clip on either side, or at fp32(1 -+ clip) moved by -2..2 ulp"""
    lo, hi = R.f32(1.0 - R.f32(clip)), R.f32(1.0 + R.f32(clip))
    near = torch.exp(0.05 * torch.randn(B, generator=g, device=device))
    far = torch.where(torch.rand(B, generator=g, device=device) < 0.5, 0.3, 3.0)
    edge = torch.where(torch.rand(B, generator=g, device=device) < 0.5, lo, hi)
    k = torch.randint(-2, 3, (B,), generator=g, device=device).float()
    edge = edge * (1 + k * 2.0 ** -23)
    pick = torch.rand(B, generator=g, device=device)
    return torch.where(pick < 0.5, near, torch.where(pick < 0.75, far, edge))


def value_inputs(B, clip, g, device="cpu"):
    """(values, old_values, returns): val - old inside the clip, outside it, or exactly +-clip in fp32 (old a multiple
    of 2^-26 in [-0.24, 0.04] and val = old + clip, both exact), a third each"""
    c = R.f32(clip)
    old = torch.randn(B, generator=g, device=device)
    val = old + 0.5 * c * torch.randn(B, generator=g, device=device)
    out = old + 3 * c * torch.sign(torch.randn(B, generator=g, device=device))
    o_edge = torch.round((-0.24 + 0.28 * torch.rand(B, generator=g, device=device)) * 2 ** 26) / 2 ** 26
    sgn = torch.where(torch.rand(B, generator=g, device=device) < 0.5, -1.0, 1.0)
    o_edge = o_edge * sgn                                     # -clip rows: old in [-0.04, 0.24]
    v_edge = o_edge + sgn * c
    pick = torch.rand(B, generator=g, device=device)
    vals = torch.where(pick < 1 / 3, val, torch.where(pick < 2 / 3, out, v_edge))
    olds = torch.where(pick < 2 / 3, old, o_edge)
    ret = vals + torch.randn(B, generator=g, device=device)
    return vals, olds, ret


def ppo_inputs(B, dist, afam, seed, device="cpu", clip=CLIP):
    mode, dims = DISTS[dist]
    g = gen(seed, device)
    head, acts = head_actions(B, mode, dims, g, device)
    lp32, _ = R._lpe32(head, acts, dims, mode)
    old = lp32 - torch.log(ratio_targets(B, clip, g, device))
    adv = adv_inputs(B, afam, g, device)
    val, oldv, ret = value_inputs(B, clip, g, device)
    return head.contiguous(), acts.contiguous(), old, adv, val, oldv, ret


# ------------------------------------------------------------------------------------------------------------ cases
PPO_BS = (2, 31, 32, 33, 255, 256, 257, 1000, 4096, 65536)


def _ppo_cases():
    out, k = {}, 0
    for B in PPO_BS:
        for dist in DISTS:
            clip_v, norm = (k % 2 == 0), (k // 2) % 2 == 0
            afam = ADV_FAMILIES[(k + k // 4) % 4]
            out[f"B{B}_{dist}_{afam}{'_vclip' if clip_v else ''}{'_norm' if norm else ''}"] = (B, dist, afam, clip_v,
                                                                                               norm)
            k += 1
    return out


PPO_CASES = _ppo_cases()
MASKS = ("none", "one", "two", "k33", "all", "prefix", "random", "last")


def make_mask(B, kind, g, device="cpu"):
    """kept rows: none, one (the first), two, 33 (or all when fewer), all, a prefix (sequence padding), a random
    subset, only the last row"""
    m = torch.zeros(B, device=device)
    if kind == "one":
        m[0] = 1
    elif kind == "two":
        m[torch.randperm(B, generator=g, device=device)[:2]] = 1
    elif kind == "k33":
        m[torch.randperm(B, generator=g, device=device)[:33]] = 1
    elif kind == "all":
        m[:] = 1
    elif kind == "prefix":
        m[: max(1, (2 * B) // 3)] = 1
    elif kind == "random":
        m = (torch.rand(B, generator=g, device=device) < 0.5).float()
        m[0] = 1
    elif kind == "last":
        m[-1] = 1
    return m


def _masked_cases():
    out, k = {}, 0
    for B in PPO_BS:
        for mk in MASKS:
            if mk == "two" and B < 2:
                continue
            dist = list(DISTS)[k % len(DISTS)]
            out[f"B{B}_{mk}_{dist}"] = (B, mk, dist, k % 2 == 0, ADV_FAMILIES[k % 4])
            k += 1
    return out


MASKED_CASES = _masked_cases()
A2C_CASES = {}
for _i, (_N, _seg, _norm) in enumerate(((1, 1, False), (2, 2, True), (2, 1, False), (257, 257, True), (257, 255, True),
                                        (257, 1, False), (65536, 4096, True), (65536, 65534, True), (65536, 1, False))):
    for _red in ("mean", "sum"):
        _dist = ("cat3x3x2", "normal6", "tanh6", "cat18", "cat128")[(_i + (_red == "sum")) % 5]
        A2C_CASES[f"N{_N}_seg{_seg}_{_dist}_{_red}{'_norm' if _norm else ''}"] = (_N, _seg, _dist, _norm, _red == "sum")
ACT_BS = (1, 127, 128, 129, 65537)
SAC_SHAPES = [(A, B) for A in (1, 6, 31, 32, 33, 64) for B in (1, 7, 8, 9, 4096, 1 << 18) if A * B <= 1 << 22]
SAC_NETS = (1, 2, 10)
CRITIC_BS = (1, 255, 256, 257, 4096, 65536)
CRITIC_NETS = (1, 2, 5, 10)
GAE_TS = (1, 15, 16, 17, 1024)
GAE_ES = (1, 255, 256, 257)
DONE_PATTERNS = ("none", "all", "alternating", "first_last")


def act_inputs(B, dist, seed, device="cpu"):
    """heads and Exp(1) noise; discrete: every fourth row has two equal top logits with equal noise (an exact tie) or
    noise 1e-5 apart in relative terms (a near tie); continuous: log-std U(-5, 2), means up to +-12 so that tanh
    saturates"""
    mode, dims = DISTS[dist]
    g = gen(seed, device)
    if mode == 0:
        W = sum(dims)
        head = 2 * torch.randn(B, W, generator=g, device=device)
        noise = torch.empty(B, W, device=device).exponential_(generator=g)
        o = 0
        for K in dims:
            tie = torch.arange(B, device=device) % 4 == 0
            near = torch.arange(B, device=device) % 4 == 1
            hd, nz = head[:, o:o + K], noise[:, o:o + K]
            if K >= 2:
                hd[:, 1] = torch.where(tie | near, hd[:, 0], hd[:, 1])
                nz[:, 1] = torch.where(tie, nz[:, 0], torch.where(near, nz[:, 0] * (1 + 1e-5), nz[:, 1]))
            o += K
        return head, noise
    A = dims[0]
    mu = 4 * torch.randn(B, A, generator=g, device=device)
    ls = -5 + 7 * torch.rand(B, A, generator=g, device=device)
    return torch.cat((mu, ls), -1), torch.randn(B, A, generator=g, device=device)


def sac_inputs(B, A, nets, seed, device="cpu"):
    """head [mean | log-std]: log-std in [-8, 4] with a tenth of the entries exactly at -5 or 2, means N(0, 3) with a
    tenth at +-12 (|x_t| >= 9: tanh saturates); scale != 1, bias != 0; dact [nets, B, A]"""
    g = gen(seed, device)
    mean = 3 * torch.randn(B, A, generator=g, device=device)
    pick = torch.rand(B, A, generator=g, device=device)
    mean = torch.where(pick < 0.1, 12 * torch.sign(mean), mean)
    ls = -8 + 12 * torch.rand(B, A, generator=g, device=device)
    pk = torch.rand(B, A, generator=g, device=device)
    ls = torch.where(pk < 0.05, -5.0, torch.where(pk < 0.1, 2.0, ls))
    eps = torch.randn(B, A, generator=g, device=device)
    scale = 0.5 + 2 * torch.rand(A, generator=g, device=device)
    bias = torch.randn(A, generator=g, device=device)
    dact = torch.randn(nets, B, A, generator=g, device=device)
    return torch.cat((mean, ls), -1).contiguous(), eps, scale, bias, dact


def critic_inputs(B, nets, seed, device="cpu"):
    """q [nets, B] with a quarter of the rows tied between two critics at the minimum, logp, rewards, a third of the
    rows terminated"""
    g = gen(seed, device)
    q = 5 * torch.randn(nets, B, generator=g, device=device)
    if nets > 1:
        tie = torch.arange(B, device=device) % 4 == 0
        m = q.min(0).values
        q[0] = torch.where(tie, m, q[0])
        q[nets - 1] = torch.where(tie, m, q[nets - 1])
    logp = 3 * torch.randn(B, generator=g, device=device)
    rew = torch.randn(B, generator=g, device=device)
    term = (torch.rand(B, generator=g, device=device) < 1 / 3).float()
    return q.contiguous(), logp, rew, term


def gae_inputs(T, E, pattern, seed, device="cpu"):
    g = gen(seed, device)
    r, v = torch.randn(T, E, generator=g, device=device), 3 * torch.randn(T, E, generator=g, device=device)
    nv = 3 * torch.randn(1, E, generator=g, device=device)
    d = torch.zeros(T, E, device=device)
    if pattern == "all":
        d[:] = 1
    elif pattern == "alternating":
        d[(torch.arange(T, device=device) % 2 == 1)] = 1
    elif pattern == "first_last":
        d[0] = 1
        d[-1] = 1
    return r, v, d, nv


# ------------------------------------------------------------------------------------------------------------ emulators
em, rem, aem, dem = EmulOps(), RecurrentEmulOps(), A2CEmulOps(), DroQEmulOps()


def emul_ppo(inp, dims, mode, clip_v, norm, mask=None, ops=None):
    head, acts, old, adv, val, oldv, ret = inp
    B, W = head.shape
    dh, dv, ls = torch.empty(B, W), torch.empty(B), torch.empty(3)
    if mask is None:
        (ops or em).ppo_loss(head, acts, old, adv, val, oldv, ret, dh, dv, ls, dims, mode, clip_v, norm, R.f32(CLIP),
                             R.f32(VF), R.f32(ENT))
    else:
        rem.ppo_loss_masked(head, acts, old, adv, val, oldv, ret, mask, dh, dv, ls, dims, mode, clip_v, norm,
                            R.f32(CLIP), R.f32(VF), R.f32(ENT))
    return {"dhead": dh, "dvalues": dv, "losses": ls}


def ref_ppo(inp, dims, mode, clip_v, norm, mask=None):
    ref, bd = R.ppo_loss(*inp, dims, mode, clip_v, norm, CLIP, VF, ENT, mask=mask)
    ref.pop("ambiguous")
    return ref, bd


CPU_PPO = [c for c, (B, *_) in PPO_CASES.items() if B <= 4096]


@pytest.mark.parametrize("case", CPU_PPO)
def test_emulator_ppo_loss_within_bounds(case):
    B, dist, afam, clip_v, norm = PPO_CASES[case]
    mode, dims = DISTS[dist]
    inp = ppo_inputs(B, dist, afam, seed=len(case) + B)
    ref, bd = ref_ppo(inp, dims, mode, clip_v, norm)
    m = worst(emul_ppo(inp, dims, mode, clip_v, norm), ref, bd)
    assert max(m.values()) <= 0.5, m


@pytest.mark.parametrize("case", [c for c, (B, *_) in MASKED_CASES.items() if B <= 4096])
def test_emulator_ppo_loss_masked_within_bounds(case):
    B, mk, dist, clip_v, afam = MASKED_CASES[case]
    mode, dims = DISTS[dist]
    inp = ppo_inputs(B, dist, afam, seed=len(case) + B)
    mask = make_mask(B, mk, gen(B))
    ref, bd = ref_ppo(inp, dims, mode, clip_v, True, mask)
    m = worst(emul_ppo(inp, dims, mode, clip_v, True, mask), ref, bd)
    assert max(m.values()) <= 0.5, m


def emul_a2c(inp, seg, dims, mode, norm, red_sum, ops=None):
    head, acts, adv, val, ret = inp
    N, W = head.shape
    dh, dv, ls = torch.empty(N, W), torch.empty(N), torch.empty((N + seg - 1) // seg, 3)
    (ops or aem).a2c_loss(head, acts, adv, val, ret, dh, dv, ls, seg, dims, mode, norm, red_sum, R.f32(VF), R.f32(ENT))
    return {"dhead": dh, "dvalues": dv, "losses": ls}


def a2c_inputs(N, dist, seed, device="cpu"):
    head, acts, _, adv, val, _, ret = ppo_inputs(N, dist, "normal", seed, device)
    return head, acts, adv, val, ret


@pytest.mark.parametrize("case", [c for c, (N, *_) in A2C_CASES.items() if N <= 257])
def test_emulator_a2c_loss_within_bounds(case):
    N, seg, dist, norm, red_sum = A2C_CASES[case]
    mode, dims = DISTS[dist]
    inp = a2c_inputs(N, dist, seed=len(case))
    ref, bd = R.a2c_loss(*inp, seg, dims, mode, norm, red_sum, VF, ENT)
    m = worst(emul_a2c(inp, seg, dims, mode, norm, red_sum), ref, bd)
    assert max(m.values()) <= 0.5, m


@pytest.mark.parametrize("greedy", [False, True])
@pytest.mark.parametrize("dist,mode", [("cat3x3x2", 0), ("cat128", 0), ("normal6", 1), ("tanh6", 2), ("tanh33", 3)])
def test_emulator_ppo_act_within_bounds(dist, mode, greedy):
    B = 1000
    dims = DISTS[dist][1]
    head, noise = act_inputs(B, dist, seed=B + mode)
    W = sum(dims)
    acts, lp = torch.empty(B, W), torch.empty(B)
    em.ppo_act(head, noise, acts, lp, dims, mode, greedy)
    ref, bd = R.ppo_act(head, noise, dims, mode, greedy)
    if mode == 0:
        assert torch.equal(acts, ref["actions"].float())
        m = worst({"logp": lp}, {"logp": ref["logp"]}, bd)
    else:
        m = worst({"logp": lp, "actions": acts}, ref, bd)
    assert max(m.values()) <= 0.5, m


@pytest.mark.parametrize("nets", SAC_NETS)
@pytest.mark.parametrize("A", (1, 6, 33, 64))
def test_emulator_sac_sample_within_bounds(A, nets):
    B = 999
    head, eps, scale, bias, dact = sac_inputs(B, A, nets, seed=A * 10 + nets)
    act, lp, y, dh = torch.empty(B, A), torch.empty(B), torch.empty(B, A), torch.empty(B, 2 * A)
    la = torch.tensor([-1.3])
    em.sac_sample_fwd(head, eps, scale, bias, act, lp, y)
    em.sac_sample_bwd(head, eps, y, scale, dact, la, dh)
    ref, bd = R.sac_sample_fwd(head, eps, scale, bias)
    m = worst({"action": act, "logp": lp, "tanh": y}, ref, bd)
    ref, bd = R.sac_sample_bwd(head, eps, scale, dact, la)
    m.update(worst({"dhead": dh}, ref, bd))
    assert max(m.values()) <= 0.5, m


@pytest.mark.parametrize("log_alpha", [-10.0, 0.0, 2.0])
@pytest.mark.parametrize("nets", CRITIC_NETS)
def test_emulator_sac_losses_within_bounds(nets, log_alpha):
    B = 4096
    q, logp, rew, term = critic_inputs(B, nets, seed=nets)
    la = torch.tensor([log_alpha])
    y = torch.empty(B)
    em.sac_target(q, logp, rew, term, la, R.f32(0.99), y)
    ref, bd = R.sac_target(q, logp, rew, term, la, 0.99)
    m = worst({"y": y}, ref, bd)
    dq, lo = torch.empty(nets, B), torch.empty(1)
    em.sac_critic_loss(q, y, dq, lo)
    ref, bd = R.sac_critic_loss(q, y)
    m.update(worst({"loss": lo, "dq": dq}, ref, bd))
    for mean_over, ops in ((False, em), (True, dem)):
        out = {k: torch.empty(1) for k in ("actor_loss", "alpha_loss", "dlog_alpha")}
        out["dq"] = torch.empty(nets, B)
        fn = ops.droq_actor_loss if mean_over else ops.sac_actor_loss
        fn(q, logp, la, R.f32(-3.0), out["dq"], out["actor_loss"], out["alpha_loss"], out["dlog_alpha"])
        ref, bd = R.sac_actor_loss(q, logp, la, -3.0, mean_over)
        m.update({f"{'droq' if mean_over else 'sac'}_{k}": v for k, v in worst(out, ref, bd).items()})
    assert max(m.values()) <= 0.5, m


def fp32_gae(r, v, d, nv, gamma, lmbda, textbook=False):
    """utils.gae in fp32; textbook: mask step t's bootstrap with dones[t + 1] (the last step keeps dones[-1])"""
    T = r.shape[0]
    adv = torch.zeros_like(r)
    last = torch.zeros_like(nv[0])
    for t in reversed(range(T)):
        nd = d[t + 1] if (textbook and t < T - 1) else d[t]
        nnt = 1.0 - nd
        nxt = nv[0] if t == T - 1 else v[t + 1]
        delta = r[t] + nxt * nnt * gamma - v[t]
        last = delta + nnt * last * gamma * lmbda
        adv[t] = last
    return {"returns": adv + v, "advantages": adv}


@pytest.mark.parametrize("pattern", DONE_PATTERNS)
@pytest.mark.parametrize("T", GAE_TS)
def test_fp32_gae_within_bounds(T, pattern):
    """no emulator method: the fp32 loop of utils.gae stands in for the kernel's specification"""
    r, v, d, nv = gae_inputs(T, 257, pattern, seed=T)
    g, lm = R.f32(0.99), R.f32(0.95)
    ref, bd = R.gae(r, v, d, nv, g, lm)
    m = worst(fp32_gae(r, v, d, nv, g, lm), ref, bd)
    assert max(m.values()) <= 0.5, m


# ------------------------------------------------------------------------------------------------------------ fixture
def reference_outputs(name, a):
    """mf_loss_ref's outputs for one fixture entry, keyed like the fixture"""
    if name.startswith("ppo"):
        o, _ = R.ppo_loss(a["head"], a["actions"], a["old_logp"], a["adv"], a["values"], a["old_values"],
                          a["returns"], a["dims"], a["mode"], a["clip_vloss"], a["normalize"], a["clip"], a["vf"],
                          a["ent"], mask=a.get("mask"))
        return o
    if name == "normalize":
        return {"adv": R.normalize64(a["x"])[0]}
    if name == "sac_sample":
        o, _ = R.sac_sample_fwd(a["head"], a["eps"], a["scale"], a["bias"])
        o2, _ = R.sac_sample_bwd(a["head"], a["eps"], a["scale"], a["dact"], a["log_alpha"])
        return {"action": o["action"], "logp": o["logp"], "dhead": o2["dhead"]}
    if name == "sac_target":
        return R.sac_target(a["q"], a["logp"], a["rewards"], a["terminated"], a["log_alpha"], a["gamma"])[0]
    if name == "sac_losses":
        o, _ = R.sac_critic_loss(a["q"], a["y"])
        o2, _ = R.sac_actor_loss(a["q"], a["logp"], a["log_alpha"], a["target_entropy"], False)
        return {"critic_loss": o["loss"], "dq_critic": o["dq"], "actor_loss": o2["actor_loss"],
                "dq_actor": o2["dq"], "alpha_loss": o2["alpha_loss"], "dlog_alpha": o2["dlog_alpha"]}
    assert name == "gae", name
    return R.gae(a["rewards"], a["values"], a["dones"], a["next_value"], a["gamma"], a["lmbda"])[0]


def _compare_fixture(fx):
    errs = {}
    for name, case in fx.items():
        got = reference_outputs(name, case["args"])
        for k, want in case["out"].items():
            w = want.double()
            err = float((got[k].double().reshape(w.shape) - w).abs().max())
            errs[f"{name}.{k}"] = err / (1.0 + float(w.abs().max()))
    return errs


FIXTURE_TOL = 1e-12


def test_reference_matches_the_committed_fixture():
    errs = _compare_fixture(torch.load(GOLDEN, weights_only=False))
    assert max(errs.values()) <= FIXTURE_TOL, errs


def test_reference_matches_the_reference_live():
    from oracle.ref_harness import reference_available

    if not reference_available():
        pytest.skip("reference package not present")
    from oracle.make_golden_mf_loss_ref import make

    errs = _compare_fixture(make())
    assert max(errs.values()) <= FIXTURE_TOL, errs


def test_all_zero_mask_gives_zeros():
    """ppo_loss_masked with no kept row: the kernel's choice (zero losses and gradients, where torch's mean over no rows
    is NaN) is what the reference returns and what the emulator does"""
    inp = ppo_inputs(33, "cat3x3x2", "normal", seed=3)
    ref, bd = ref_ppo(inp, (3, 3, 2), 0, True, True, torch.zeros(33))
    got = emul_ppo(inp, (3, 3, 2), 0, True, True, torch.zeros(33))
    for k in ref:
        assert bool((ref[k] == 0).all()) and bool((got[k] == 0).all()), k


# ------------------------------------------------------------------------------------------------------------ mutants
def fp32_ppo(inp, dims, mode, clip_v, norm, mutant=None):
    """the PPO objective in fp32 torch with autograd (the emulator's recipe), with one defect switched on"""
    head, acts, old, adv, val, oldv, ret = inp
    B = head.shape[0]
    c, vf, ec = R.f32(CLIP), R.f32(VF), R.f32(ENT)
    h = head.clone().requires_grad_(True)
    v = val.clone().requires_grad_(True)
    if mode == 0 and mutant == "one_lse_over_all_heads":
        lg = torch.log_softmax(h, -1)
        lp, ent = (lg * acts).sum(-1), -(lg.exp() * lg).sum(-1)
    elif mode == 2 and mutant == "tanh_corr_at_atanh":
        mean, ls = h.chunk(2, -1)
        x = torch.atanh(acts.clamp(-R.SAFE_LIM, R.SAFE_LIM))
        corr = 2.0 * (math.log(2.0) - x - F.softplus(-2.0 * x)).sum(-1)
        lp = (-((x - mean) ** 2) / (2 * ls.exp() ** 2) - ls - R.C0).sum(-1) - corr
        ent = (0.5 + R.C0 + ls).sum(-1)
    else:
        lp, ent = R._lpe32(h, acts, dims, mode)
    a = adv
    if norm:
        if mutant == "biased_std":
            a = (a - a.mean()) / (a.std(unbiased=False) + 1e-8)
        elif mutant == "eps_in_sqrt":
            a = (a - a.mean()) / torch.sqrt(a.var() + 1e-8)
        else:
            a = (a - a.mean()) / (a.std() + 1e-8)
    r = (lp - old).exp()
    rc = r.clamp(1 - c, 1 + c)
    if mutant == "grad_through_clipped_branch":
        rc = r + (rc - r).detach()
    pg = -torch.min(a * r, a * rc).mean()
    if clip_v:
        dv = v - oldv
        cl = dv.clamp(-c, c)
        if mutant == "strict_value_clip_mask":
            cl = torch.where(dv.abs() < c, dv, cl.detach())
        vl = 0.5 * torch.max((v - ret) ** 2, (oldv + cl - ret) ** 2).mean()
    else:
        vl = ((v - ret) ** 2).mean()
    el = (-ent).mean()
    gh, gv = torch.autograd.grad(pg + vf * vl + ec * el, [h, v])
    if mutant == "entropy_grad_without_H":                      # -dent p (log p + H) -> -dent p log p
        o = 0
        for K in dims:
            lg = torch.log_softmax(head[:, o:o + K], -1)
            hh = -(lg.exp() * lg).sum(-1, keepdim=True)
            gh[:, o:o + K] += (-ec / B) * lg.exp() * hh
            o += K
    return {"dhead": gh, "dvalues": gv, "losses": torch.stack([pg, vl, el]).detach()}


def _ppo_mutant(mutant):
    B, dist, afam, clip_v = {"grad_through_clipped_branch": (300, "cat18", "normal", False),
                             "biased_std": (31, "normal6", "normal", False),
                             "eps_in_sqrt": (300, "cat18", "near_const", False),
                             "strict_value_clip_mask": (300, "cat3x3x2", "normal", True),
                             "entropy_grad_without_H": (300, "cat18", "normal", False),
                             "one_lse_over_all_heads": (300, "cat3x3x2", "normal", False),
                             "tanh_corr_at_atanh": (300, "tanh6", "normal", False)}[mutant]
    mode, dims = DISTS[dist]
    inp = ppo_inputs(B, dist, afam, seed=21)
    ref, bd = ref_ppo(inp, dims, mode, clip_v, True)
    return worst(fp32_ppo(inp, dims, mode, clip_v, True), ref, bd), \
        worst(fp32_ppo(inp, dims, mode, clip_v, True, mutant), ref, bd)


def _sac_mutant(mutant):
    B, A, nets = 500, 6, 2
    head, eps, scale, bias, dact = sac_inputs(B, A, nets, seed=22)
    la = torch.tensor([0.5])
    y = torch.tanh(head[:, :A] + head[:, A:].clamp(-5, 2).exp() * eps)
    ref, bd = R.sac_sample_bwd(head, eps, scale, dact, la)

    def run(m=None):
        dh = torch.empty(B, 2 * A)
        em.sac_sample_bwd(head, eps, y, scale, dact, la, dh)
        if m is not None:
            raw = head[:, A:]
            std = raw.clamp(-5.0, 2.0).exp()
            dlogp = la.exp() / B
            om = 1 - y * y
            den = scale * om if m == "sac_corr_without_1e-6" else scale * om + 1e-6
            dxt = dact.sum(0) * scale * om + dlogp * (2 * scale * y * om) / den
            dstd = dxt * eps - dlogp / std
            dh[:, :A] = dxt
            dh[:, A:] = dstd * std if m == "log_std_clamp_passes_gradient" else \
                torch.where((raw >= -5.0) & (raw <= 2.0), dstd * std, torch.zeros_like(std))
        return {"dhead": dh}

    return worst(run(), ref, bd), worst(run(mutant), ref, bd)


def _droq_mutant(mutant):
    nets, B = 2, 1000
    q, logp, _, _ = critic_inputs(B, nets, seed=23)
    la = torch.tensor([0.0])
    ref, bd = R.sac_actor_loss(q, logp, la, -3.0, True)

    def run(m=None):
        out = {k: torch.empty(1) for k in ("actor_loss", "alpha_loss", "dlog_alpha")}
        out["dq"] = torch.empty(nets, B)
        dem.droq_actor_loss(q, logp, la, R.f32(-3.0), out["dq"], out["actor_loss"], out["alpha_loss"],
                            out["dlog_alpha"])
        if m:
            out["dq"].fill_(-1.0 / B)
        return out

    return worst(run(), ref, bd), worst(run(mutant), ref, bd)


def _a2c_mutant(mutant):
    N, seg, dist = 256, 64, "cat18"
    mode, dims = DISTS[dist]
    inp = a2c_inputs(N, dist, seed=24)
    ref, bd = R.a2c_loss(*inp, seg, dims, mode, True, False, VF, ENT)

    class Shifted(A2CEmulOps):
        """normalises minibatch i with the statistics of its rows shifted down by one"""
        def a2c_loss(self, head, actions, adv, values, returns, dhead, dvalues, losses, seg, *args):
            a2 = adv.clone()
            for r0 in range(0, N, seg):
                r1 = min(N, r0 + seg)
                s0, s1 = min(r0 + 1, N - (r1 - r0)), min(r0 + 1, N - (r1 - r0)) + (r1 - r0)
                src = adv[s0:s1]
                a2[r0:r1] = (adv[r0:r1] - src.mean()) / (src.std() + 1e-8)
            super().a2c_loss(head, actions, a2, values, returns, dhead, dvalues, losses, seg, args[0], args[1],
                             False, *args[3:])

    return (worst(emul_a2c(inp, seg, dims, mode, True, False), ref, bd),
            worst(emul_a2c(inp, seg, dims, mode, True, False, ops=Shifted()), ref, bd))


def _gae_mutant(mutant):
    r, v, d, nv = gae_inputs(17, 257, "alternating", seed=25)
    g, lm = R.f32(0.99), R.f32(0.95)
    ref, bd = R.gae(r, v, d, nv, g, lm)
    return worst(fp32_gae(r, v, d, nv, g, lm), ref, bd), worst(fp32_gae(r, v, d, nv, g, lm, textbook=True), ref, bd)


MUTANTS = {
    "grad_through_clipped_branch": _ppo_mutant,       # the policy gradient through the clipped ratio
    "biased_std": _ppo_mutant,                        # advantage std divided by n, B = 31
    "eps_in_sqrt": _ppo_mutant,                       # sqrt(var + 1e-8), near-constant advantages
    "strict_value_clip_mask": _ppo_mutant,            # |val - old| < clip: rows exactly at +-clip lose half dval
    "entropy_grad_without_H": _ppo_mutant,            # the categorical entropy gradient without + H
    "one_lse_over_all_heads": _ppo_mutant,            # one logsumexp over every head
    "tanh_corr_at_atanh": _ppo_mutant,                # the tanh correction at atanh(a), the "corrected" formula
    "sac_corr_without_1e-6": _sac_mutant,             # SAC's correction derivative without the 1e-6
    "log_std_clamp_passes_gradient": _sac_mutant,     # the log-std gradient outside [-5, 2]
    "droq_dq_minus_1_over_B": _droq_mutant,           # DroQ dq = -1 / B instead of -1 / (nets B)
    "a2c_segment_shifted_by_one": _a2c_mutant,        # A2C normalisation statistics one row off
    "gae_textbook_dones": _gae_mutant,                # GAE masking with dones[t + 1]
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_bounds_reject_subtly_wrong_implementations(mutant):
    honest, wrong = MUTANTS[mutant](mutant)
    assert max(honest.values()) <= 0.5, honest
    assert max(wrong.values()) >= 4.0, wrong
