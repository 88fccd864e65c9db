"""The persistent RSSM scan kernels (csrc/rssm_scan.cu: forward and BPTT, each one cooperative launch) called directly
through `CudaOps.rssm_scan_fwd` / `rssm_scan_bwd` on seeded tensors, against the float64 reference
oracle/rssm_scan_ref.py, across the envelope `scan_check` admits: both instantiations (`fix`: the compile-time S widths,
`generic`), one or two 4-column groups per CTA in each layer (mh, mx, mr), partial last groups, ragged and empty
sampling units, one to sixteen rows, and the refusals at the envelope's edges."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle.rssm_scan_ref import scan_reference

pytestmark = pytest.mark.gpu

SCAN_G = 128          # CTAs of the persistent kernels
EPS = 1e-3
NAN = float("nan")
FWD_RTOL = 3e-6       # x sqrt(reduction length), relative to the tensor's largest magnitude (tests/test_gpu_ops.py)
BWD_RTOL = 5e-5       # relative to the gradient's largest magnitude (tests/test_gpu_engine.py fused-vs-per-step)
MARGINS = {}          # case id -> {tensor: worst error / bound}, kept for reporting


def owned(width):
    """4-column groups of `width` owned by CTA 0 (the most any CTA owns)"""
    return ((width + 3) // 4 + SCAN_G - 1) // SCAN_G


#          T   B   S   D    R     Dx   Dr   A   what it reaches
CASES = {
    "01": (64, 16, 32, 32, 512, 512, 512, 6),    # fix, production S
    "02": (9, 5, 32, 32, 512, 512, 512, 2),      # fix with a partial MMA tile
    "03": (64, 16, 32, 32, 256, 256, 256, 18),   # generic, production XS
    "04": (12, 1, 8, 16, 128, 96, 64, 4),        # one row
    "05": (6, 16, 64, 16, 256, 256, 256, 3),     # S = 64: 8-row sampling units (MAXRPU)
    "06": (10, 13, 10, 12, 96, 64, 80, 5),       # ragged and empty sampling units; rows starting at t = 0 from zeros
    "07": (8, 16, 1, 32, 64, 32, 32, 1),         # sixteen one-row sampling units
    "08": (8, 7, 6, 5, 26, 34, 30, 3),           # partial last 4-column group in every layer
    "09a": (6, 16, 8, 8, 520, 520, 64, 4),       # two groups per CTA in the GRU and x layers
    "09b": (6, 16, 16, 16, 256, 1024, 256, 4),   # two x groups per CTA at the Dx limit
    "10": (1, 16, 16, 32, 128, 128, 128, 2),     # T = 1: nothing carried
    "11a": (8, 4, 8, 2, 64, 64, 64, 2),          # two classes
    "11b": (8, 4, 8, 1, 64, 64, 64, 2),          # one class
}
ZERO_START = ("06", "08")                        # cases with rows whose first step is not a sequence start


def case_id(key, unimix):
    T, B, S, D, R, Dx, Dr, A = CASES[key]
    inst = "fix" if (S, D, R, Dx, Dr) == (32, 32, 512, 512, 512) else "generic"
    return f"c{key}-{inst}-mh{owned(R)}-mx{owned(Dx)}-mr{owned(Dr)}-B{B}-S{S}x{D}-unimix{unimix:g}"


PARAMS = ([pytest.param(k, 0.01, id=case_id(k, 0.01)) for k in CASES]
          + [pytest.param(k, 0.0, id=case_id(k, 0.0)) for k in ("03", "08")])


def make_first(T, B, g, zero_start):
    """is_first [T*B]: first[0] = 1 (the trainer forces it), ~10 % resets mid-sequence, one step at which every row
    resets, one row that resets at every step; `zero_start`: some rows do not start a sequence at t = 0"""
    first = (torch.rand(T, B, generator=g) < 0.1).float()
    first[0] = 1.0
    if zero_start:
        first[0, : (B + 1) // 2] = 0.0
    if T > 2:
        first[T // 2] = 1.0
    if B > 1:
        first[:, B - 1] = 1.0
    return first.reshape(-1)


def make_problem(shape, seed, zero_start=False):
    """(dims, tensors, grads) of one scan on the GPU.  Outputs are NaN-filled so that an element the kernel does not
    write stays visible; inputs the kernels must not read (the prior's weights, d_prior_mix, latent padding of d_latent)
    are NaN so that reading them poisons the results."""
    T, B, S, D, R, Dx, Dr, A = shape
    Z, N = S * D, T * B
    ld_lat, ld_wr1 = Z + R + 5, R + 7
    g = torch.Generator().manual_seed(seed)

    def w(rows, cols, fan_in):
        return torch.randn(rows, cols, generator=g) / math.sqrt(fan_in)

    def gamma(n):
        return 1.0 + 0.2 * torch.randn(n, generator=g)

    def beta(n):
        return 0.2 * torch.randn(n, generator=g)

    t = dict(W_in=w(Dx, Z + A, S + A), lnx_g=gamma(Dx), lnx_b=beta(Dx), W_g=w(3 * R, R + Dx, R + Dx),
             lng_g=gamma(3 * R), lng_b=beta(3 * R), W_r1=w(Dr, ld_wr1, R), lnr_g=gamma(Dr), lnr_b=beta(Dr),
             W_r2=w(Z, Dr, Dr) * 2.0, b_r2=beta(Z), h0=torch.tanh(torch.randn(R, generator=g)),
             z0=F.one_hot(torch.randint(D, (S,), generator=g), D).float().reshape(Z),
             pe=torch.randn(N, Dr, generator=g), actions=torch.randn(N, A, generator=g),
             first=make_first(T, B, g, zero_start), noise=torch.empty(N, Z).exponential_(generator=g))
    for k in ("W_t1", "lnt_g", "lnt_b", "W_t2", "b_t2"):
        t[k] = torch.full((8,), NAN)
    for k, width in (("latent", ld_lat), ("z_in", Z), ("h_in", R), ("a_in", A), ("x_pre", Dx), ("x_act", Dx),
                     ("g_pre", 3 * R), ("g_ln", 3 * R), ("tr_pre", 8), ("tr_act", 8), ("rp_pre", Dr), ("rp_act", Dr),
                     ("post_raw", Z), ("prior_raw", Z), ("post_mix", Z), ("prior_mix", Z)):
        t[k] = torch.full((N, width), NAN)
    d_latent = torch.randn(N, ld_lat, generator=g) * 0.1
    d_latent[:, Z + R:] = NAN
    gr = dict(d_latent=d_latent, d_post_mix=torch.randn(N, Z, generator=g) * 0.1, d_prior_mix=torch.full((N, Z), NAN),
              d_h0=torch.full((R,), NAN), q_r=torch.zeros(N, R), q_g=torch.zeros(N, R + Dx), q_x=torch.zeros(N, Z))
    for k, width in (("d_post_raw", Z), ("d_prior_raw", Z), ("d_rp_act", Dr), ("d_rp_pre", Dr), ("d_tr_act", 8),
                     ("d_tr_pre", 8), ("d_g_ln", 3 * R), ("d_g_pre", 3 * R), ("d_x_act", Dx), ("d_x_pre", Dx)):
        gr[k] = torch.full((N, width), NAN)
    dims = dict(T=T, B=B, S=S, D=D, R=R, A=A, Dx=Dx, Dt=8, Dr=Dr, ld_lat=ld_lat, ld_wr1=ld_wr1)
    return dims, {k: v.cuda() for k, v in t.items()}, {k: v.cuda() for k, v in gr.items()}


FWD_OUT = ("latent", "z_in", "h_in", "a_in", "x_pre", "x_act", "g_pre", "g_ln", "rp_pre", "rp_act", "post_raw", "post_mix")
FWD_UNUSED = ("tr_pre", "tr_act", "prior_raw", "prior_mix")
BWD_OUT = ("d_post_raw", "d_rp_act", "d_g_ln", "d_x_act", "d_h0")
BWD_UNUSED = ("d_prior_raw", "d_rp_pre", "d_tr_act", "d_tr_pre", "d_g_pre", "d_x_pre")


def run_fwd(ops, dims, unimix, t, ws):
    ops.rssm_scan_fwd(dims, EPS, unimix, t, ws)
    assert ops.rssm_scan_error(ws) == 0, "a hand-off of the forward scan timed out"
    return {k: t[k].clone() for k in FWD_OUT}


def run_bwd(ops, dims, unimix, t, gr, ws):
    ops.rssm_scan_bwd(dims, EPS, unimix, t, gr, ws)
    assert ops.rssm_scan_error(ws) == 0, "a hand-off of the backward scan timed out"
    return {k: gr[k].clone() for k in BWD_OUT}


def pre_products(ops, dims, t, gr):
    """the three batched `pre-activation x weight` products the backward kernel consumes (as
    engine._scan_backward_fused computes them)"""
    R, Z = dims["R"], dims["S"] * dims["D"]
    ops.gemm(t["rp_pre"], t["W_r1"][:, :R], gr["q_r"], False, False)
    ops.gemm(t["g_pre"], t["W_g"], gr["q_g"], False, False)
    ops.gemm(t["x_pre"], t["W_in"][:, :Z], gr["q_x"], False, False)


@pytest.fixture(scope="module")
def ops():
    from sheeprl_b200.lib import CudaOps

    return CudaOps()


@pytest.mark.parametrize("key,unimix", PARAMS)
def test_scan_kernels_match_float64_reference(ops, key, unimix):
    T, B, S, D, R, Dx, Dr, A = CASES[key]
    Z = S * D
    dims, t, gr = make_problem(CASES[key], seed=100 + list(CASES).index(key), zero_start=key in ZERO_START)
    assert ops.rssm_scan_supported(dims, backward=False) and ops.rssm_scan_supported(dims, backward=True)
    ws = ops.rssm_scan_workspace(T, B, S, D, Dx, R, Dr)
    fwd = run_fwd(ops, dims, unimix, t, ws)
    pre_products(ops, dims, t, gr)
    bwd = run_bwd(ops, dims, unimix, t, gr, ws)
    cpu = {k: v.cpu() for k, v in (t | gr).items()}
    lat = cpu["latent"]

    # ---- the kernels write exactly what they own
    assert lat[:, Z + R:].isnan().all(), "latent padding columns were written"
    for k in FWD_OUT:
        v = lat[:, : Z + R] if k == "latent" else cpu[k]
        assert torch.isfinite(v).all(), (k, "not every owned element was written (or it is not finite)")
    for k in BWD_OUT:
        assert torch.isfinite(cpu[k]).all(), (k, "not every owned element was written (or it is not finite)")
    for k in FWD_UNUSED + BWD_UNUSED:
        assert cpu[k].isnan().all(), (k, "documented as unused, but written")

    # ---- chain consistency, bit-exact: the carried rows are the masked previous step's (or the initial state)
    f = cpu["first"].reshape(T, B, 1) != 0
    lat3 = lat.reshape(T, B, -1)
    prev_z = torch.cat((torch.zeros(1, B, Z), lat3[:-1, :, :Z]), 0)
    prev_h = torch.cat((torch.zeros(1, B, R), lat3[:-1, :, Z:Z + R]), 0)
    assert torch.equal(cpu["z_in"].reshape(T, B, Z), torch.where(f, cpu["z0"].expand(T, B, Z), prev_z)), "z_in"
    assert torch.equal(cpu["h_in"].reshape(T, B, R), torch.where(f, cpu["h0"].expand(T, B, R), prev_h)), "h_in"
    acts = cpu["actions"].reshape(T, B, A)
    assert torch.equal(cpu["a_in"].reshape(T, B, A), torch.where(f, torch.zeros_like(acts), acts)), "a_in"

    # ---- forward, one step at a time from the kernel's own chain inputs, teacher-forced
    one = scan_reference(dims, EPS, unimix, cpu, one_step=True)
    got = {k: cpu[k] for k in one if k not in ("h", "scores")} | {"h": lat[:, Z:Z + R]}
    K = dict(x_pre=Z + A, x_act=Z + A, g_pre=R + Dx, g_ln=R + Dx, h=R + Dx, rp_pre=R, rp_act=R, post_raw=Dr, post_mix=Dr)
    margins = {}
    for k, kk in K.items():
        err = float((got[k].double() - one[k]).abs().max())
        margins[k] = err / (FWD_RTOL * math.sqrt(kk) * max(1e-3, float(one[k].abs().max())))

    # ---- samples: exactly one-hot, and the pick is an argmax of the float64 scores p / q
    z = lat[:, :Z].reshape(-1, S, D)
    assert torch.all((z == 0) | (z == 1)) and torch.all(z.sum(-1) == 1), "samples are not one-hot per group"
    s = one["scores"]
    pick = z.argmax(-1)
    smax = s.max(-1).values
    assert torch.all(smax - s.gather(-1, pick.unsqueeze(-1)).squeeze(-1) <= 1e-5 * smax), "a pick is not an argmax"
    assert float((pick != s.argmax(-1)).double().mean()) < 1e-3, "too many picks differ from the strict argmax"

    # ---- backward against float64 autograd of the carried, teacher-forced chain
    ref = scan_reference(dims, EPS, unimix, cpu, d_latent=cpu["d_latent"][:, : Z + R], d_post_mix=cpu["d_post_mix"])
    for k in BWD_OUT:
        err = float((cpu[k].double() - ref[k]).abs().max())
        margins[k] = err / (BWD_RTOL * max(1e-3, float(ref[k].abs().max())))   # (one class: d_post_raw = 0)
    MARGINS[case_id(key, unimix)] = margins
    assert max(margins.values()) <= 1.0, {k: round(v, 3) for k, v in margins.items()}

    # ---- bit-reproducible (fixed-order K-slice sums).  The backward reruns on the same q_r / q_g / q_x: the GEMM
    # that makes them may split K with atomics, so recomputing them is not bit-reproducible itself.
    fwd2 = run_fwd(ops, dims, unimix, t, ws)
    for k in FWD_OUT:
        v1, v2 = (x[:, : Z + R] if k == "latent" else x for x in (fwd[k], fwd2[k]))
        assert torch.equal(v1, v2), (k, "second forward differs")
    bwd2 = run_bwd(ops, dims, unimix, t, gr, ws)
    for k in BWD_OUT:
        assert torch.equal(bwd[k], bwd2[k]), (k, "second backward differs")


#            T  B   S   D    R     Dx    Dr   A
REFUSALS = {
    "B17": (4, 17, 4, 4, 64, 64, 64, 2),
    "D33": (4, 4, 4, 33, 64, 64, 64, 2),
    "S65": (4, 4, 65, 2, 64, 64, 64, 2),
    "SxD_odd": (4, 4, 3, 3, 64, 64, 64, 2),
    "Dr_odd": (4, 4, 4, 4, 64, 64, 63, 2),
    "Dx1026": (4, 4, 4, 4, 64, 1026, 64, 2),
    "R1028_mh3": (4, 4, 4, 4, 1028, 64, 64, 2),
    "smem": (4, 4, 32, 32, 1024, 1024, 1024, 2),
    "short_workspace": (4, 4, 4, 4, 64, 64, 64, 2),
}


@pytest.mark.parametrize("name", list(REFUSALS))
def test_scan_check_and_launches_refuse_outside_envelope(ops, name):
    """The envelope query refuses every model outside the envelope in both directions (the engine asks it once, at
    construction, to choose between the persistent and the per-step kernels); the launches refuse the same models, and a
    short workspace, before anything is launched (all outputs stay untouched)."""
    from sheeprl_b200.lib import B200RLError

    T, B, S, D, R, Dx, Dr, A = REFUSALS[name]
    dims, t, gr = make_problem(REFUSALS[name], seed=7)
    ws = ops.rssm_scan_workspace(T, B, S, D, Dx, R, Dr)
    in_envelope = name == "short_workspace"           # the query reads dims only
    assert ops.rssm_scan_supported(dims, backward=False) == in_envelope
    assert ops.rssm_scan_supported(dims, backward=True) == in_envelope
    if name == "short_workspace":
        ws, match = ws[:-1], "workspace"
    else:
        match = "supports|shared memory"
    for call in (lambda: ops.rssm_scan_fwd(dims, EPS, 0.01, t, ws),
                 lambda: ops.rssm_scan_bwd(dims, EPS, 0.01, t, gr, ws)):
        with pytest.raises(B200RLError, match=match):
            call()
    torch.cuda.synchronize()
    for k in FWD_OUT + FWD_UNUSED:
        assert t[k].isnan().all(), (k, "written by a refused call")
    for k in BWD_OUT + BWD_UNUSED:
        assert gr[k].isnan().all(), (k, "written by a refused call")
