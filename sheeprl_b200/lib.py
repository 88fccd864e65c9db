"""ctypes binding of the C-ABI in `include/b200rl.h` (library: `sheeprl_b200/libb200rl.so`).

`CudaOps` exposes one method per entry point, taking torch tensors purely as (device pointer, shape,
leading dimension) carriers; all work is enqueued on torch's current CUDA stream.  There is NO
fallback: constructing `CudaOps` without the built library or without an sm_90 (H100) GPU raises.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional, Sequence

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200rl.so")

c_int, c_ll, c_float, c_void_p = ctypes.c_int, ctypes.c_longlong, ctypes.c_float, ctypes.c_void_p

_lib = None


class B200RLError(RuntimeError):
    pass


def load_library(path: str = LIB_PATH) -> ctypes.CDLL:
    """Loads the shared library (no GPU needed to load; kernels need one to run)."""
    global _lib
    if _lib is None:
        if not os.path.exists(path):
            raise B200RLError(
                f"{path} not found: build it with `python -m sheeprl_b200.build` (nvcc, sm_90a). "
                "The B200 engine has no CPU / PyTorch fallback.")
        _lib = ctypes.CDLL(path)
        _lib.b200rl_last_error.restype = ctypes.c_char_p
        _lib.b200rl_build_arch.restype = ctypes.c_char_p
    return _lib


def declared_symbols(header: Optional[str] = None) -> Sequence[str]:
    """Names of every function declared in include/b200rl.h."""
    import re

    header = header or os.path.join(os.path.dirname(_HERE), "include", "b200rl.h")
    src = open(header).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200rl_[a-z0-9_]+)\s*\(", src)))


def _p(t: Optional[torch.Tensor]):
    return c_void_p(0) if t is None else c_void_p(t.data_ptr())


def _ld(t: torch.Tensor) -> int:
    """Row stride of a 2-D view with unit inner stride (1-D tensors are single rows)."""
    if t.dim() == 1:
        assert t.numel() <= 1 or t.stride(0) == 1, "1-D views must be contiguous"
        return max(t.numel(), 1)
    assert t.dim() == 2, f"expected a 2-D view, got {tuple(t.shape)}"
    assert t.shape[1] == 1 or t.stride(1) == 1, f"inner stride must be 1, got {t.stride()}"
    return t.stride(0) if t.shape[0] > 1 else max(t.stride(0), t.shape[1])


def _f32(*ts):
    for t in ts:
        if t is not None:
            assert t.dtype == torch.float32 and t.is_cuda, (t.dtype, t.device)


class RssmScanArgs(ctypes.Structure):
    """Mirror of `b200rl_rssm_scan_args` (include/b200rl.h) — field order must match the C struct."""
    POINTERS = ("W_in", "lnx_g", "lnx_b", "W_g", "lng_g", "lng_b", "W_t1", "lnt_g", "lnt_b", "W_t2", "b_t2",
                "W_r1", "lnr_g", "lnr_b", "W_r2", "b_r2", "h0", "z0", "pe", "actions", "first", "noise", "latent",
                "z_in", "h_in", "a_in", "x_pre", "x_act", "g_pre", "g_ln", "tr_pre", "tr_act", "rp_pre", "rp_act",
                "post_raw", "prior_raw", "post_mix", "prior_mix")
    _fields_ = ([(n, c_int) for n in ("T", "B", "S", "D", "R", "A", "Dx", "Dt", "Dr", "ld_lat", "ld_wr1")]
                + [("eps", c_float), ("unimix", c_float)]
                + [(n, c_void_p) for n in POINTERS]
                + [("workspace", c_void_p), ("workspace_bytes", c_ll)])


class RssmScanGrads(ctypes.Structure):
    """Mirror of `b200rl_rssm_scan_grads`."""
    POINTERS = ("d_latent", "d_post_mix", "d_prior_mix", "d_post_raw", "d_prior_raw", "d_rp_act", "d_rp_pre",
                "d_tr_act", "d_tr_pre", "d_g_ln", "d_g_pre", "d_x_act", "d_x_pre", "d_h0", "q_r", "q_g", "q_x")
    _fields_ = [(n, c_void_p) for n in POINTERS]


class CudaOps:
    name = "cuda"

    def __init__(self, device="cuda"):
        if not torch.cuda.is_available():
            raise B200RLError("no CUDA device visible: the B200 engine has no CPU fallback")
        self.lib = load_library()
        self.device = torch.device(device)
        if self.device.index is not None:
            torch.cuda.set_device(self.device)
        if self.lib.b200rl_device_check() != 0:
            raise B200RLError(self.lib.b200rl_last_error().decode())
        self.launches = 0
        self.use_tc = os.environ.get("B200RL_DISABLE_TC", "0") != "1"   # tensor-core (wgmma) paths
        self._pack_bufs = {}
        self._scratch_bufs = {}

    # ------------------------------------------------------------------ plumbing
    def _st(self):
        return c_void_p(torch.cuda.current_stream().cuda_stream)

    def _ck(self, rc: int):
        self.launches += 1
        if rc != 0:
            raise B200RLError(self.lib.b200rl_last_error().decode())

    # ------------------------------------------------------------------ GEMM family
    def set_matmul_precision(self, precision: str) -> None:
        """"highest": fp32-accurate 3xTF32 products (default); "high" / "medium": one TF32 product per k-step — what
        torch.set_float32_matmul_precision("high") gives the reference on a GPU (sheeprl/configs/config.yaml:18)."""
        p = str(precision).lower()
        if p not in ("highest", "high", "medium"):
            raise ValueError(f"float32_matmul_precision must be highest / high / medium, got {precision}")
        self._ck(self.lib.b200rl_set_matmul_precision(c_int(3 if p == "highest" else 1)))
        self.launches -= 1

    def matmul_precision(self) -> str:
        return "highest" if int(self.lib.b200rl_get_matmul_precision()) == 3 else "high"

    def gemm(self, A, B, C, transA: bool, transB: bool, bias=None, accumulate: bool = False):
        _f32(A, B, C, bias)
        M, N = C.shape
        K = A.shape[0] if transA else A.shape[1]
        assert (A.shape[1] if transA else A.shape[0]) == M, (A.shape, C.shape, transA)
        assert (B.shape[0] if transB else B.shape[1]) == N and (B.shape[1] if transB else B.shape[0]) == K, \
            (A.shape, B.shape, C.shape, transA, transB)
        # every layout goes to one entry point: transposed operands are read in place as MN-major tiles
        self._ck(self.lib.b200rl_gemm_f32(_p(A), _p(B), _p(C), _p(bias), c_int(M), c_int(N), c_int(K), c_int(_ld(A)),
                                          c_int(_ld(B)), c_int(_ld(C)), c_int(int(transA)), c_int(int(transB)),
                                          c_int(int(accumulate)), self._st()))

    def gemm_ln_supported(self, A, W, mode: int = 0) -> bool:
        M, K = A.shape
        return self.use_tc and bool(self.lib.b200rl_gemm_ln_supported(_p(A), _p(W), c_int(M), c_int(W.shape[0]), c_int(K),
                                                                     c_int(_ld(A)), c_int(_ld(W)), c_int(mode)))

    def gemm_ln_act(self, A, W, gamma, beta, eps: float, act: int, out, pre=None):
        """out = act(LayerNorm(A W^T)); `pre` (optional) receives A W^T.  Two launches (product, fused reduce + LN)."""
        _f32(A, W, gamma, beta, out, pre)
        M, K = A.shape
        N = W.shape[0]
        assert W.shape[1] == K and out.shape == (M, N)
        self._ck(self.lib.b200rl_gemm_ln(_p(A), _p(W), c_int(M), c_int(N), c_int(K), c_int(_ld(A)), c_int(_ld(W)), _p(gamma),
                                         _p(beta), c_float(eps), c_int(act), _p(pre), c_ll(_ld(pre) if pre is not None else 0),
                                         _p(out), c_ll(_ld(out)), c_int(0), _p(None), c_ll(0), _p(None), c_ll(0), _p(None), c_ll(0),
                                         self._st()))
        self.launches += 1

    def gemm_ln_gru(self, A, W, gamma, beta, eps: float, h_prev, h_out, h_out2=None, g_pre=None, g_ln=None):
        """LayerNormGRUCell on [h | x] rows `A`: h_out = gate(LayerNorm(A W^T), h_prev) (models.py:396-403)."""
        _f32(A, W, gamma, beta, h_prev, h_out, h_out2, g_pre, g_ln)
        M, K = A.shape
        N = W.shape[0]
        assert W.shape[1] == K and h_prev.shape == (M, N // 3) and h_out.shape == (M, N // 3)
        self._ck(self.lib.b200rl_gemm_ln(_p(A), _p(W), c_int(M), c_int(N), c_int(K), c_int(_ld(A)), c_int(_ld(W)), _p(gamma),
                                         _p(beta), c_float(eps), c_int(0), _p(g_pre),
                                         c_ll(_ld(g_pre) if g_pre is not None else 0), _p(g_ln),
                                         c_ll(_ld(g_ln) if g_ln is not None else 0), c_int(1), _p(h_prev), c_ll(_ld(h_prev)),
                                         _p(h_out), c_ll(_ld(h_out)), _p(h_out2),
                                         c_ll(_ld(h_out2) if h_out2 is not None else 0), self._st()))
        self.launches += 1

    def _scratch(self, slot: str, numel: int) -> torch.Tensor:
        buf = self._scratch_bufs.get(slot)
        if buf is None or buf.numel() < numel:
            buf = torch.empty(numel, dtype=torch.float32, device=self.device)
            self._scratch_bufs[slot] = buf
        return buf

    def col_sum(self, X, out, accumulate: bool = False):
        _f32(X, out)
        self._ck(self.lib.b200rl_col_sum(_p(X), _p(out), c_ll(X.shape[0]), c_int(X.shape[1]), c_ll(_ld(X)),
                                         c_int(int(accumulate)), self._st()))

    def ln_act_fwd(self, X, gamma, beta, eps: float, act: int, Y):
        _f32(X, gamma, beta, Y)
        self._ck(self.lib.b200rl_ln_act_fwd(_p(X), _p(gamma), _p(beta), _p(Y), c_ll(X.shape[0]), c_int(X.shape[1]),
                                            c_ll(_ld(X)), c_ll(_ld(Y)), c_float(eps), c_int(act), self._st()))

    def ln_act_bwd(self, X, gamma, beta, eps: float, act: int, dY, dX, dgamma, dbeta, accumulate: bool = False):
        _f32(X, gamma, beta, dY, dX, dgamma, dbeta)
        self._ck(self.lib.b200rl_ln_act_bwd(_p(X), _p(gamma), _p(beta), _p(dY), _p(dX), _p(dgamma), _p(dbeta),
                                            c_ll(X.shape[0]), c_int(X.shape[1]), c_ll(_ld(X)), c_ll(_ld(dY)),
                                            c_ll(_ld(dX)), c_float(eps), c_int(act), c_int(int(accumulate)), self._st()))

    # ------------------------------------------------------------------ convolutions
    def obs_prep(self, obs, out):
        assert obs.is_cuda and obs.is_contiguous() and out.is_contiguous()
        assert obs.dtype in (torch.uint8, torch.float32), obs.dtype
        NB, C, H, W = obs.shape
        self._ck(self.lib.b200rl_obs_prep(_p(obs), c_int(int(obs.dtype == torch.uint8)), _p(out), c_ll(NB), c_int(C),
                                          c_int(H * W), self._st()))

    def transpose_batched(self, X, Y):
        _f32(X, Y)
        assert X.is_contiguous() and Y.is_contiguous()
        NB, a, b = X.shape
        self._ck(self.lib.b200rl_transpose_batched(_p(X), _p(Y), c_int(NB), c_int(a), c_int(b), self._st()))

    def conv_down(self, big, W, small):
        _f32(big, W, small)
        assert big.is_contiguous() and small.is_contiguous() and W.is_contiguous()
        NB, h, w, Cs = small.shape
        Cb = big.shape[-1]
        assert tuple(big.shape) == (NB, 2 * h, 2 * w, Cb) and tuple(W.shape) == (Cs, Cb, 4, 4)
        if self.use_tc and self.lib.b200rl_conv_tc_supported(0, NB, h, w, Cs, Cb):
            Wp = self._packed(W, 0, Cs, Cb)
            self._ck(self.lib.b200rl_conv_down_tc(_p(big), _p(Wp), _p(small), c_int(NB), c_int(h), c_int(w), c_int(Cs),
                                                  c_int(Cb), self._st()))
            return
        self._ck(self.lib.b200rl_conv_down(_p(big), _p(W), _p(small), c_int(NB), c_int(h), c_int(w), c_int(Cs),
                                           c_int(Cb), self._st()))

    def _packed(self, W, mode_up: int, Cs: int, Cb: int):
        """Tap-major copy of a conv weight for the tensor-core kernels (caller-owned workspace, refreshed on every
        use because the optimiser rewrites W each step; 16*Cs*Cb floats, a few microseconds)."""
        key = (W.data_ptr(), mode_up)
        buf = self._pack_bufs.get(key)
        self.lib.b200rl_conv_pack_floats.restype = c_ll
        need = int(self.lib.b200rl_conv_pack_floats(c_int(mode_up), c_int(Cs), c_int(Cb)))
        if buf is None or buf.numel() != need:
            buf = torch.empty(need, dtype=torch.float32, device=W.device)
            self._pack_bufs[key] = buf
        self._ck(self.lib.b200rl_conv_pack(_p(W), _p(buf), c_int(mode_up), c_int(Cs), c_int(Cb), self._st()))
        return buf

    def conv_up(self, small, W, big, bias=None):
        _f32(big, W, small, bias)
        assert big.is_contiguous() and small.is_contiguous() and W.is_contiguous()
        NB, h, w, Cs = small.shape
        Cb = big.shape[-1]
        assert tuple(big.shape) == (NB, 2 * h, 2 * w, Cb) and tuple(W.shape) == (Cs, Cb, 4, 4)
        if self.use_tc and self.lib.b200rl_conv_tc_supported(1, NB, h, w, Cs, Cb):
            Wp = self._packed(W, 1, Cs, Cb)
            self._ck(self.lib.b200rl_conv_up_tc(_p(small), _p(Wp), _p(big), _p(bias), c_int(NB), c_int(h), c_int(w),
                                                c_int(Cs), c_int(Cb), self._st()))
            return
        self._ck(self.lib.b200rl_conv_up(_p(small), _p(W), _p(big), _p(bias), c_int(NB), c_int(h), c_int(w), c_int(Cs),
                                         c_int(Cb), self._st()))

    def conv_wgrad(self, small, big, dW, accumulate: bool = False):
        _f32(big, dW, small)
        assert big.is_contiguous() and small.is_contiguous() and dW.is_contiguous()
        NB, h, w, Cs = small.shape
        Cb = big.shape[-1]
        assert tuple(big.shape) == (NB, 2 * h, 2 * w, Cb) and tuple(dW.shape) == (Cs, Cb, 4, 4)
        if self.use_tc and NB * h * w >= 1024 and Cs >= 48 and Cb >= 8:
            self.lib.b200rl_conv_wgrad_tc_workspace.restype = c_ll
            n = int(self.lib.b200rl_conv_wgrad_tc_workspace(c_int(NB), c_int(h), c_int(w), c_int(Cs), c_int(Cb)))
            ws = self._scratch("wgrad", n)
            self._ck(self.lib.b200rl_conv_wgrad_tc(_p(small), _p(big), _p(dW), _p(ws), c_int(NB), c_int(h), c_int(w),
                                                   c_int(Cs), c_int(Cb), c_int(int(accumulate)), self._st()))
            return
        self._ck(self.lib.b200rl_conv_wgrad(_p(small), _p(big), _p(dW), c_int(NB), c_int(h), c_int(w), c_int(Cs),
                                            c_int(Cb), c_int(int(accumulate)), self._st()))

    # ------------------------------------------------------------------ RSSM pieces
    def gru_gate_fwd(self, G, Hin, Hout):
        _f32(G, Hin, Hout)
        M, R = Hin.shape
        self._ck(self.lib.b200rl_gru_gate_fwd(_p(G), _p(Hin), _p(Hout), c_ll(M), c_int(R), c_ll(_ld(G)), c_ll(_ld(Hin)),
                                              c_ll(_ld(Hout)), self._st()))

    def gru_gate_bwd(self, G, Hin, dH, dG, dHin):
        _f32(G, Hin, dH, dG, dHin)
        M, R = Hin.shape
        self._ck(self.lib.b200rl_gru_gate_bwd(_p(G), _p(Hin), _p(dH), _p(dG), _p(dHin), c_ll(M), c_int(R), c_ll(_ld(G)),
                                              c_ll(_ld(Hin)), c_ll(_ld(dH)), c_ll(_ld(dG)), c_ll(_ld(dHin)), self._st()))

    def mask_mix(self, prev, init, first, out):
        _f32(prev, init, first, out)
        M, C = out.shape
        self._ck(self.lib.b200rl_mask_mix(_p(prev), _p(init), _p(first), _p(out), c_ll(M), c_int(C), c_ll(_ld(prev)),
                                          c_ll(_ld(out)), self._st()))

    def mask_rows(self, X, first, out):
        self.mask_mix(X, None, first, out)

    def mask_bwd(self, dIn, first, dPrev, dInit):
        _f32(dIn, first, dPrev, dInit)
        M, C = dIn.shape
        self._ck(self.lib.b200rl_mask_bwd(_p(dIn), _p(first), _p(dPrev), _p(dInit), c_int(M), c_int(C), c_ll(_ld(dIn)),
                                          c_ll(_ld(dPrev)), self._st()))

    def cat_sample(self, raw, noise, unimix: float, groups: int, classes: int, onehot, mix_out=None):
        _f32(raw, noise, onehot, mix_out)
        M = raw.shape[0]
        if noise is not None and noise.dim() != 2:
            noise = noise.reshape(M, -1)
        self._ck(self.lib.b200rl_cat_sample(
            _p(raw), _p(noise), _p(onehot), _p(mix_out), c_ll(M), c_int(groups), c_int(classes), c_ll(_ld(raw)),
            c_ll(_ld(noise) if noise is not None else 0), c_ll(_ld(onehot) if onehot is not None else 0),
            c_ll(_ld(mix_out) if mix_out is not None else 0), c_float(unimix), self._st()))

    def head_sample_supported(self, X, W) -> bool:
        return (W.shape[0] <= 32 and X.shape[1] <= 1024 and X.shape[1] % 4 == 0 and _ld(X) % 4 == 0 and _ld(W) % 4 == 0
                and X.data_ptr() % 16 == 0 and W.data_ptr() % 16 == 0)

    def head_sample(self, X, W, bias, noise, unimix: float, raw, onehot):
        """raw = X W^T + bias; onehot = straight-through categorical sample of unimix(raw) — one launch."""
        _f32(X, W, bias, noise, raw, onehot)
        M, Kin = X.shape
        A = W.shape[0]
        assert raw.shape == (M, A) and onehot.shape == (M, A) and W.shape[1] == Kin
        self._ck(self.lib.b200rl_head_sample(_p(X), _p(W), _p(bias), _p(noise), _p(raw), _p(onehot), c_ll(M), c_int(Kin),
                                             c_int(A), c_ll(_ld(X)), c_ll(_ld(W)), c_ll(_ld(raw)),
                                             c_ll(_ld(noise) if noise is not None else 0), c_ll(_ld(onehot)),
                                             c_float(unimix), self._st()))

    def cat_sample_bwd(self, raw, dz, dmix, unimix: float, groups: int, classes: int, draw):
        _f32(raw, dz, dmix, draw)
        M = raw.shape[0]
        self._ck(self.lib.b200rl_cat_sample_bwd(
            _p(raw), _p(dz), _p(dmix), _p(draw), c_ll(M), c_int(groups), c_int(classes), c_ll(_ld(raw)),
            c_ll(_ld(dz) if dz is not None else 0), c_ll(_ld(dmix) if dmix is not None else 0), c_ll(_ld(draw)),
            c_float(unimix), self._st()))

    def kl_loss_grad(self, post_mix, prior_mix, groups, classes, kl_dyn, kl_rep, free_nats, regularizer, scale,
                     d_post, d_prior, rows):
        _f32(post_mix, prior_mix, d_post, d_prior, rows)
        assert rows.is_contiguous() and rows.shape[1] == 4
        self._ck(self.lib.b200rl_kl_loss_grad(
            _p(post_mix), _p(prior_mix), _p(d_post), _p(d_prior), _p(rows), c_ll(post_mix.shape[0]), c_int(groups),
            c_int(classes), c_ll(_ld(post_mix)), c_ll(_ld(prior_mix)), c_ll(_ld(d_post)), c_ll(_ld(d_prior)),
            c_float(kl_dyn), c_float(kl_rep), c_float(free_nats), c_float(regularizer), c_float(scale), self._st()))

    # ------------------------------------------------------------------ losses
    def mse_loss_grad(self, pred, target, scale: float, loss_row, grad):
        _f32(pred, target, loss_row, grad)
        assert pred.is_contiguous() and target.is_contiguous() and grad.is_contiguous()
        M, P = pred.shape
        self._ck(self.lib.b200rl_mse_loss_grad(_p(pred), _p(target), _p(loss_row), _p(grad), c_ll(M), c_int(P),
                                               c_float(scale), self._st()))

    def twohot_loss_grad(self, logits, x, weight, scale, low, high, loss_row, dlogits, accumulate: bool = False):
        _f32(logits, x, weight, loss_row, dlogits)
        M, nb = logits.shape
        assert x.numel() == M and x.is_contiguous()
        self._ck(self.lib.b200rl_twohot_loss_grad(
            _p(logits), _p(x), _p(weight), _p(loss_row), _p(dlogits), c_ll(M), c_int(nb), c_ll(_ld(logits)),
            c_ll(_ld(dlogits)), c_float(low), c_float(high), c_float(scale), c_int(int(accumulate)), self._st()))

    def bce_loss_grad(self, logit, target, loss_scale, scale, loss_row, dlogit):
        _f32(logit, target, loss_row, dlogit)
        assert logit.is_contiguous() and target.is_contiguous() and dlogit.is_contiguous()
        self._ck(self.lib.b200rl_bce_loss_grad(_p(logit), _p(target), _p(loss_row), _p(dlogit), c_ll(logit.numel()),
                                               c_float(loss_scale), c_float(scale), self._st()))

    def twohot_mean(self, logits, low, high, out):
        _f32(logits, out)
        self._ck(self.lib.b200rl_twohot_mean(_p(logits), _p(out), c_ll(logits.shape[0]), c_int(logits.shape[1]),
                                             c_ll(_ld(logits)), c_float(low), c_float(high), self._st()))

    def lambda_returns(self, rew, val, cont_logit, true_cont, gamma, lmbda, lam, discount):
        _f32(rew, val, cont_logit, true_cont, lam, discount)
        for t in (rew, val, cont_logit, lam, discount):
            assert t.is_contiguous()
        H, N = lam.shape
        self._ck(self.lib.b200rl_lambda_returns(_p(rew), _p(val), _p(cont_logit), _p(true_cont), _p(lam), _p(discount),
                                                c_int(H), c_int(N), c_float(gamma), c_float(lmbda), self._st()))

    def moments_update(self, x, state, decay, max_, p_low, p_high, out):
        _f32(x, state, out)
        assert x.is_contiguous()
        self._ck(self.lib.b200rl_moments_update(_p(x), c_ll(x.numel()), _p(state), _p(out), c_float(decay),
                                                c_float(max_), c_float(p_low), c_float(p_high), self._st()))

    def actor_loss_grad(self, raw, actions, lam, val, discount, moments, head_dims, unimix, ent_coef, scale, rows,
                        draw):
        _f32(raw, actions, lam, val, discount, moments, rows, draw)
        for t in (raw, actions, draw):
            assert t.is_contiguous()
        hd = (c_int * len(head_dims))(*[int(x) for x in head_dims])
        self._ck(self.lib.b200rl_actor_loss_grad(_p(raw), _p(actions), _p(lam), _p(val), _p(discount), _p(moments),
                                                 _p(rows), _p(draw), c_ll(raw.shape[0]), hd, c_int(len(head_dims)),
                                                 c_float(unimix), c_float(ent_coef), c_float(scale), self._st()))

    def sum_rows(self, X, out, scale: float):
        _f32(X, out)
        self._ck(self.lib.b200rl_sum_rows(_p(X), _p(out), c_ll(X.shape[0]), c_int(X.shape[1]), c_ll(_ld(X)),
                                          c_float(scale), self._st()))

    def weighted_mean(self, x, w, scale: float, out):
        _f32(x, w, out)
        self._ck(self.lib.b200rl_weighted_mean(_p(x), _p(w), _p(out), c_ll(x.numel()), c_float(scale), self._st()))

    # ------------------------------------------------------------------ optimiser / utilities
    def sumsq(self, x, out):
        assert out.dtype == torch.float64 and x.is_contiguous()
        self._ck(self.lib.b200rl_sumsq(_p(x), c_ll(x.numel()), _p(out), self._st()))

    def adam_step(self, p, g, m, v, normsq, max_norm, lr, b1, b2, eps, step_t, norm_out):
        _f32(p, g, m, v, norm_out)
        assert step_t.dtype == torch.int32 and normsq.dtype == torch.float64
        self._ck(self.lib.b200rl_adam_step(_p(p), _p(g), _p(m), _p(v), _p(normsq), _p(step_t), _p(norm_out),
                                           c_ll(p.numel()), c_float(max_norm), c_float(lr), c_float(b1), c_float(b2),
                                           c_float(eps), self._st()))

    def ema(self, target, src, tau: float):
        _f32(target, src)
        self._ck(self.lib.b200rl_ema(_p(target), _p(src), c_ll(target.numel()), c_float(tau), self._st()))

    def fill_exponential(self, out, seed: int, stream_id: int, counter=None):
        """Exp(1) noise from Philox4x32-10 keyed by (seed, stream_id, *counter); `counter` is a device int32
        incremented once per train step so that graph replays draw fresh noise."""
        _f32(out)
        assert out.is_contiguous()
        self._ck(self.lib.b200rl_fill_exponential(_p(out), c_ll(out.numel()), ctypes.c_ulonglong(seed & (2 ** 64 - 1)),
                                                  ctypes.c_uint(stream_id & 0xFFFFFFFF), _p(counter), self._st()))

    def increment(self, step_t):
        self._ck(self.lib.b200rl_increment(_p(step_t), self._st()))

    def zero(self, x):
        assert x.is_contiguous()
        if x.dtype == torch.float32:
            self._ck(self.lib.b200rl_zero(_p(x), c_ll(x.numel()), self._st()))
        else:
            x.zero_()

    def copy(self, src, dst):
        _f32(src, dst)
        if src.dim() == 1:
            src, dst = src.view(1, -1), dst.view(1, -1)
        M, C = src.shape
        self._ck(self.lib.b200rl_copy2d(_p(src), _p(dst), c_ll(M), c_int(C), c_ll(_ld(src)), c_ll(_ld(dst)), self._st()))

    def axpy(self, x, y, alpha: float = 1.0):
        _f32(x, y)
        assert x.is_contiguous() and y.is_contiguous()
        self._ck(self.lib.b200rl_axpy(_p(x), _p(y), c_ll(x.numel()), c_float(alpha), self._st()))

    def affine(self, x, out, alpha: float, beta: float):
        _f32(x, out)
        assert x.is_contiguous() and out.is_contiguous()
        self._ck(self.lib.b200rl_affine(_p(x), _p(out), c_ll(x.numel()), c_float(alpha), c_float(beta), self._st()))

    def symlog(self, x, y):
        """y[M,C] = symlog(x[M,C]); both may be column slices of wider buffers"""
        _f32(x, y)
        M, C = x.shape
        assert tuple(y.shape) == (M, C)
        self._ck(self.lib.b200rl_symlog(_p(x), _p(y), c_ll(M), c_int(C), c_ll(_ld(x)), c_ll(_ld(y)), self._st()))

    def tanh_fwd(self, x, y):
        _f32(x, y)
        self._ck(self.lib.b200rl_tanh_fwd(_p(x), _p(y), c_ll(x.numel()), self._st()))

    def tanh_bwd(self, y, dy, dx, accumulate: bool = False):
        _f32(y, dy, dx)
        self._ck(self.lib.b200rl_tanh_bwd(_p(y), _p(dy), _p(dx), c_ll(y.numel()), c_int(int(accumulate)), self._st()))

    # ------------------------------------------------------------------ persistent RSSM scan
    def rssm_scan_workspace(self, T: int, B: int, S: int, D: int, Dx: int, R: int, Dr: int) -> torch.Tensor:
        self.lib.b200rl_rssm_scan_workspace_bytes.restype = c_ll
        n = int(self.lib.b200rl_rssm_scan_workspace_bytes(c_int(T), c_int(B), c_int(S), c_int(D), c_int(Dx), c_int(R),
                                                          c_int(Dr)))
        return torch.zeros((n + 3) // 4, dtype=torch.int32, device=self.device)

    def _scan_args(self, dims: dict, eps: float, unimix: float, tensors: dict, workspace: torch.Tensor):
        a = RssmScanArgs()
        for k in ("T", "B", "S", "D", "R", "A", "Dx", "Dt", "Dr", "ld_lat", "ld_wr1"):
            setattr(a, k, int(dims[k]))
        a.eps, a.unimix = float(eps), float(unimix)
        for name in RssmScanArgs.POINTERS:
            t = tensors[name]
            assert t.is_cuda and t.dtype == torch.float32, name
            setattr(a, name, t.data_ptr())
        a.workspace = workspace.data_ptr()
        a.workspace_bytes = workspace.numel() * workspace.element_size()
        return a

    def rssm_scan_fwd(self, dims: dict, eps: float, unimix: float, tensors: dict, workspace: torch.Tensor):
        """dims: T,B,S,D,R,A,Dx,Dt,Dr,ld_lat,ld_wr1; tensors: name -> device tensor for every pointer field of
        `b200rl_rssm_scan_args` (include/b200rl.h)."""
        a = self._scan_args(dims, eps, unimix, tensors, workspace)
        self._ck(self.lib.b200rl_rssm_scan_fwd(ctypes.byref(a), self._st()))

    def rssm_scan_bwd_check(self, dims: dict, eps: float, unimix: float, tensors: dict, grads: dict,
                            workspace: torch.Tensor):
        """raises if the model is outside the backward kernel's envelope; launches nothing"""
        a = self._scan_args(dims, eps, unimix, tensors, workspace)
        rc = self.lib.b200rl_rssm_scan_bwd_check(ctypes.byref(a))
        if rc != 0:
            raise B200RLError(self.lib.b200rl_last_error().decode())

    def rssm_scan_bwd(self, dims: dict, eps: float, unimix: float, tensors: dict, grads: dict,
                      workspace: torch.Tensor):
        a = self._scan_args(dims, eps, unimix, tensors, workspace)
        q = RssmScanGrads()
        for name in RssmScanGrads.POINTERS:
            t = grads[name]
            assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous(), name
            setattr(q, name, t.data_ptr())
        self._ck(self.lib.b200rl_rssm_scan_bwd(ctypes.byref(a), ctypes.byref(q), self._st()))

    def rssm_scan_error(self, workspace: torch.Tensor) -> int:
        return int(self.lib.b200rl_rssm_scan_error(_p(workspace), self._st()))

    def rssm_scan_profile(self, workspace: torch.Tensor):
        """per-phase cycle counters of CTA 0 and CTA 1 of the last scan launch: [2][32] int64"""
        out = (ctypes.c_longlong * 64)()
        rc = self.lib.b200rl_rssm_scan_profile(_p(workspace), out, self._st())
        if rc != 0:
            raise B200RLError(self.lib.b200rl_last_error().decode())
        return [list(out[:32]), list(out[32:])]

    # ------------------------------------------------------------------ replay / PPO
    def replay_gather(self, storage, idx, out, n_samples: int, batch: int, seq_len: int):
        assert storage.is_contiguous() and out.is_contiguous() and idx.dtype == torch.int64 and idx.is_contiguous()
        row_bytes = storage[0].numel() * storage.element_size()
        self._ck(self.lib.b200rl_replay_gather(_p(storage), _p(idx), _p(out), c_int(n_samples), c_int(batch),
                                               c_int(seq_len), c_ll(row_bytes), self._st()))

    def replay_scatter(self, src, dst_rows, storage):
        assert storage.is_contiguous() and src.is_contiguous() and dst_rows.dtype == torch.int64
        row_bytes = storage[0].numel() * storage.element_size()
        self._ck(self.lib.b200rl_replay_scatter(_p(src), _p(dst_rows), _p(storage), c_ll(dst_rows.numel()),
                                                c_ll(row_bytes), self._st()))

    def gae(self, rewards, values, dones, next_value, gamma, lmbda, returns, advantages):
        _f32(rewards, values, dones, next_value, returns, advantages)
        T, E = rewards.shape[0], rewards[0].numel()
        self._ck(self.lib.b200rl_gae(_p(rewards), _p(values), _p(dones), _p(next_value), _p(returns), _p(advantages),
                                     c_int(T), c_int(E), c_float(gamma), c_float(lmbda), self._st()))

    # ------------------------------------------------------------------ SAC / PPO dense layers (csrc/mlp.cu)
    EPI = {"none": 0, "relu": 1, "tanh": 2, "drelu": 3, "dtanh": 4}

    def bgemm(self, A, B, C, bias=None, aux=None, rsum=None, epi: str = "none", accumulate: bool = False):
        """C[n] = epi(A[n] @ B[n] + bias[n]) for 3-D *views* A [n|1, M, K], B [n|1, K, N] (any strides: pass
        `.transpose(-1, -2)` views for the NT / TN products), C [n, M, N] (unit inner stride).  A leading dim of
        1 broadcasts the operand over the `n` networks.  rsum [n, M] (optional) receives the row sums of A."""
        _f32(A, B, C, bias, aux, rsum)
        nets, M, N = C.shape
        K = A.shape[2]
        assert A.shape[1:] == (M, K) and B.shape[1:] == (K, N) and C.stride(2) == 1, (A.shape, B.shape, C.shape)

        def ns(t):  # stride between networks (0 = shared)
            return 0 if t.shape[0] == 1 else t.stride(0)

        if aux is not None:
            assert aux.shape == C.shape and aux.stride(2) == 1
        if bias is not None:
            assert bias.shape[1] == N and (N == 1 or bias.stride(1) == 1)
        if rsum is not None:
            assert rsum.shape == (nets, M) and (M == 1 or rsum.stride(1) == 1)
        self._ck(self.lib.b200rl_bgemm(
            _p(A), c_ll(A.stride(1)), c_ll(A.stride(2)), c_ll(ns(A)), _p(B), c_ll(B.stride(1)), c_ll(B.stride(2)),
            c_ll(ns(B)), _p(C), c_ll(C.stride(1)), c_ll(ns(C)), _p(bias), c_ll(0 if bias is None else ns(bias)),
            _p(aux), c_ll(0 if aux is None else aux.stride(1)), c_ll(0 if aux is None else ns(aux)), _p(rsum),
            c_ll(0 if rsum is None else ns(rsum)), c_int(M), c_int(N), c_int(K), c_int(nets), c_int(self.EPI[epi]),
            c_int(int(accumulate)), self._st()))

    # ------------------------------------------------------------------ SAC element-wise stages (csrc/sac.cu)
    def sac_sample_fwd(self, head, eps, scale, abias, action, logp, tanh_out=None):
        """action: a [B, A] view (unit inner stride, any row stride) — e.g. the action columns of the critics' input."""
        _f32(head, eps, scale, abias, action, logp, tanh_out)
        B, A = eps.shape
        assert head.shape == (B, 2 * A) and head.is_contiguous() and eps.is_contiguous() and action.stride(1) == 1
        self._ck(self.lib.b200rl_sac_sample_fwd(_p(head), _p(eps), _p(scale), _p(abias), _p(action),
                                                c_ll(action.stride(0)), _p(logp), _p(tanh_out), c_int(B), c_int(A),
                                                self._st()))

    def sac_sample_bwd(self, head, eps, tanh_y, scale, dact, log_alpha, dhead):
        """dact: [nets, B, A] contiguous input gradients of the critics' action columns."""
        _f32(head, eps, tanh_y, scale, dact, log_alpha, dhead)
        nets, B, A = dact.shape
        assert dact.is_contiguous() and dhead.is_contiguous() and head.is_contiguous()
        self._ck(self.lib.b200rl_sac_sample_bwd(_p(head), _p(eps), _p(tanh_y), _p(scale), _p(dact), c_ll(B * A),
                                                c_int(nets), _p(log_alpha), _p(dhead), c_int(B), c_int(A), self._st()))

    def sac_target(self, q_target, logp, rewards, terminated, log_alpha, gamma: float, y):
        _f32(q_target, logp, rewards, terminated, log_alpha, y)
        nets, B = q_target.shape
        assert q_target.is_contiguous()
        self._ck(self.lib.b200rl_sac_target(_p(q_target), c_ll(B), c_int(nets), _p(logp), _p(rewards), _p(terminated),
                                            _p(log_alpha), c_float(gamma), _p(y), c_int(B), self._st()))

    def sac_critic_loss(self, q, y, dq, loss_out):
        _f32(q, y, dq, loss_out)
        nets, B = q.shape
        assert q.is_contiguous() and dq.is_contiguous()
        self._ck(self.lib.b200rl_sac_critic_loss(_p(q), c_ll(B), c_int(nets), _p(y), _p(dq), _p(loss_out), c_int(B),
                                                 self._st()))

    def sac_actor_loss(self, q, logp, log_alpha, target_entropy: float, dq, actor_loss, alpha_loss, dlog_alpha):
        _f32(q, logp, log_alpha, dq, actor_loss, alpha_loss, dlog_alpha)
        nets, B = q.shape
        assert q.is_contiguous() and dq.is_contiguous()
        self._ck(self.lib.b200rl_sac_actor_loss(_p(q), c_ll(B), c_int(nets), _p(logp), _p(log_alpha),
                                                c_float(target_entropy), _p(dq), _p(actor_loss), _p(alpha_loss),
                                                _p(dlog_alpha), c_int(B), self._st()))

    def fill_normal(self, out, seed: int, stream_id: int, counter=None):
        _f32(out)
        self._ck(self.lib.b200rl_fill_normal(_p(out), c_ll(out.numel()), ctypes.c_ulonglong(seed),
                                             ctypes.c_uint(stream_id), _p(counter), self._st()))

    # ------------------------------------------------------------------ PPO (csrc/ppo.cu)
    def im2col(self, x, col, k: int, stride: int):
        """x [B,H,W,C] channel-last -> col [B*Ho*Wo, k*k*C]"""
        _f32(x, col)
        B, H, W, C = x.shape
        assert x.is_contiguous() and col.is_contiguous()
        self._ck(self.lib.b200rl_im2col(_p(x), _p(col), c_int(B), c_int(H), c_int(W), c_int(C), c_int(k), c_int(stride),
                                        self._st()))

    def col2im(self, dcol, act, dx, k: int, stride: int):
        """dx [B,H,W,C] = scatter-sum of dcol, masked by (act > 0) when act is given"""
        _f32(dcol, act, dx)
        B, H, W, C = dx.shape
        assert dx.is_contiguous() and dcol.is_contiguous() and (act is None or act.is_contiguous())
        self._ck(self.lib.b200rl_col2im(_p(dcol), _p(act), _p(dx), c_int(B), c_int(H), c_int(W), c_int(C), c_int(k),
                                        c_int(stride), self._st()))

    def ppo_loss(self, head, actions, old_logp, adv, values, old_values, returns, dhead, dvalues, losses, head_dims,
                 is_continuous: bool, clip_vloss: bool, normalize_adv: bool, clip_coef: float, vf_coef: float,
                 ent_coef: float):
        _f32(head, actions, old_logp, adv, values, old_values, returns, dhead, dvalues, losses)
        for t in (head, actions, dhead):
            assert t.is_contiguous()
        dims = (c_int * len(head_dims))(*head_dims)
        self._ck(self.lib.b200rl_ppo_loss(_p(head), _p(actions), _p(old_logp), _p(adv), _p(values), _p(old_values),
                                          _p(returns), _p(dhead), _p(dvalues), _p(losses), c_int(head.shape[0]), dims,
                                          c_int(len(head_dims)), c_int(int(is_continuous)), c_int(int(clip_vloss)),
                                          c_int(int(normalize_adv)), c_float(clip_coef), c_float(vf_coef),
                                          c_float(ent_coef), self._st()))

    def ppo_loss_masked(self, head, actions, old_logp, adv, values, old_values, returns, mask, dhead, dvalues, losses,
                        head_dims, is_continuous: bool, clip_vloss: bool, normalize_adv: bool, clip_coef: float,
                        vf_coef: float, ent_coef: float):
        _f32(head, actions, old_logp, adv, values, old_values, returns, mask, dhead, dvalues, losses)
        for t in (head, actions, dhead, mask):
            assert t.is_contiguous()
        dims = (c_int * len(head_dims))(*head_dims)
        self._ck(self.lib.b200rl_ppo_loss_masked(_p(head), _p(actions), _p(old_logp), _p(adv), _p(values),
                                                 _p(old_values), _p(returns), _p(mask), _p(dhead), _p(dvalues),
                                                 _p(losses), c_int(head.shape[0]), dims, c_int(len(head_dims)),
                                                 c_int(int(is_continuous)), c_int(int(clip_vloss)),
                                                 c_int(int(normalize_adv)), c_float(clip_coef), c_float(vf_coef),
                                                 c_float(ent_coef), self._st()))

    # ------------------------------------------------------------------ recurrent PPO: LSTM sequences (csrc/lstm.cu)
    def lstm_seq_fwd(self, xw, W_hh, h0, c0, lengths, out, gates=None, cs=None, hT=None, cT=None):
        """xw [T,B,4H], W_hh [4H,H], h0/c0 [B,H], lengths int32 [B]; out [T,B,H]; gates/cs kept for the backward"""
        _f32(xw, W_hh, h0, c0, out, gates, cs, hT, cT)
        T, B, G = xw.shape
        H = G // 4
        assert lengths.dtype == torch.int32 and lengths.is_cuda and lengths.numel() == B
        for t in (xw, W_hh, h0, c0, lengths, out, gates, cs, hT, cT):
            assert t is None or t.is_contiguous()
        assert W_hh.shape == (G, H) and out.numel() == T * B * H and h0.numel() == B * H and c0.numel() == B * H
        self._ck(self.lib.b200rl_lstm_seq_fwd(_p(xw), _p(W_hh), _p(h0), _p(c0), _p(lengths), _p(out), _p(gates), _p(cs),
                                              _p(hT), _p(cT), c_int(T), c_int(B), c_int(H), self._st()))

    def lstm_seq_bwd(self, d_out, W_hh, gates, cs, c0, lengths, d_gates):
        _f32(d_out, W_hh, gates, cs, c0, d_gates)
        T, B, G = d_gates.shape
        H = G // 4
        assert lengths.dtype == torch.int32 and lengths.is_cuda and lengths.numel() == B
        for t in (d_out, W_hh, gates, cs, c0, lengths, d_gates):
            assert t.is_contiguous()
        self._ck(self.lib.b200rl_lstm_seq_bwd(_p(d_out), _p(W_hh), _p(gates), _p(cs), _p(c0), _p(lengths), _p(d_gates),
                                              c_int(T), c_int(B), c_int(H), self._st()))

    # ------------------------------------------------------------------ imagination: Linear([one-hot z, a]) as a gather
    def transpose2d(self, X, Y):
        """Y [cols, rows] = X [rows, cols]^T (2-D views with unit inner stride)"""
        _f32(X, Y)
        rows, cols = X.shape
        self._ck(self.lib.b200rl_transpose2d(_p(X), _p(Y), c_int(rows), c_int(cols), c_ll(_ld(X)), c_ll(_ld(Y)), self._st()))

    def onehot_linear(self, z, act, WT, out, groups: int, classes: int):
        _f32(z, act, WT, out)
        M, A, N = z.shape[0], act.shape[1], WT.shape[1]
        assert WT.is_contiguous() and WT.shape[0] == groups * classes + A and out.shape == (M, N)
        self._ck(self.lib.b200rl_onehot_linear(_p(z), _p(act), _p(WT), _p(out), c_ll(M), c_int(groups), c_int(classes),
                                               c_int(A), c_int(N), c_ll(_ld(z)), c_ll(_ld(act)), c_ll(_ld(out)), self._st()))

    def onehot_linear_ln_supported(self, WT, out, pre=None) -> bool:
        N = WT.shape[1]
        ok = 128 <= N <= 1024 and N % 128 == 0 and out.data_ptr() % 16 == 0 and _ld(out) % 4 == 0 and WT.data_ptr() % 16 == 0
        return ok and (pre is None or (pre.data_ptr() % 16 == 0 and _ld(pre) % 4 == 0))

    def onehot_linear_ln(self, z, act, WT, gamma, beta, eps: float, out, groups: int, classes: int, pre=None):
        """out = SiLU(LayerNorm(Linear([one-hot z, act]))) in one launch; `pre` (optional) keeps the Linear output."""
        _f32(z, act, WT, gamma, beta, out, pre)
        M, A, N = z.shape[0], act.shape[1], WT.shape[1]
        assert WT.is_contiguous() and WT.shape[0] == groups * classes + A and out.shape == (M, N) and N <= 1024
        self._ck(self.lib.b200rl_onehot_linear_ln(_p(z), _p(act), _p(WT), _p(gamma), _p(beta), c_float(eps), _p(pre),
                                                  c_ll(_ld(pre) if pre is not None else 0), _p(out), c_ll(M), c_int(groups),
                                                  c_int(classes), c_int(A), c_int(N), c_ll(_ld(z)), c_ll(_ld(act)),
                                                  c_ll(_ld(out)), self._st()))

    # ------------------------------------------------------------------ Dreamer-V3 continuous actions (csrc/dv3_cont.cu)
    def cont_action_fwd(self, head, eps, action, ent, min_std: float, max_std: float, init_std: float, clip: float):
        _f32(head, eps, action, ent)
        M, A = eps.shape
        assert head.shape == (M, 2 * A) and head.is_contiguous() and eps.is_contiguous()
        self._ck(self.lib.b200rl_cont_action_fwd(_p(head), _p(eps), _p(action), c_ll(_ld(action)), _p(ent), c_ll(M),
                                                 c_int(A), c_float(min_std), c_float(max_std), c_float(init_std),
                                                 c_float(clip), self._st()))

    def cont_action_bwd(self, head, eps, d_action, discount, dhead, min_std: float, max_std: float, init_std: float,
                        clip: float, ent_scale: float):
        _f32(head, eps, d_action, discount, dhead)
        M, A = eps.shape
        assert head.is_contiguous() and eps.is_contiguous() and dhead.is_contiguous() and discount.numel() >= M
        self._ck(self.lib.b200rl_cont_action_bwd(_p(head), _p(eps), _p(d_action), c_ll(_ld(d_action)), _p(discount),
                                                 _p(dhead), c_ll(M), c_int(A), c_float(min_std), c_float(max_std),
                                                 c_float(init_std), c_float(clip), c_float(ent_scale), self._st()))

    def lambda_returns_bwd(self, cont_logit, discount, moments, lam, val, ent, gamma, lmbda, ent_coef, scale, d_val,
                           d_rew, rows):
        _f32(cont_logit, discount, moments, lam, val, ent, d_val, d_rew, rows)
        H, N = lam.shape
        self._ck(self.lib.b200rl_lambda_returns_bwd(_p(cont_logit), _p(discount), _p(moments), _p(lam), _p(val), _p(ent),
                                                    _p(d_val), _p(d_rew), _p(rows), c_int(H), c_int(N), c_float(gamma),
                                                    c_float(lmbda), c_float(ent_coef), c_float(scale), self._st()))

    def twohot_mean_bwd(self, logits, d_mean, low: float, high: float, d_logits):
        _f32(logits, d_mean, d_logits)
        M, nb = logits.shape
        self._ck(self.lib.b200rl_twohot_mean_bwd(_p(logits), _p(d_mean), _p(d_logits), c_ll(M), c_int(nb),
                                                 c_ll(_ld(logits)), c_ll(_ld(d_logits)), c_float(low), c_float(high),
                                                 self._st()))

    def ppo_act(self, head, noise, actions, logp, head_dims, is_continuous: bool, greedy: bool):
        _f32(head, noise, actions, logp)
        assert head.is_contiguous() and actions.is_contiguous() and (noise is None or noise.is_contiguous())
        dims = (c_int * len(head_dims))(*head_dims)
        self._ck(self.lib.b200rl_ppo_act(_p(head), _p(noise), _p(actions), _p(logp), c_int(head.shape[0]), dims,
                                         c_int(len(head_dims)), c_int(int(is_continuous)), c_int(int(greedy)), self._st()))
