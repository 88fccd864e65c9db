"""ctypes binding of the C-ABI in `include/b200rl.h` (library: `sheeprl_b200/libb200rl.so`), typed from the header.

`CudaOps` exposes one method per entry point, taking torch tensors purely as (device pointer, shape, leading dimension)
carriers; all work is enqueued on torch's current CUDA stream.  There is NO fallback: constructing `CudaOps` without the
built library or without an sm_90 (H100) GPU raises.
"""
from __future__ import annotations

import ctypes
import os
import re
from typing import Optional, Sequence

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200rl.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "b200rl.h")

_lib = None

# Tensor-core products with at least this many rows take B as pre-split TF32 planes: one streaming split pass over B
# (12 bytes per element) in place of the kernel splitting the B tile again in every one of the M / 128 row tiles.  At
# 32 row tiles and more the pass costs a small fraction of what it saves (DESIGN.md §4, "Pre-split weight operands").
PRESPLIT_MIN_ROWS = 4096


class B200RLError(RuntimeError):
    pass


# the C scalar types the header uses; every pointer and cudaStream_t is a c_void_p, a `const char*` result a c_char_p
_SCALARS = {"int": ctypes.c_int, "long long": ctypes.c_longlong, "unsigned int": ctypes.c_uint,
            "unsigned long long": ctypes.c_ulonglong, "float": ctypes.c_float}


def _decl(text: str, where: Optional[str] = None, result: bool = False):
    """(name, ctypes type) of one declaration such as `const float* A`; `where` names it in errors (default: itself)."""
    m = re.fullmatch(r"\s*(.+?)\s*\b(\w+)\s*", text, re.S)
    if m is None:
        raise B200RLError(f"{where}: cannot parse the declaration {text.strip()!r}")
    words = m.group(1).replace("*", " * ").split()
    base = " ".join(w for w in words if w not in ("const", "*"))
    if "*" in words or base == "cudaStream_t":
        return m.group(2), ctypes.c_char_p if result and base == "char" else ctypes.c_void_p
    if base not in _SCALARS:
        raise B200RLError(f"{where or m.group(2)}: C type {m.group(1)!r} has no ctypes binding")
    return m.group(2), _SCALARS[base]


def parse_header(text: str):
    """({function: (restype, argtypes)}, {struct typedef: [(field, type)]}) of a header written like b200rl.h."""
    text = re.sub(r"/\*.*?\*/|^\s*#[^\n]*", " ", text, flags=re.S | re.M)     # comments, preprocessor lines
    structs, typedef = {}, r"typedef\s+struct\s+\w+\s*\{(.*?)\}\s*(\w+)\s*;"
    for body, name in re.findall(typedef, text, re.S):
        structs[name] = []
        for stmt in filter(str.strip, body.split(";")):              # `const float *W_in, *lnx_g`: one type, many names
            first, *more = stmt.split(",")
            base = re.match(r"\s*(.*?)[\s*]*\w+\s*$", first, re.S).group(1)
            structs[name] += [_decl(d, name) for d in [first] + [base + " " + d for d in more]]
    functions = {}
    for stmt in re.sub(typedef, " ", text, flags=re.S).split(";"):
        stmt = re.split(r"[{}]", stmt)[-1].strip()                  # drops `extern "C" {` and the closing brace
        if not stmt:
            continue
        m = re.fullmatch(r"(.+?)\((.*)\)", stmt, re.S)
        if m is None:
            raise B200RLError(f"cannot parse the declaration {stmt!r}")
        name, restype = _decl(m.group(1), result=True)
        params = m.group(2).strip()
        functions[name] = (restype, [] if params in ("", "void") else [_decl(p, name)[1] for p in params.split(",")])
    return functions, structs


with open(HEADER_PATH) as _f:
    _FUNCTIONS, _STRUCTS = parse_header(_f.read())


def _bind(fn, restype, argtypes):
    fn.restype, fn.argtypes, n = restype, argtypes, len(argtypes)

    def call(*args):
        if len(args) != n:       # ctypes refuses too few arguments but would pass extra ones on as C varargs
            raise TypeError(f"{fn.__name__} takes {n} arguments ({len(args)} given)")
        return fn(*args)

    call.__name__, call.restype, call.argtypes = fn.__name__, restype, argtypes
    return call


def load_library(path: str = LIB_PATH) -> ctypes.CDLL:
    """Loads the library and binds every declared function (no GPU needed to load; kernels need one to run)."""
    global _lib
    if _lib is None:
        if not os.path.exists(path):
            raise B200RLError(f"{path} not found: build it with `python -m sheeprl_b200.build` (nvcc, sm_90a). "
                              "The B200 engine has no CPU / PyTorch fallback.")
        lib = ctypes.CDLL(path)
        for name, (restype, argtypes) in _FUNCTIONS.items():
            setattr(lib, name, _bind(getattr(lib, name), restype, argtypes))
        _lib = lib
    return _lib


def declared_symbols() -> Sequence[str]:
    """Names of every function declared in include/b200rl.h."""
    return sorted(_FUNCTIONS)


def sync_deterministic(ops) -> bool:
    """Puts `ops` in deterministic mode when torch.are_deterministic_algorithms_enabled(), the process-wide switch the
    reference's CLI sets from `torch_use_deterministic_algorithms` (configs/config.yaml), and out of it otherwise.
    Every engine train() and player call starts with it, so a run that flips torch's switch between calls follows it.
    Backends without the setter (the CPU test doubles) are left alone.  Returns the mode."""
    on = torch.are_deterministic_algorithms_enabled()
    setter = getattr(ops, "set_deterministic", None)
    if setter is not None:
        setter(on)
    return on


def _p(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _ld(t: Optional[torch.Tensor]) -> int:
    """Row stride of a 2-D view with unit inner stride (1-D tensors are single rows); 0 for an absent tensor."""
    if t is None:
        return 0
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


def _struct(name: str, typedef: str, exclude=()):
    """Structure of a typedef of the header; POINTERS: the device tensors rssm_scan_fwd / _bwd take by name."""
    fields = _STRUCTS[typedef]
    pointers = tuple(n for n, t in fields if t is ctypes.c_void_p and n not in exclude)
    return type(name, (ctypes.Structure,), {"_fields_": fields, "POINTERS": pointers})


RssmScanArgs = _struct("RssmScanArgs", "b200rl_rssm_scan_args", exclude=("workspace",))   # passed on its own
RssmScanGrads = _struct("RssmScanGrads", "b200rl_rssm_scan_grads")
GruScanArgs = _struct("GruScanArgs", "b200rl_gru_scan_args", exclude=("workspace",))
GruScanGrads = _struct("GruScanGrads", "b200rl_gru_scan_grads")


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
        return torch.cuda.current_stream().cuda_stream

    def _ck(self, rc: int, launches: int = 1):
        """Checks the return code of an entry point that enqueues `launches` kernels."""
        self.launches += launches
        if rc != 0:
            raise B200RLError(self.lib.b200rl_last_error().decode())

    # ------------------------------------------------------------------ GEMM family
    def set_matmul_precision(self, precision: str) -> None:
        """"highest": fp32-accurate 3xTF32 products (default); "high" / "medium": one TF32 product per k-step — what
        torch.set_float32_matmul_precision("high") gives the reference on a GPU (sheeprl/configs/config.yaml:18)."""
        p = str(precision).lower()
        if p not in ("highest", "high", "medium"):
            raise ValueError(f"float32_matmul_precision must be highest / high / medium, got {precision}")
        self._ck(self.lib.b200rl_set_matmul_precision(3 if p == "highest" else 1), 0)

    def matmul_precision(self) -> str:
        return "highest" if self.lib.b200rl_get_matmul_precision() == 3 else "high"

    def set_deterministic(self, on: bool) -> None:
        """Deterministic mode of the library (process-wide): every float reduction in a fixed order, so that the same
        inputs give bit-identical outputs on the same GPU type.  Engines follow torch's switch (`sync_deterministic`)."""
        self._ck(self.lib.b200rl_set_deterministic(int(bool(on))), 0)

    def deterministic(self) -> bool:
        return bool(self.lib.b200rl_get_deterministic())

    def gemm(self, A, B, C, transA: bool, transB: bool, bias=None, accumulate: bool = False):
        _f32(A, B, C, bias)
        M, N = C.shape
        K = A.shape[0] if transA else A.shape[1]
        assert (A.shape[1] if transA else A.shape[0]) == M, (A.shape, C.shape, transA)
        assert (B.shape[0] if transB else B.shape[1]) == N and (B.shape[1] if transB else B.shape[0]) == K, \
            (A.shape, B.shape, C.shape, transA, transB)
        if (not transA and M >= PRESPLIT_MIN_ROWS and self.use_tc
                and self.lib.b200rl_gemm_tc_supported(_p(A), _p(B), M, N, K, _ld(A), _ld(B), 0, int(transB))):
            hi, lo, ld = self._planes(B, transB, N, K)
            self._ck(self.lib.b200rl_gemm_tc_presplit(_p(A), _p(hi), _p(lo), _p(C), _p(bias), M, N, K, _ld(A), ld, _ld(C),
                                                      int(accumulate), self._st()))
            return
        # every layout goes to one entry point: transposed operands are read in place as MN-major tiles
        self._ck(self.lib.b200rl_gemm_f32(_p(A), _p(B), _p(C), _p(bias), M, N, K, _ld(A), _ld(B), _ld(C), int(transA),
                                          int(transB), int(accumulate), self._st()))

    def _planes(self, B, transB: bool, N: int, K: int):
        """(hi, lo, ld): B as the K-major [N][K] TF32 planes (row stride ld) of b200rl_gemm_tc_presplit, in a workspace
        reused by consecutive products on the stream.  A [N][K] B keeps its row stride (the split runs over the whole
        strided span); a [K][N] B is split transposed, rows padded to a multiple of 4 floats."""
        ldb = _ld(B)
        ld = ldb if transB else (K + 3) // 4 * 4
        buf = self._scratch("b_planes", 2 * N * ld)
        hi, lo = buf[:N * ld], buf[N * ld:2 * N * ld]
        if transB:
            self._ck(self.lib.b200rl_tf32_split(_p(B), _p(hi), _p(lo), (N - 1) * ldb + K, self._st()))
        else:
            self._ck(self.lib.b200rl_tf32_split_t(_p(B), _p(hi), _p(lo), K, N, ldb, ld, self._st()))
        return hi, lo, ld

    def gemm_ln_supported(self, A, W, mode: int = 0) -> bool:
        M, K = A.shape
        return self.use_tc and bool(self.lib.b200rl_gemm_ln_supported(_p(A), _p(W), M, W.shape[0], K, _ld(A), _ld(W),
                                                                     mode))

    def gemm_ln_act(self, A, W, gamma, beta, eps: float, act: int, out, pre=None):
        """out = act(LayerNorm(A W^T)); `pre` (optional) receives A W^T.  Two launches (product, fused reduce + LN)."""
        _f32(A, W, gamma, beta, out, pre)
        M, K = A.shape
        N = W.shape[0]
        assert W.shape[1] == K and out.shape == (M, N)
        self._ck(self.lib.b200rl_gemm_ln(_p(A), _p(W), M, N, K, _ld(A), _ld(W), _p(gamma), _p(beta), eps, act, _p(pre),
                                         _ld(pre), _p(out), _ld(out), 0, None, 0, None, 0, None, 0, self._st()), 2)

    def gemm_ln_gru(self, A, W, gamma, beta, eps: float, h_prev, h_out, h_out2=None, g_pre=None, g_ln=None):
        """LayerNormGRUCell on [h | x] rows `A`: h_out = gate(LayerNorm(A W^T), h_prev) (models.py:396-403)."""
        _f32(A, W, gamma, beta, h_prev, h_out, h_out2, g_pre, g_ln)
        M, K = A.shape
        N = W.shape[0]
        assert W.shape[1] == K and h_prev.shape == (M, N // 3) and h_out.shape == (M, N // 3)
        self._ck(self.lib.b200rl_gemm_ln(_p(A), _p(W), M, N, K, _ld(A), _ld(W), _p(gamma), _p(beta), eps, 0, _p(g_pre),
                                         _ld(g_pre), _p(g_ln), _ld(g_ln), 1, _p(h_prev), _ld(h_prev), _p(h_out),
                                         _ld(h_out), _p(h_out2), _ld(h_out2), self._st()), 2)

    def _scratch(self, slot: str, numel: int) -> torch.Tensor:
        buf = self._scratch_bufs.get(slot)
        if buf is None or buf.numel() < numel:
            buf = torch.empty(numel, dtype=torch.float32, device=self.device)
            self._scratch_bufs[slot] = buf
        return buf

    def col_sum(self, X, out, accumulate: bool = False):
        _f32(X, out)
        self._ck(self.lib.b200rl_col_sum(_p(X), _p(out), X.shape[0], X.shape[1], _ld(X), int(accumulate), self._st()))

    def ln_act_fwd(self, X, gamma, beta, eps: float, act: int, Y):
        _f32(X, gamma, beta, Y)
        self._ck(self.lib.b200rl_ln_act_fwd(_p(X), _p(gamma), _p(beta), _p(Y), X.shape[0], X.shape[1], _ld(X), _ld(Y),
                                            eps, act, self._st()))

    def ln_act_bwd(self, X, gamma, beta, eps: float, act: int, dY, dX, dgamma, dbeta, accumulate: bool = False):
        _f32(X, gamma, beta, dY, dX, dgamma, dbeta)
        self._ck(self.lib.b200rl_ln_act_bwd(_p(X), _p(gamma), _p(beta), _p(dY), _p(dX), _p(dgamma), _p(dbeta),
                                            X.shape[0], X.shape[1], _ld(X), _ld(dY), _ld(dX), eps, act,
                                            int(accumulate), self._st()))

    # ------------------------------------------------------------------ convolutions
    def obs_prep(self, obs, out):
        assert obs.is_cuda and obs.is_contiguous() and out.is_contiguous()
        assert obs.dtype in (torch.uint8, torch.float32), obs.dtype
        NB, C, H, W = obs.shape
        self._ck(self.lib.b200rl_obs_prep(_p(obs), int(obs.dtype == torch.uint8), _p(out), NB, C, H * W, self._st()))

    def transpose_batched(self, X, Y):
        _f32(X, Y)
        assert X.is_contiguous() and Y.is_contiguous()
        NB, a, b = X.shape
        self._ck(self.lib.b200rl_transpose_batched(_p(X), _p(Y), NB, a, b, self._st()))

    def conv_down(self, big, W, small):
        _f32(big, W, small)
        assert big.is_contiguous() and small.is_contiguous() and W.is_contiguous()
        NB, h, w, Cs = small.shape
        Cb = big.shape[-1]
        assert tuple(big.shape) == (NB, 2 * h, 2 * w, Cb) and tuple(W.shape) == (Cs, Cb, 4, 4)
        if self.use_tc and self.lib.b200rl_conv_tc_supported(0, NB, h, w, Cs, Cb):
            hi, lo = self._packed(W, 0, Cs, Cb)
            self._ck(self.lib.b200rl_conv_down_tc_presplit(_p(big), _p(hi), _p(lo), _p(small), NB, h, w, Cs, Cb,
                                                           self._st()))
            return
        self._ck(self.lib.b200rl_conv_down(_p(big), _p(W), _p(small), NB, h, w, Cs, Cb, self._st()))

    def _packed(self, W, mode_up: int, Cs: int, Cb: int):
        """Tap-major copy of a conv weight for the tensor-core kernels as its TF32 hi / lo planes (caller-owned
        workspace, refreshed on every use because the optimiser rewrites W each step; 2 x 16*Cs*Cb floats, a few
        microseconds).  The split here spares the kernel splitting the weight tile again for every output tile."""
        key = (W.data_ptr(), mode_up)
        buf = self._pack_bufs.get(key)
        need = self.lib.b200rl_conv_pack_floats(mode_up, Cs, Cb)
        if buf is None or buf.shape != (2, need):
            buf = torch.empty(2, need, dtype=torch.float32, device=W.device)
            self._pack_bufs[key] = buf
        self._ck(self.lib.b200rl_conv_pack_split(_p(W), _p(buf[0]), _p(buf[1]), mode_up, Cs, Cb, self._st()))
        return buf[0], buf[1]

    def conv_up(self, small, W, big, bias=None):
        _f32(big, W, small, bias)
        assert big.is_contiguous() and small.is_contiguous() and W.is_contiguous()
        NB, h, w, Cs = small.shape
        Cb = big.shape[-1]
        assert tuple(big.shape) == (NB, 2 * h, 2 * w, Cb) and tuple(W.shape) == (Cs, Cb, 4, 4)
        if self.use_tc and self.lib.b200rl_conv_tc_supported(1, NB, h, w, Cs, Cb):
            hi, lo = self._packed(W, 1, Cs, Cb)
            self._ck(self.lib.b200rl_conv_up_tc_presplit(_p(small), _p(hi), _p(lo), _p(big), _p(bias), NB, h, w, Cs, Cb,
                                                         self._st()))
            return
        self._ck(self.lib.b200rl_conv_up(_p(small), _p(W), _p(big), _p(bias), NB, h, w, Cs, Cb, self._st()))

    def conv_wgrad(self, small, big, dW, accumulate: bool = False):
        _f32(big, dW, small)
        assert big.is_contiguous() and small.is_contiguous() and dW.is_contiguous()
        NB, h, w, Cs = small.shape
        Cb = big.shape[-1]
        assert tuple(big.shape) == (NB, 2 * h, 2 * w, Cb) and tuple(dW.shape) == (Cs, Cb, 4, 4)
        if self.use_tc and self.lib.b200rl_conv_wgrad_tc_supported(NB, h, w, Cs, Cb):
            ws = self._scratch("wgrad", self.lib.b200rl_conv_wgrad_tc_workspace(NB, h, w, Cs, Cb))
            self._ck(self.lib.b200rl_conv_wgrad_tc(_p(small), _p(big), _p(dW), _p(ws), NB, h, w, Cs, Cb,
                                                   int(accumulate), self._st()))
            return
        self._ck(self.lib.b200rl_conv_wgrad(_p(small), _p(big), _p(dW), NB, h, w, Cs, Cb, int(accumulate), self._st()))

    # ------------------------------------------------------------------ RSSM pieces
    def gru_gate_fwd(self, G, Hin, Hout):
        _f32(G, Hin, Hout)
        M, R = Hin.shape
        self._ck(self.lib.b200rl_gru_gate_fwd(_p(G), _p(Hin), _p(Hout), M, R, _ld(G), _ld(Hin), _ld(Hout), self._st()))

    def gru_gate_bwd(self, G, Hin, dH, dG, dHin):
        _f32(G, Hin, dH, dG, dHin)
        M, R = Hin.shape
        self._ck(self.lib.b200rl_gru_gate_bwd(_p(G), _p(Hin), _p(dH), _p(dG), _p(dHin), M, R, _ld(G), _ld(Hin), _ld(dH),
                                              _ld(dG), _ld(dHin), self._st()))

    def mask_mix(self, prev, init, first, out):
        _f32(prev, init, first, out)
        M, C = out.shape
        self._ck(self.lib.b200rl_mask_mix(_p(prev), _p(init), _p(first), _p(out), M, C, _ld(prev), _ld(out), self._st()))

    def mask_rows(self, X, first, out):
        self.mask_mix(X, None, first, out)

    def mask_bwd(self, dIn, first, dPrev, dInit):
        _f32(dIn, first, dPrev, dInit)
        M, C = dIn.shape
        self._ck(self.lib.b200rl_mask_bwd(_p(dIn), _p(first), _p(dPrev), _p(dInit), M, C, _ld(dIn), _ld(dPrev),
                                          self._st()))

    def cat_sample(self, raw, noise, unimix: float, groups: int, classes: int, onehot, mix_out=None):
        _f32(raw, noise, onehot, mix_out)
        M = raw.shape[0]
        if noise is not None and noise.dim() != 2:
            noise = noise.reshape(M, -1)
        self._ck(self.lib.b200rl_cat_sample(_p(raw), _p(noise), _p(onehot), _p(mix_out), M, groups, classes, _ld(raw),
                                            _ld(noise), _ld(onehot), _ld(mix_out), unimix, self._st()))

    def head_sample_supported(self, X, W) -> bool:
        return bool(self.lib.b200rl_head_sample_supported(_p(X), _p(W), X.shape[1], W.shape[0], _ld(X), _ld(W)))

    def head_sample(self, X, W, bias, noise, unimix: float, raw, onehot):
        """raw = X W^T + bias; onehot = straight-through categorical sample of unimix(raw) — one launch."""
        _f32(X, W, bias, noise, raw, onehot)
        M, Kin = X.shape
        A = W.shape[0]
        assert raw.shape == (M, A) and onehot.shape == (M, A) and W.shape[1] == Kin
        self._ck(self.lib.b200rl_head_sample(_p(X), _p(W), _p(bias), _p(noise), _p(raw), _p(onehot), M, Kin, A, _ld(X),
                                             _ld(W), _ld(raw), _ld(noise), _ld(onehot), unimix, self._st()))

    def cat_sample_bwd(self, raw, dz, dmix, unimix: float, groups: int, classes: int, draw):
        _f32(raw, dz, dmix, draw)
        self._ck(self.lib.b200rl_cat_sample_bwd(_p(raw), _p(dz), _p(dmix), _p(draw), raw.shape[0], groups, classes,
                                                _ld(raw), _ld(dz), _ld(dmix), _ld(draw), unimix, self._st()))

    def kl_loss_grad(self, post_mix, prior_mix, groups, classes, kl_dyn, kl_rep, free_nats, regularizer, scale,
                     d_post, d_prior, rows):
        _f32(post_mix, prior_mix, d_post, d_prior, rows)
        assert rows.is_contiguous() and rows.shape[1] == 4
        self._ck(self.lib.b200rl_kl_loss_grad(_p(post_mix), _p(prior_mix), _p(d_post), _p(d_prior), _p(rows),
                                              post_mix.shape[0], groups, classes, _ld(post_mix), _ld(prior_mix),
                                              _ld(d_post), _ld(d_prior), kl_dyn, kl_rep, free_nats, regularizer, scale,
                                              self._st()))

    # ------------------------------------------------------------------ losses
    def mse_loss_grad(self, pred, target, scale: float, loss_row, grad):
        _f32(pred, target, loss_row, grad)
        assert pred.is_contiguous() and target.is_contiguous() and grad.is_contiguous()
        M, P = pred.shape
        self._ck(self.lib.b200rl_mse_loss_grad(_p(pred), _p(target), _p(loss_row), _p(grad), M, P, scale, self._st()))

    def twohot_loss_grad(self, logits, x, weight, scale, low, high, loss_row, dlogits, accumulate: bool = False):
        _f32(logits, x, weight, loss_row, dlogits)
        M, nb = logits.shape
        assert x.numel() == M and x.is_contiguous()
        self._ck(self.lib.b200rl_twohot_loss_grad(_p(logits), _p(x), _p(weight), _p(loss_row), _p(dlogits), M, nb,
                                                  _ld(logits), _ld(dlogits), low, high, scale, int(accumulate),
                                                  self._st()))

    def bce_loss_grad(self, logit, target, loss_scale, scale, loss_row, dlogit):
        _f32(logit, target, loss_row, dlogit)
        assert logit.is_contiguous() and target.is_contiguous() and dlogit.is_contiguous()
        self._ck(self.lib.b200rl_bce_loss_grad(_p(logit), _p(target), _p(loss_row), _p(dlogit), logit.numel(),
                                               loss_scale, scale, self._st()))

    def twohot_mean(self, logits, low, high, out):
        _f32(logits, out)
        self._ck(self.lib.b200rl_twohot_mean(_p(logits), _p(out), logits.shape[0], logits.shape[1], _ld(logits), low,
                                             high, self._st()))

    def lambda_returns(self, rew, val, cont_logit, true_cont, gamma, lmbda, lam, discount):
        _f32(rew, val, cont_logit, true_cont, lam, discount)
        for t in (rew, val, cont_logit, lam, discount):
            assert t.is_contiguous()
        H, N = lam.shape
        self._ck(self.lib.b200rl_lambda_returns(_p(rew), _p(val), _p(cont_logit), _p(true_cont), _p(lam), _p(discount),
                                                H, N, gamma, lmbda, self._st()))

    def moments_update(self, x, state, decay, max_, p_low, p_high, out):
        _f32(x, state, out)
        assert x.is_contiguous()
        self._ck(self.lib.b200rl_moments_update(_p(x), x.numel(), _p(state), _p(out), decay, max_, p_low, p_high,
                                                self._st()))

    def actor_loss_grad(self, raw, actions, lam, val, discount, moments, head_dims, unimix, ent_coef, scale, rows,
                        draw):
        _f32(raw, actions, lam, val, discount, moments, rows, draw)
        for t in (raw, actions, draw):
            assert t.is_contiguous()
        hd = (ctypes.c_int * len(head_dims))(*[int(x) for x in head_dims])
        self._ck(self.lib.b200rl_actor_loss_grad(_p(raw), _p(actions), _p(lam), _p(val), _p(discount), _p(moments),
                                                 _p(rows), _p(draw), raw.shape[0], hd, len(head_dims), unimix, ent_coef,
                                                 scale, self._st()))

    def sum_rows(self, X, out, scale: float):
        _f32(X, out)
        self._ck(self.lib.b200rl_sum_rows(_p(X), _p(out), X.shape[0], X.shape[1], _ld(X), scale, self._st()))

    def weighted_mean(self, x, w, scale: float, out):
        _f32(x, w, out)
        self._ck(self.lib.b200rl_weighted_mean(_p(x), _p(w), _p(out), x.numel(), scale, self._st()))

    # ------------------------------------------------------------------ optimiser / utilities
    def sumsq(self, x, out):
        assert out.dtype == torch.float64 and x.is_contiguous()
        self._ck(self.lib.b200rl_sumsq(_p(x), x.numel(), _p(out), self._st()))

    def adam_step(self, p, g, m, v, normsq, max_norm, lr, b1, b2, eps, step_t, norm_out, weight_decay=0.0):
        """clip + torch.optim.Adam; weight_decay is torch's L2 term, added to the clipped gradient"""
        _f32(p, g, m, v, norm_out)
        assert step_t.dtype == torch.int32 and normsq.dtype == torch.float64
        self._ck(self.lib.b200rl_adam_step_wd(_p(p), _p(g), _p(m), _p(v), _p(normsq), _p(step_t), _p(norm_out),
                                              p.numel(), max_norm, lr, b1, b2, eps, weight_decay, self._st()))

    def rmsprop_step(self, p, g, square_avg, momentum_buf, grad_avg, normsq, max_norm, lr, alpha, eps, weight_decay,
                     momentum, norm_out):
        """clip + torch.optim.RMSprop; momentum_buf is used when momentum > 0, grad_avg (not None) selects centered"""
        _f32(p, g, square_avg, momentum_buf, grad_avg, norm_out)
        assert normsq.dtype == torch.float64
        for t in (g, square_avg, momentum_buf, grad_avg):
            assert t is None or t.numel() == p.numel()
        self._ck(self.lib.b200rl_rmsprop_step(_p(p), _p(g), _p(square_avg), _p(momentum_buf), _p(grad_avg), _p(normsq),
                                              _p(norm_out), p.numel(), max_norm, lr, alpha, eps, weight_decay, momentum,
                                              self._st()))

    def ema(self, target, src, tau: float):
        _f32(target, src)
        self._ck(self.lib.b200rl_ema(_p(target), _p(src), target.numel(), tau, self._st()))

    def fill_exponential(self, out, seed: int, stream_id: int, counter=None):
        """Exp(1) noise from Philox4x32-10 keyed by (seed, stream_id, *counter); `counter` is a device int32
        incremented once per train step so that graph replays draw fresh noise."""
        _f32(out)
        assert out.is_contiguous()
        self._ck(self.lib.b200rl_fill_exponential(_p(out), out.numel(), seed, stream_id, _p(counter), self._st()))

    def increment(self, step_t):
        self._ck(self.lib.b200rl_increment(_p(step_t), self._st()))

    def zero(self, x):
        assert x.is_contiguous()
        if x.dtype == torch.float32:
            self._ck(self.lib.b200rl_zero(_p(x), x.numel(), self._st()))
        else:
            x.zero_()

    def copy(self, src, dst):
        _f32(src, dst)
        if src.dim() == 1:
            src, dst = src.view(1, -1), dst.view(1, -1)
        M, C = src.shape
        self._ck(self.lib.b200rl_copy2d(_p(src), _p(dst), M, C, _ld(src), _ld(dst), self._st()))

    def axpy(self, x, y, alpha: float = 1.0):
        _f32(x, y)
        assert x.is_contiguous() and y.is_contiguous()
        self._ck(self.lib.b200rl_axpy(_p(x), _p(y), x.numel(), alpha, self._st()))

    def affine(self, x, out, alpha: float, beta: float):
        _f32(x, out)
        assert x.is_contiguous() and out.is_contiguous()
        self._ck(self.lib.b200rl_affine(_p(x), _p(out), x.numel(), alpha, beta, self._st()))

    def symlog(self, x, y):
        """y[M,C] = symlog(x[M,C]); both may be column slices of wider buffers"""
        _f32(x, y)
        M, C = x.shape
        assert tuple(y.shape) == (M, C)
        self._ck(self.lib.b200rl_symlog(_p(x), _p(y), M, C, _ld(x), _ld(y), self._st()))

    def tanh_fwd(self, x, y):
        _f32(x, y)
        self._ck(self.lib.b200rl_tanh_fwd(_p(x), _p(y), x.numel(), self._st()))

    def tanh_bwd(self, y, dy, dx, accumulate: bool = False):
        _f32(y, dy, dx)
        self._ck(self.lib.b200rl_tanh_bwd(_p(y), _p(dy), _p(dx), y.numel(), int(accumulate), self._st()))

    # ------------------------------------------------------------------ persistent RSSM scan
    def rssm_scan_workspace(self, T: int, B: int, S: int, D: int, Dx: int, R: int, Dr: int) -> torch.Tensor:
        n = self.lib.b200rl_rssm_scan_workspace_bytes(T, B, S, D, Dx, R, Dr)
        return torch.zeros((n + 3) // 4, dtype=torch.int32, device=self.device)

    @staticmethod
    def _scan_dims(dims: dict) -> RssmScanArgs:
        return RssmScanArgs(**{k: int(dims[k]) for k, t in RssmScanArgs._fields_ if t is ctypes.c_int})

    def _scan_args(self, dims: dict, eps: float, unimix: float, tensors: dict, workspace: torch.Tensor):
        a = self._scan_dims(dims)
        a.eps, a.unimix = float(eps), float(unimix)
        for name in RssmScanArgs.POINTERS:
            t = tensors[name]
            assert t.is_cuda and t.dtype == torch.float32, name
            setattr(a, name, t.data_ptr())
        a.workspace, a.workspace_bytes = workspace.data_ptr(), workspace.numel() * workspace.element_size()
        return a

    def rssm_scan_fwd(self, dims: dict, eps: float, unimix: float, tensors: dict, workspace: torch.Tensor):
        """dims: the int fields of `b200rl_rssm_scan_args` (include/b200rl.h); tensors: name -> device tensor for every
        pointer field but the workspace (RssmScanArgs.POINTERS)."""
        a = self._scan_args(dims, eps, unimix, tensors, workspace)
        self._ck(self.lib.b200rl_rssm_scan_fwd(ctypes.byref(a), self._st()))

    def rssm_scan_supported(self, dims: dict, backward: bool) -> bool:
        """whether the forward / backward kernel runs a model of these dims (`rssm_scan_fwd`'s keys); launches nothing"""
        return self.lib.b200rl_rssm_scan_check(ctypes.byref(self._scan_dims(dims)), int(backward)) == 0

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
        return self.lib.b200rl_rssm_scan_error(_p(workspace), self._st())

    def rssm_scan_profile(self, workspace: torch.Tensor):
        """per-phase cycle counters of CTA 0 and CTA 1 of the last scan launch: [2][32] int64"""
        out = (ctypes.c_longlong * 64)()
        self._ck(self.lib.b200rl_rssm_scan_profile(_p(workspace), out, self._st()), 0)
        return [list(out[:32]), list(out[32:])]

    # ------------------------------------------------------------------ persistent GRU-only scan (decoupled RSSM)
    def gru_scan_workspace(self, T: int, B: int, R: int) -> torch.Tensor:
        n = self.lib.b200rl_gru_scan_workspace_bytes(T, B, R)
        return torch.zeros((n + 3) // 4, dtype=torch.int32, device=self.device)

    @staticmethod
    def _gru_scan_dims(dims: dict) -> GruScanArgs:
        return GruScanArgs(**{k: int(dims[k]) for k, t in GruScanArgs._fields_ if t is ctypes.c_int})

    def _gru_scan_args(self, dims: dict, eps: float, tensors: dict, workspace: torch.Tensor) -> GruScanArgs:
        a = self._gru_scan_dims(dims)
        a.eps = float(eps)
        for name in GruScanArgs.POINTERS:
            t = tensors[name]
            assert t.is_cuda and t.dtype == torch.float32, name
            assert name in ("W_g", "latent") or t.is_contiguous(), name     # those two carry their leading dimension
            setattr(a, name, t.data_ptr())
        assert _ld(tensors["W_g"]) == a.ld_wg and _ld(tensors["latent"]) == a.ld_lat
        a.workspace, a.workspace_bytes = workspace.data_ptr(), workspace.numel() * workspace.element_size()
        return a

    def gru_scan_supported(self, dims: dict, backward: bool) -> bool:
        """whether the forward / backward kernel runs these dims (the int fields of `b200rl_gru_scan_args`); launches
        nothing"""
        return self.lib.b200rl_gru_scan_check(ctypes.byref(self._gru_scan_dims(dims)), int(backward)) == 0

    def gru_scan_fwd(self, dims: dict, eps: float, tensors: dict, workspace: torch.Tensor):
        """tensors: name -> device tensor for every pointer field but the workspace (GruScanArgs.POINTERS)"""
        a = self._gru_scan_args(dims, eps, tensors, workspace)
        self._ck(self.lib.b200rl_gru_scan_fwd(ctypes.byref(a), self._st()))

    def gru_scan_bwd(self, dims: dict, eps: float, tensors: dict, grads: dict, workspace: torch.Tensor):
        a = self._gru_scan_args(dims, eps, tensors, workspace)
        q = GruScanGrads()
        for name in GruScanGrads.POINTERS:
            t = grads[name]
            assert t.is_cuda and t.dtype == torch.float32, name
            assert name == "d_latent" or t.is_contiguous(), name
            setattr(q, name, t.data_ptr())
        assert _ld(grads["d_latent"]) == a.ld_lat
        self._ck(self.lib.b200rl_gru_scan_bwd(ctypes.byref(a), ctypes.byref(q), self._st()))

    # ------------------------------------------------------------------ replay / PPO
    def replay_gather(self, storage, idx, out, n_samples: int, batch: int, seq_len: int):
        assert storage.is_contiguous() and out.is_contiguous() and idx.dtype == torch.int64 and idx.is_contiguous()
        row_bytes = storage[0].numel() * storage.element_size()
        self._ck(self.lib.b200rl_replay_gather(_p(storage), _p(idx), _p(out), n_samples, batch, seq_len, row_bytes,
                                               self._st()))

    def replay_scatter(self, src, dst_rows, storage):
        assert storage.is_contiguous() and src.is_contiguous() and dst_rows.dtype == torch.int64
        row_bytes = storage[0].numel() * storage.element_size()
        self._ck(self.lib.b200rl_replay_scatter(_p(src), _p(dst_rows), _p(storage), dst_rows.numel(), row_bytes,
                                                self._st()))

    def gae(self, rewards, values, dones, next_value, gamma, lmbda, returns, advantages):
        _f32(rewards, values, dones, next_value, returns, advantages)
        T, E = rewards.shape[0], rewards[0].numel()
        self._ck(self.lib.b200rl_gae(_p(rewards), _p(values), _p(dones), _p(next_value), _p(returns), _p(advantages),
                                     T, E, gamma, lmbda, self._st()))

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

        def ns(t):  # stride between networks (0 = shared or absent)
            return 0 if t is None or t.shape[0] == 1 else t.stride(0)

        if aux is not None:
            assert aux.shape == C.shape and aux.stride(2) == 1
        if bias is not None:
            assert bias.shape[1] == N and (N == 1 or bias.stride(1) == 1)
        if rsum is not None:
            assert rsum.shape == (nets, M) and (M == 1 or rsum.stride(1) == 1)
        self._ck(self.lib.b200rl_bgemm(_p(A), A.stride(1), A.stride(2), ns(A), _p(B), B.stride(1), B.stride(2), ns(B),
                                       _p(C), C.stride(1), ns(C), _p(bias), ns(bias), _p(aux),
                                       0 if aux is None else aux.stride(1), ns(aux), _p(rsum), ns(rsum), M, N, K, nets,
                                       self.EPI[epi], int(accumulate), self._st()))

    # ------------------------------------------------------------------ SAC element-wise stages (csrc/sac.cu)
    def sac_sample_fwd(self, head, eps, scale, abias, action, logp, tanh_out=None):
        """action: a [B, A] view (unit inner stride, any row stride) — e.g. the action columns of the critics' input."""
        _f32(head, eps, scale, abias, action, logp, tanh_out)
        B, A = eps.shape
        assert head.shape == (B, 2 * A) and head.is_contiguous() and eps.is_contiguous() and action.stride(1) == 1
        self._ck(self.lib.b200rl_sac_sample_fwd(_p(head), _p(eps), _p(scale), _p(abias), _p(action), action.stride(0),
                                                _p(logp), _p(tanh_out), B, A, self._st()))

    def sac_sample_bwd(self, head, eps, tanh_y, scale, dact, log_alpha, dhead):
        """dact: [nets, B, A] contiguous input gradients of the critics' action columns."""
        _f32(head, eps, tanh_y, scale, dact, log_alpha, dhead)
        nets, B, A = dact.shape
        assert dact.is_contiguous() and dhead.is_contiguous() and head.is_contiguous()
        self._ck(self.lib.b200rl_sac_sample_bwd(_p(head), _p(eps), _p(tanh_y), _p(scale), _p(dact), B * A, nets,
                                                _p(log_alpha), _p(dhead), B, A, self._st()))

    def sac_target(self, q_target, logp, rewards, terminated, log_alpha, gamma: float, y):
        _f32(q_target, logp, rewards, terminated, log_alpha, y)
        nets, B = q_target.shape
        assert q_target.is_contiguous()
        self._ck(self.lib.b200rl_sac_target(_p(q_target), B, nets, _p(logp), _p(rewards), _p(terminated), _p(log_alpha),
                                            gamma, _p(y), B, self._st()))

    def sac_critic_loss(self, q, y, dq, loss_out):
        _f32(q, y, dq, loss_out)
        nets, B = q.shape
        assert q.is_contiguous() and dq.is_contiguous()
        self._ck(self.lib.b200rl_sac_critic_loss(_p(q), B, nets, _p(y), _p(dq), _p(loss_out), B, self._st()))

    def sac_actor_loss(self, q, logp, log_alpha, target_entropy: float, dq, actor_loss, alpha_loss, dlog_alpha):
        _f32(q, logp, log_alpha, dq, actor_loss, alpha_loss, dlog_alpha)
        nets, B = q.shape
        assert q.is_contiguous() and dq.is_contiguous()
        self._ck(self.lib.b200rl_sac_actor_loss(_p(q), B, nets, _p(logp), _p(log_alpha), target_entropy, _p(dq),
                                                _p(actor_loss), _p(alpha_loss), _p(dlog_alpha), B, self._st()))

    def fill_normal(self, out, seed: int, stream_id: int, counter=None):
        _f32(out)
        self._ck(self.lib.b200rl_fill_normal(_p(out), out.numel(), seed, stream_id, _p(counter), self._st()))

    # ------------------------------------------------------------------ DroQ critics (csrc/droq.cu)
    def droq_actor_loss(self, q, logp, log_alpha, target_entropy: float, dq, actor_loss, alpha_loss, dlog_alpha):
        """sac_actor_loss with the mean over the critics in place of the min"""
        _f32(q, logp, log_alpha, dq, actor_loss, alpha_loss, dlog_alpha)
        nets, B = q.shape
        assert q.is_contiguous() and dq.is_contiguous()
        self._ck(self.lib.b200rl_droq_actor_loss(_p(q), B, nets, _p(logp), _p(log_alpha), target_entropy, _p(dq),
                                                 _p(actor_loss), _p(alpha_loss), _p(dlog_alpha), B, self._st()))

    def dropout_mask(self, mask, p: float, seed: int, stream_id: int, counter=None):
        """mask: int32 words, bit-packed keep masks (`[..., ceil(H/32)]` per [..., H] activation)"""
        assert mask.dtype == torch.int32 and mask.is_cuda and mask.is_contiguous()
        self._ck(self.lib.b200rl_dropout_mask(_p(mask), mask.numel(), p, seed, stream_id, _p(counter), self._st()))

    def dropout_ln_relu_supported(self, H: int) -> bool:
        return bool(self.lib.b200rl_dropout_ln_relu_supported(H))

    @staticmethod
    def _dln_args(z, mask, gamma, stats):
        nets, B, H = z.shape
        assert z.is_contiguous() and stats.is_contiguous() and stats.shape == (nets, B, 2)
        assert gamma.shape == (nets, H) and (H == 1 or gamma.stride(1) == 1)
        if mask is not None:
            assert mask.dtype == torch.int32 and mask.is_contiguous() and mask.shape == (nets, B, (H + 31) // 32)
        return nets, B, H, (gamma.stride(0) if nets > 1 else H)

    def dropout_ln_relu_fwd(self, z, mask, p: float, gamma, beta, eps: float, y, stats):
        """y = relu(LayerNorm(z * mask / (1-p))) for all critics; z, y [n, B, H]; gamma / beta [n, H] strided views"""
        _f32(z, gamma, beta, y, stats)
        nets, B, H, sp = self._dln_args(z, mask, gamma, stats)
        assert y.shape == z.shape and y.is_contiguous() and beta.stride() == gamma.stride()
        self._ck(self.lib.b200rl_dropout_ln_relu_fwd(_p(z), _p(mask), p, _p(gamma), _p(beta), sp, eps, _p(y), _p(stats),
                                                     nets, B, H, self._st()))

    def dropout_ln_relu_bwd(self, dy, y, z, mask, p: float, stats, gamma, dz, dgamma=None, dbeta=None):
        _f32(dy, y, z, stats, gamma, dz, dgamma, dbeta)
        nets, B, H, sp = self._dln_args(z, mask, gamma, stats)
        for t in (dy, y, dz):
            assert t.shape == z.shape and t.is_contiguous()
        for t in (dgamma, dbeta):
            assert t is None or t.stride() == gamma.stride()
        self._ck(self.lib.b200rl_dropout_ln_relu_bwd(_p(dy), _p(y), _p(z), _p(mask), p, _p(stats), _p(gamma), sp,
                                                     _p(dz), _p(dgamma), _p(dbeta), nets, B, H, self._st()))

    # ------------------------------------------------------------------ PPO (csrc/ppo.cu)
    def im2col(self, x, col, k: int, stride: int):
        """x [B,H,W,C] channel-last -> col [B*Ho*Wo, k*k*C]"""
        _f32(x, col)
        B, H, W, C = x.shape
        assert x.is_contiguous() and col.is_contiguous()
        self._ck(self.lib.b200rl_im2col(_p(x), _p(col), B, H, W, C, k, stride, self._st()))

    def col2im(self, dcol, act, dx, k: int, stride: int):
        """dx [B,H,W,C] = scatter-sum of dcol, masked by (act > 0) when act is given"""
        _f32(dcol, act, dx)
        B, H, W, C = dx.shape
        assert dx.is_contiguous() and dcol.is_contiguous() and (act is None or act.is_contiguous())
        self._ck(self.lib.b200rl_col2im(_p(dcol), _p(act), _p(dx), B, H, W, C, k, stride, self._st()))

    def ppo_loss(self, head, actions, old_logp, adv, values, old_values, returns, dhead, dvalues, losses, head_dims,
                 is_continuous: bool, clip_vloss: bool, normalize_adv: bool, clip_coef: float, vf_coef: float,
                 ent_coef: float):
        _f32(head, actions, old_logp, adv, values, old_values, returns, dhead, dvalues, losses)
        for t in (head, actions, dhead):
            assert t.is_contiguous()
        dims = (ctypes.c_int * len(head_dims))(*head_dims)
        self._ck(self.lib.b200rl_ppo_loss(_p(head), _p(actions), _p(old_logp), _p(adv), _p(values), _p(old_values),
                                          _p(returns), _p(dhead), _p(dvalues), _p(losses), head.shape[0], dims,
                                          len(head_dims), int(is_continuous), int(clip_vloss), int(normalize_adv),
                                          clip_coef, vf_coef, ent_coef, self._st()))

    def ppo_loss_masked(self, head, actions, old_logp, adv, values, old_values, returns, mask, dhead, dvalues, losses,
                        head_dims, is_continuous: bool, clip_vloss: bool, normalize_adv: bool, clip_coef: float,
                        vf_coef: float, ent_coef: float):
        _f32(head, actions, old_logp, adv, values, old_values, returns, mask, dhead, dvalues, losses)
        for t in (head, actions, dhead, mask):
            assert t.is_contiguous()
        dims = (ctypes.c_int * len(head_dims))(*head_dims)
        self._ck(self.lib.b200rl_ppo_loss_masked(_p(head), _p(actions), _p(old_logp), _p(adv), _p(values),
                                                 _p(old_values), _p(returns), _p(mask), _p(dhead), _p(dvalues),
                                                 _p(losses), head.shape[0], dims, len(head_dims), int(is_continuous),
                                                 int(clip_vloss), int(normalize_adv), clip_coef, vf_coef, ent_coef,
                                                 self._st()))

    def a2c_loss(self, head, actions, adv, values, returns, dhead, dvalues, losses, seg: int, head_dims,
                 is_continuous: int, normalize_adv: bool, reduce_sum: bool, vf_coef: float, ent_coef: float):
        """A2C objective of every minibatch (rows [i*seg, min(N, (i+1)*seg))) of a rollout; losses [n_seg, 3]"""
        _f32(head, actions, adv, values, returns, dhead, dvalues, losses)
        for t in (head, actions, adv, values, returns, dhead, dvalues, losses):
            assert t.is_contiguous()
        N = head.shape[0]
        assert losses.numel() == 3 * ((N + seg - 1) // seg)
        dims = (ctypes.c_int * len(head_dims))(*head_dims)
        self._ck(self.lib.b200rl_a2c_loss(_p(head), _p(actions), _p(adv), _p(values), _p(returns), _p(dhead),
                                          _p(dvalues), _p(losses), N, seg, dims, len(head_dims), int(is_continuous),
                                          int(normalize_adv), int(reduce_sum), vf_coef, ent_coef, self._st()))

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
                                              _p(hT), _p(cT), T, B, H, self._st()))

    def lstm_seq_bwd(self, d_out, W_hh, gates, cs, c0, lengths, d_gates):
        _f32(d_out, W_hh, gates, cs, c0, d_gates)
        T, B, G = d_gates.shape
        H = G // 4
        assert lengths.dtype == torch.int32 and lengths.is_cuda and lengths.numel() == B
        for t in (d_out, W_hh, gates, cs, c0, lengths, d_gates):
            assert t.is_contiguous()
        self._ck(self.lib.b200rl_lstm_seq_bwd(_p(d_out), _p(W_hh), _p(gates), _p(cs), _p(c0), _p(lengths), _p(d_gates),
                                              T, B, H, self._st()))

    # ------------------------------------------------------------------ imagination: Linear([one-hot z, a]) as a gather
    def transpose2d(self, X, Y):
        """Y [cols, rows] = X [rows, cols]^T (2-D views with unit inner stride)"""
        _f32(X, Y)
        rows, cols = X.shape
        self._ck(self.lib.b200rl_transpose2d(_p(X), _p(Y), rows, cols, _ld(X), _ld(Y), self._st()))

    def onehot_linear_supported(self, groups: int, classes: int, A: int, N: int) -> bool:
        """whether `onehot_linear` runs [groups * classes + A] -> N (groups and action columns are limited)"""
        return bool(self.lib.b200rl_onehot_linear_supported(groups, classes, A, N))

    def onehot_linear(self, z, act, WT, out, groups: int, classes: int):
        _f32(z, act, WT, out)
        M, A, N = z.shape[0], act.shape[1], WT.shape[1]
        assert WT.is_contiguous() and WT.shape[0] == groups * classes + A and out.shape == (M, N)
        self._ck(self.lib.b200rl_onehot_linear(_p(z), _p(act), _p(WT), _p(out), M, groups, classes, A, N, _ld(z),
                                               _ld(act), _ld(out), self._st()))

    def onehot_linear_ln_supported(self, WT, out, pre=None) -> bool:
        """whether `onehot_linear_ln` takes these operands, for dims `onehot_linear_supported` accepts"""
        return bool(self.lib.b200rl_onehot_linear_ln_supported(_p(WT), None, None, _p(out), _p(pre), WT.shape[1],
                                                               _ld(out), _ld(pre)))

    def onehot_linear_ln(self, z, act, WT, gamma, beta, eps: float, out, groups: int, classes: int, pre=None):
        """out = SiLU(LayerNorm(Linear([one-hot z, act]))) in one launch; `pre` (optional) keeps the Linear output."""
        _f32(z, act, WT, gamma, beta, out, pre)
        M, A, N = z.shape[0], act.shape[1], WT.shape[1]
        assert WT.is_contiguous() and WT.shape[0] == groups * classes + A and out.shape == (M, N)
        self._ck(self.lib.b200rl_onehot_linear_ln(_p(z), _p(act), _p(WT), _p(gamma), _p(beta), eps, _p(pre), _ld(pre),
                                                  _p(out), M, groups, classes, A, N, _ld(z), _ld(act), _ld(out),
                                                  self._st()))

    # ------------------------------------------------------------------ Dreamer-V3 continuous actions (csrc/dv3_cont.cu)
    def cont_action_fwd(self, head, eps, action, ent, min_std: float, max_std: float, init_std: float, clip: float):
        _f32(head, eps, action, ent)
        M, A = eps.shape
        assert head.shape == (M, 2 * A) and head.is_contiguous() and eps.is_contiguous()
        self._ck(self.lib.b200rl_cont_action_fwd(_p(head), _p(eps), _p(action), _ld(action), _p(ent), M, A, min_std,
                                                 max_std, init_std, clip, self._st()))

    def cont_action_bwd(self, head, eps, d_action, discount, dhead, min_std: float, max_std: float, init_std: float,
                        clip: float, ent_scale: float):
        _f32(head, eps, d_action, discount, dhead)
        M, A = eps.shape
        assert head.is_contiguous() and eps.is_contiguous() and dhead.is_contiguous() and discount.numel() >= M
        self._ck(self.lib.b200rl_cont_action_bwd(_p(head), _p(eps), _p(d_action), _ld(d_action), _p(discount),
                                                 _p(dhead), M, A, min_std, max_std, init_std, clip, ent_scale,
                                                 self._st()))

    def lambda_returns_bwd(self, cont_logit, discount, moments, lam, val, ent, gamma, lmbda, ent_coef, scale, d_val,
                           d_rew, rows):
        _f32(cont_logit, discount, moments, lam, val, ent, d_val, d_rew, rows)
        H, N = lam.shape
        self._ck(self.lib.b200rl_lambda_returns_bwd(_p(cont_logit), _p(discount), _p(moments), _p(lam), _p(val), _p(ent),
                                                    _p(d_val), _p(d_rew), _p(rows), H, N, gamma, lmbda, ent_coef, scale,
                                                    self._st()))

    def twohot_mean_bwd(self, logits, d_mean, low: float, high: float, d_logits):
        _f32(logits, d_mean, d_logits)
        M, nb = logits.shape
        self._ck(self.lib.b200rl_twohot_mean_bwd(_p(logits), _p(d_mean), _p(d_logits), M, nb, _ld(logits), _ld(d_logits),
                                                 low, high, self._st()))

    def ppo_act(self, head, noise, actions, logp, head_dims, is_continuous: bool, greedy: bool):
        _f32(head, noise, actions, logp)
        assert head.is_contiguous() and actions.is_contiguous() and (noise is None or noise.is_contiguous())
        dims = (ctypes.c_int * len(head_dims))(*head_dims)
        self._ck(self.lib.b200rl_ppo_act(_p(head), _p(noise), _p(actions), _p(logp), head.shape[0], dims,
                                         len(head_dims), int(is_continuous), int(greedy), self._st()))
