"""Times gemm_tc_kernel alone on the step's main product shapes (CUDA events, L2-sized operands rotate through 4 buffers).
Products with a non-transposed A are timed twice: with raw B (split per tile in the kernel) and with B given as its
pre-split TF32 planes (the weight-operand route; a [K][N] B becomes the transposed planes of the input gradient).

    python tools/gemm_bench.py [--json out.json]
"""
import argparse, ctypes, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from sheeprl_b200.lib import CudaOps


def _vp(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def planes(cu, B, transB):
    """(hi, lo, ld) of B as the [N][K] TF32 planes the pre-split product reads"""
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    if transB:
        hi, lo = torch.empty_like(B), torch.empty_like(B)
        assert cu.lib.b200rl_tf32_split(_vp(B), _vp(hi), _vp(lo), B.numel(), st) == 0
        return hi, lo, B.shape[1]
    K, N = B.shape
    ld = (K + 3) // 4 * 4
    hi, lo = torch.empty(N, ld, device=B.device), torch.empty(N, ld, device=B.device)
    assert cu.lib.b200rl_tf32_split_t(_vp(B), _vp(hi), _vp(lo), K, N, N, ld, st) == 0
    return hi, lo, ld


def gemm_presplit(cu, A, P, C):
    hi, lo, ld = P
    M, K = A.shape
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = cu.lib.b200rl_gemm_tc_presplit(_vp(A), _vp(hi), _vp(lo), _vp(C), None, M, C.shape[1], K, K, ld, C.shape[1], 0, st)
    assert rc == 0, cu.lib.b200rl_last_error().decode()

SHAPES = [  # M, N, K, transA, transB  (C[M,N] = op(A) op(B))
    (16384, 512, 1536, False, True), (16384, 512, 512, False, True), (1024, 1536, 1024, False, True),
    (1024, 512, 512, False, True), (15360, 1536, 512, False, False), (512, 1536, 15360, True, False),
    (4096, 12288, 5120, False, True), (65536, 1024, 5120, False, True), (65536, 1024, 1024, False, True),
    (64, 12288, 4096, False, True),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    cu = CudaOps("cuda")
    out = []
    for prec in ("highest", "high"):
        cu.set_matmul_precision(prec)
        for M, N, K, tA, tB in SHAPES:
            nbuf = 4
            As = [torch.randn((K, M) if tA else (M, K), device="cuda") for _ in range(nbuf)]
            Bs = [torch.randn((N, K) if tB else (K, N), device="cuda") for _ in range(nbuf)]
            C = torch.empty(M, N, device="cuda")
            routes = [("raw", lambda i: cu.gemm(As[i % nbuf], Bs[i % nbuf], C, tA, tB))]
            if not tA:
                Ps = [planes(cu, B, tB) for B in Bs]
                routes.append(("presplit", lambda i: gemm_presplit(cu, As[i % nbuf], Ps[i % nbuf], C)))
            for route, fn in routes:
                for i in range(3):
                    fn(i)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                for i in range(a.reps):
                    fn(i)
                e1.record()
                torch.cuda.synchronize()
                us = e0.elapsed_time(e1) * 1e3 / a.reps
                tf = 2.0 * M * N * K / us / 1e6
                out.append({"precision": prec, "route": route, "M": M, "N": N, "K": K, "transA": tA, "transB": tB,
                            "us": round(us, 2), "tflops_fp32_equiv": round(tf, 1)})
                print(f"{prec:8s} {route:8s} M{M} N{N} K{K} {'T' if tA else 'N'}{'T' if tB else 'N'}: {us:9.1f} us  "
                      f"{tf:7.1f} TF/s", flush=True)
            del As, Bs, C, routes
    cu.set_matmul_precision("highest")
    # stride-2 k4 convolutions of the S encoder / decoder (1024 images): forward, transposed forward, weight gradient
    for NB, h, Cs, Cb in ((1024, 16, 64, 32), (1024, 8, 128, 64), (1024, 4, 256, 128), (1024, 32, 32, 3)):
        small = torch.randn(NB, h, h, Cs, device="cuda")
        big = torch.randn(NB, 2 * h, 2 * h, Cb, device="cuda")
        W = torch.randn(Cs, Cb, 4, 4, device="cuda") * 0.05
        dW = torch.empty_like(W)
        flops = 2.0 * NB * h * h * Cs * Cb * 16
        for name, fn in (("conv_down", lambda: cu.conv_down(big, W, small)), ("conv_up", lambda: cu.conv_up(small, W, big)),
                         ("conv_wgrad", lambda: cu.conv_wgrad(small, big, dW))):
            for _ in range(3):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(a.reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / a.reps
            out.append({"op": name, "NB": NB, "h": h, "Cs": Cs, "Cb": Cb, "us": round(us, 2),
                        "tflops_fp32_equiv": round(flops / us / 1e6, 1)})
            print(f"{name:10s} {NB}x{h}x{h}x{Cs} <-> {NB}x{2*h}x{2*h}x{Cb}: {us:8.1f} us  {flops / us / 1e6:6.1f} TF/s", flush=True)
    if a.json:
        json.dump(out, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
