"""SHA-256 of every tensor-core product route on seeded inputs, in both matmul precisions: the shapes of
tools/gemm_bench.py, the fused split-K LayerNorm / GRU tails and the S convolution layers (forward, transposed forward,
weight gradient).  Two builds that must compute the same bits write the same JSON.

    python tools/gemm_hash.py --json out.json
    python tools/gemm_hash.py --json new.json --compare old.json     # exit status 1 on any difference
"""
import argparse, hashlib, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from sheeprl_b200.lib import CudaOps

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gemm_bench import SHAPES, gemm_presplit, planes  # noqa: E402

CONV_LAYERS = ((1024, 16, 64, 32), (1024, 8, 128, 64), (1024, 4, 256, 128))   # NB, h, Cs, Cb (tensor-core eligible)


def draw(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, generator=g, device="cuda") * scale


def digest(t):
    torch.cuda.synchronize()
    return hashlib.sha256(t.contiguous().view(torch.int32).cpu().numpy().tobytes()).hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", required=True)
    ap.add_argument("--compare", default=None, help="a JSON written by this tool to compare against")
    a = ap.parse_args()
    cu = CudaOps("cuda")
    out = {}
    for prec in ("highest", "high"):
        cu.set_matmul_precision(prec)
        for i, (M, N, K, tA, tB) in enumerate(SHAPES):
            A = draw((K, M) if tA else (M, K), 100 * i + 1)
            B = draw((N, K) if tB else (K, N), 100 * i + 2)
            C = torch.empty(M, N, device="cuda")
            cu.gemm(A, B, C, tA, tB)
            tag = f"{prec}/gemm_M{M}_N{N}_K{K}_{'T' if tA else 'N'}{'T' if tB else 'N'}"
            out[tag] = digest(C)
            if not tA:              # B as pre-split TF32 planes: must give the raw-B bits
                C.fill_(float("nan"))
                gemm_presplit(cu, A, planes(cu, B, tB), C)
                out[tag + "_presplit"] = digest(C)
            del A, B, C
        # the imagination tails: product + LayerNorm + SiLU, product + LayerNorm + GRU gate
        M, N, K = 1024, 512, 1536
        A, W = draw((M, K), 7), draw((N, K), 8)
        gamma, beta = 1.0 + draw((N,), 9, 0.1), draw((N,), 10, 0.1)
        o, p = torch.empty(M, N, device="cuda"), torch.empty(M, N, device="cuda")
        cu.gemm_ln_act(A, W, gamma, beta, 1e-3, 1, o, p)
        out[f"{prec}/gemm_ln_act"], out[f"{prec}/gemm_ln_act_pre"] = digest(o), digest(p)
        M, R = 1024, 512
        N, K = 3 * R, R + 1024
        A, W = draw((M, K), 11), draw((N, K), 12)
        gamma, beta, h_prev = 1.0 + draw((N,), 13, 0.1), draw((N,), 14, 0.1), draw((M, R), 15, 0.5)
        h = torch.empty(M, R, device="cuda")
        cu.gemm_ln_gru(A, W, gamma, beta, 1e-3, h_prev, h)
        out[f"{prec}/gemm_ln_gru"] = digest(h)
        for NB, h_, Cs, Cb in CONV_LAYERS:
            small, big = draw((NB, h_, h_, Cs), 16), draw((NB, 2 * h_, 2 * h_, Cb), 17)
            W, b = draw((Cs, Cb, 4, 4), 18, 0.05), draw((Cb,), 19)
            s, bg, dW = torch.empty_like(small), torch.empty_like(big), torch.empty_like(W)
            cu.conv_down(big, W, s)
            cu.conv_up(small, W, bg, b)
            cu.conv_wgrad(small, big, dW)
            tag = f"{prec}/conv_{NB}x{h_}x{h_}x{Cs}_{Cb}"
            out[tag + "_down"], out[tag + "_up"], out[tag + "_wgrad"] = digest(s), digest(bg), digest(dW)
    cu.set_matmul_precision("highest")
    json.dump(out, open(a.json, "w"), indent=1, sort_keys=True)
    print(f"{len(out)} outputs hashed -> {a.json}")
    routes = sorted(k for k in out if k.endswith("_presplit") and out[k] != out[k[: -len("_presplit")]])
    for k in routes:
        print(f"PRE-SPLIT DIFFERS FROM RAW B: {k}")
    if a.compare:
        ref = json.load(open(a.compare))
        both = set(ref) & set(out)
        diff = sorted(k for k in both if ref[k] != out[k])
        for k in diff:
            print(f"DIFFERS: {k}")
        print(f"{len(both) - len(diff)} / {len(both)} outputs both builds hash bit-identical to {a.compare}"
              f" ({len(set(ref) ^ set(out))} routes hashed by one build only)")
        sys.exit(1 if diff or routes else 0)
    sys.exit(1 if routes else 0)


if __name__ == "__main__":
    main()
