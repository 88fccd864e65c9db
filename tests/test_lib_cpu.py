"""CPU-side checks of the native library: it builds, loads, and exports every symbol the header declares; the binding
takes every prototype and struct from the header and refuses malformed calls before entering the library; the routing
queries answer on the host.  No kernel is launched here (no GPU in this container)."""
import ctypes
import os
import re
import subprocess

import pytest

from sheeprl_b200 import lib as L

# Routing-query boundaries, shared with the GPU test that checks each launch accepts exactly what its query accepts
# (tests/test_gpu_ops.py).  Offsets are in floats from a 16-byte aligned address; row strides are the row widths.
HEAD_SAMPLE = {            # Kin, A, X offset, W offset -> b200rl_head_sample_supported
    "A32_Kin1024": (1024, 32, 0, 0, True), "A33": (64, 33, 0, 0, False), "Kin1028": (1028, 8, 0, 0, False),
    "Kin_not_multiple_of_4": (510, 8, 0, 0, False), "X_misaligned": (512, 8, 1, 0, False),
    "W_misaligned": (512, 8, 0, 1, False),
}
ONEHOT_LINEAR = {          # S, K, A, N, out offset -> (gather form, fused-LayerNorm form)
    "N128": (4, 4, 2, 128, 0, True, True), "N1024": (4, 4, 2, 1024, 0, True, True),
    "N1152": (4, 4, 2, 1152, 0, True, False), "N_not_multiple_of_128": (4, 4, 2, 192, 0, True, False),
    "S64": (64, 4, 2, 128, 0, True, True), "S65": (65, 4, 2, 128, 0, False, False),
    "A32": (4, 4, 32, 128, 0, True, True), "A33": (4, 4, 33, 128, 0, False, False),
    "out_misaligned": (4, 4, 2, 128, 1, True, False),
}
WGRAD_TC = {               # NB, h, w, Cs, Cb -> b200rl_conv_wgrad_tc_supported
    "P1024": (1, 32, 32, 48, 8, True), "P1023": (1, 1023, 1, 48, 8, False), "Cs47": (1, 32, 32, 47, 8, False),
    "Cb7": (1, 32, 32, 48, 7, False), "P2e9": (2000000000, 1, 1, 48, 8, True),
    "P_above_2e9": (2000000001, 1, 1, 48, 8, False),
}
LN_ROUTE = {               # C, row stride (all three rows), base offset of (row 0, row 1, row 2, gamma) -> route
    "vec_C32": (32, 32, (0, 0, 0, 0), 1), "vec_C48": (48, 48, (0, 0, 0, 0), 1), "vec_C640": (640, 640, (0, 0, 0, 0), 1),
    "vec_C1536": (1536, 1536, (0, 0, 0, 0), 1), "vec_C256_ld260": (256, 260, (0, 0, 0, 0), 1),
    "vec_C256_ld257": (256, 257, (0, 0, 0, 0), 0), "vec_C256_dX_misaligned": (256, 256, (0, 0, 1, 0), 0),
    "vec_C256_gamma_misaligned": (256, 256, (0, 0, 0, 1), 0), "C100": (100, 100, (0, 0, 0, 0), 0),
    "C1537": (1537, 1540, (0, 0, 0, 0), 0), "C2050_not_multiple_of_4": (2050, 2052, (0, 0, 0, 0), 0),
    "wide_C1540": (1540, 1540, (0, 0, 0, 0), 2), "wide_C16384": (16384, 16384, (0, 0, 0, 0), 2),
    "C16388": (16388, 16388, (0, 0, 0, 0), 0), "wide_C3072_ld3073": (3072, 3073, (0, 0, 0, 0), 0),
    "wide_C3072_X_misaligned": (3072, 3072, (1, 0, 0, 0), 0), "C1": (1, 1, (0, 0, 0, 0), 0),
}
ADDR = 1 << 20             # synthetic 16-byte aligned device address: the queries compare pointer values only


@pytest.fixture(scope="module")
def built():
    from sheeprl_b200.build import build

    return build()


@pytest.fixture(scope="module")
def lib(built):
    return L.load_library(built)


def test_library_exports_every_declared_symbol(built):
    lib = ctypes.CDLL(built)
    names = L.declared_symbols()
    assert len(names) >= 40
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing


def test_library_identity(built):
    lib = L.load_library()
    assert lib.b200rl_abi_version() == 1
    assert lib.b200rl_build_arch() == b"sm_90a"


def test_every_declared_function_is_bound(lib):
    with open(L.HEADER_PATH) as f:
        header = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    names = sorted(set(re.findall(r"\b(b200rl_\w+)\s*\(", header)))
    assert names == list(L.declared_symbols())
    unbound = [n for n in names if getattr(lib, n).argtypes is None]
    assert not unbound, unbound
    P, I = ctypes.c_void_p, ctypes.c_int
    assert lib.b200rl_gemm_f32.argtypes == [P] * 4 + [I] * 9 + [P] and lib.b200rl_gemm_f32.restype is I
    assert lib.b200rl_fill_exponential.argtypes == [P, ctypes.c_longlong, ctypes.c_ulonglong, ctypes.c_uint, P, P]
    assert lib.b200rl_conv_pack_floats.restype is ctypes.c_longlong
    assert lib.b200rl_conv_pack_floats(1, 64, 32) == 36 * 64 * 32
    assert lib.b200rl_last_error.restype is ctypes.c_char_p and isinstance(lib.b200rl_last_error(), bytes)


@pytest.mark.parametrize("header", ["int b200rl_f(int n, double x, cudaStream_t stream);",
                                    "size_t b200rl_f(int n);",
                                    "typedef struct s { int n; short k; } s;\nint b200rl_g(void);"])
def test_parser_refuses_types_outside_the_table(header):
    where = "b200rl_f" if "b200rl_f" in header else "s"
    with pytest.raises(L.B200RLError, match=f"{where}: C type"):
        L.parse_header(header)


def test_bad_calls_raise_before_entering_the_library(lib):
    with pytest.raises(TypeError, match="takes 3 arguments"):
        lib.b200rl_conv_pack_floats(1, 64)                              # too few
    with pytest.raises(TypeError, match="takes 2 arguments"):
        lib.b200rl_thin_up_supported(32, 3, 0)                          # too many: ctypes alone passes them on
    with pytest.raises(ctypes.ArgumentError):
        lib.b200rl_conv_wgrad_tc_supported(1.0, 32, 32, 48, 8)          # a float where an int is declared
    with pytest.raises(ctypes.ArgumentError):
        lib.b200rl_head_sample_supported(ADDR, ADDR, 64, 8, ctypes.c_int(64), 64)    # c_int for a long long


def test_scan_structs_match_the_c_layout(tmp_path):
    """Every field of the two ctypes structs at the offset, size and kind (pointer / float / integer) the C compiler
    gives it, and the same struct sizes."""
    from sheeprl_b200.build import NVCC

    kind = {ctypes.c_void_p: "p", ctypes.c_float: "f", ctypes.c_int: "i", ctypes.c_longlong: "i"}
    structs = {"b200rl_rssm_scan_args": L.RssmScanArgs, "b200rl_rssm_scan_grads": L.RssmScanGrads}
    lines, want = [], []
    for cname, st in structs.items():
        lines.append(f'std::printf("{cname} %zu\\n", sizeof({cname}));')
        want.append(f"{cname} {ctypes.sizeof(st)}")
        for name, t in st._fields_:
            m = f"(({cname}*)0)->{name}"
            lines.append(f'std::printf("{name} %zu %zu %c\\n", offsetof({cname}, {name}), sizeof({m}), '
                         f"std::is_pointer<decltype({m})>::value ? 'p' : "
                         f"std::is_floating_point<decltype({m})>::value ? 'f' : 'i');")
            want.append(f"{name} {getattr(st, name).offset} {getattr(st, name).size} {kind[t]}")
    src = tmp_path / "layout.cpp"
    src.write_text("#include <cstddef>\n#include <cstdio>\n#include <type_traits>\n#include \"b200rl.h\"\n"
                   "int main() {\n" + "\n".join(lines) + "\nreturn 0;\n}\n")
    exe = str(tmp_path / "layout")
    subprocess.run([NVCC, "-std=c++17", "-I", os.path.dirname(L.HEADER_PATH), str(src), "-o", exe], check=True)
    got = subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split("\n")
    assert got[:-1] == want
    assert len(L.RssmScanArgs.POINTERS) == 38 and "workspace" not in L.RssmScanArgs.POINTERS
    assert len(L.RssmScanGrads.POINTERS) == len(L.RssmScanGrads._fields_) == 17


@pytest.mark.parametrize("case", list(HEAD_SAMPLE))
def test_head_sample_query_boundaries(lib, case):
    Kin, A, xo, wo, ok = HEAD_SAMPLE[case]
    assert lib.b200rl_head_sample_supported(ADDR + 4 * xo, 2 * ADDR + 4 * wo, Kin, A, Kin, Kin) == ok


@pytest.mark.parametrize("case", list(ONEHOT_LINEAR))
def test_onehot_linear_query_boundaries(lib, case):
    S, K, A, N, oo, gather, ln = ONEHOT_LINEAR[case]
    assert lib.b200rl_onehot_linear_supported(S, K, A, N) == gather
    fused = lib.b200rl_onehot_linear_ln_supported(ADDR, 2 * ADDR, 3 * ADDR, 4 * ADDR + 4 * oo, None, N, N, 0)
    assert bool(gather and fused) == ln


def test_onehot_linear_ln_query_alignment(lib):
    """the LayerNorm parameters and the optional `pre` output need 16-byte aligned rows too; a NULL `pre` passes"""
    assert lib.b200rl_onehot_linear_ln_supported(ADDR, 2 * ADDR, 3 * ADDR, 4 * ADDR, None, 128, 128, 0)
    assert not lib.b200rl_onehot_linear_ln_supported(ADDR, 2 * ADDR + 4, 3 * ADDR, 4 * ADDR, None, 128, 128, 0)
    assert not lib.b200rl_onehot_linear_ln_supported(ADDR, 2 * ADDR, 3 * ADDR, 4 * ADDR, 5 * ADDR + 8, 128, 128, 128)
    assert not lib.b200rl_onehot_linear_ln_supported(ADDR, 2 * ADDR, 3 * ADDR, 4 * ADDR, 5 * ADDR, 128, 128, 130)


@pytest.mark.parametrize("case", list(LN_ROUTE))
def test_ln_act_route_query(lib, case):
    C, ld, (o0, o1, o2, og), route = LN_ROUTE[case]
    assert lib.b200rl_ln_act_route(C, ld, ld, ld, ADDR + 4 * o0, 2 * ADDR + 4 * o1, 3 * ADDR + 4 * o2, 4 * ADDR + 4 * og,
                                   5 * ADDR) == route
    if o2 == 0:                # the forward passes no third row: ld2 = 0, p2 = NULL
        assert lib.b200rl_ln_act_route(C, ld, ld, 0, ADDR + 4 * o0, 2 * ADDR + 4 * o1, None, 4 * ADDR + 4 * og,
                                       5 * ADDR) == route


@pytest.mark.parametrize("case", list(WGRAD_TC))
def test_conv_wgrad_tc_query_boundaries(lib, case):
    *shape, ok = WGRAD_TC[case]
    assert lib.b200rl_conv_wgrad_tc_supported(*shape) == ok


def test_product_path_refuses_to_run_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from sheeprl_b200.configs import make_dv3_cfg
    from sheeprl_b200.engine import DV3Engine

    with pytest.raises(L.B200RLError):
        DV3Engine(make_dv3_cfg("S", per_rank_batch_size=2, per_rank_sequence_length=2), (2,), device="cuda")


def test_product_never_imports_oracle():
    root = os.path.dirname(os.path.abspath(L.__file__))
    for dp, _, files in os.walk(root):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, os.path.join(dp, f)
