"""Plan2Explore exploration update on the DIAMBRA shape (`reward` encoded only, the MLP decoder over `[opp, own]`)
through the C-ABI against the executed reference (tests/golden/p2e_dec_diambra.pt)."""
import pytest

from tests.test_p2e_cpu import check_engine, make_engine
from tests.test_p2e_decoder_keys_cpu import load

pytestmark = pytest.mark.gpu


def test_engine_cuda_matches_reference():
    from sheeprl_b200.lib import CudaOps

    fx, cfg = load()
    eng = make_engine(fx, cfg, device="cuda", ops=CudaOps())
    assert eng.has_vec_dec and not eng.vec_dec_same
    check_engine(fx, cfg, eng)
