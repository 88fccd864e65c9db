"""Data parallelism with a decoder absent: two gloo ranks drive the engine (op specification as test double) on the
Crafter shape (no MLP decoder) and on an image-encoder-only shape (no CNN decoder), with the world-model gradient
all-reduced in its three buckets (encoder | rssm | decoders, reward, continue) as the backward finishes each.  The
buckets must tile the flat gradient, and the reduced gradient must be the mean of the single-process gradients."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = ["dv3_dec_crafter", "dv3_dec_nocnn"]


def _engine(name):
    from oracle.ops_emul_decoupled import DecoupledEmulOps
    from sheeprl_b200.engine import DV3Engine
    from tests.helpers import image_channels, load_fixture

    fx, cfg = load_fixture(name)
    cfg.algo.overlap_allreduce = True                  # the bucketed reductions, whatever the scan route
    eng = DV3Engine(cfg, fx["actions_dim"], in_channels=image_channels(cfg), device="cpu", ops=DecoupledEmulOps(),
                    is_continuous=fx["is_continuous"])
    eng.wm.load(fx["init"]["wm"]), eng.actor.load(fx["init"]["actor"]), eng.critic.load(fx["init"]["critic"])
    eng.target.load(fx["init"]["target"])
    return fx, eng


def _worker(rank, world, port, name, out):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(2)
    from sheeprl_b200.parallel import attach_data_parallel, init_process_group_from_env

    init_process_group_from_env("gloo")
    fx, eng = _engine(name)
    attach_data_parallel(eng)
    calls = []
    inner = eng.allreduce_async
    eng.allreduce_async = lambda sl: (calls.append((sl.storage_offset(), sl.numel())), inner(sl))
    eng.train_step({k: v.clone().float() for k, v in fx["data"][rank].items()}, fx["noise"][rank])
    out[rank] = {"wm": eng.wm.flat.clone(), "actor": eng.actor.flat.clone(), "critic": eng.critic.flat.clone(),
                 "wm_grad": eng.wm.grad.clone(), "calls": calls}
    dist.destroy_process_group()


@pytest.mark.parametrize("name", FIXTURES)
def test_two_rank_gloo_buckets_with_a_decoder_absent(name):
    mp.set_start_method("spawn", force=True)
    out = mp.Manager().dict()
    port = 31900 + FIXTURES.index(name) * 50 + (os.getpid() % 50)
    mp.spawn(_worker, args=(2, port, name, out), nprocs=2, join=True)
    a, b = out[0], out[1]
    for k in ("wm", "actor", "critic", "wm_grad"):
        assert torch.equal(a[k], b[k]), k
    sys.path.insert(0, ROOT)
    grads = []
    for r in range(2):
        fx, eng = _engine(name)
        eng.train_step({k: v.clone().float() for k, v in fx["data"][r].items()}, fx["noise"][r])
        grads.append(eng.wm.grad.clone())
    # the three buckets: tail, rssm, encoder — contiguous, in that order, covering the whole flat gradient
    base = eng.wm.grad.storage_offset()
    (t0, tn), (r0, rn), (e0, en) = [(o - base, n) for o, n in a["calls"]]
    assert e0 == 0 and e0 + en == r0 and r0 + rn == t0 and t0 + tn == eng.wm.grad.numel()
    off = eng.wm.offsets
    for k, o in off.items():
        want = 0 if k.startswith("encoder.") else 1 if k.startswith("rssm.") else 2
        assert (0 if o < r0 else 1 if o < t0 else 2) == want, k
    assert not (eng.has_cnn_dec and eng.has_vec_dec)                     # one decoder is absent
    want = 0.5 * (grads[0] + grads[1])
    assert float((a["wm_grad"] - want).abs().max()) <= 1e-5 * float(want.abs().max())
