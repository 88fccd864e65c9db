"""Recurrent PPO train() calls on one GPU (eager), next to the reference's own train() (torch eager, cuDNN LSTM) on the
same GPU when the reference package is present under oracle/_ref (placed there by build()):

    python tests/perf/bench_ppo_recurrent.py [--steps 200]        -> one JSON line per workload

(lives under tests/: it uses the oracle's rollout generator and the reference harness, which only tests/, smoke() and
bench.py may import)
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def timed_eager(step, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def bench_ppo_recurrent(args, cu):
    """Recurrent PPO train() at the default experiment shapes (configs/exp/ppo_recurrent.yaml: 16 envs x 512 rollout
    steps cut into sequences of 16, 8 batches, 8 epochs, LSTM 64) on vector observations, the same with LSTM 256, and on
    84x84 x 4 stacked frames; next to the reference's own train() in torch eager (cuDNN LSTM) on the same GPU."""
    from oracle import ppo_recurrent_oracle as RO
    from oracle import ref_harness
    from oracle.make_golden_ppo import obs_space
    from oracle.make_golden_ppo_recurrent import rec_cfg
    from sheeprl_b200.algos.ppo.agent import default_init
    from sheeprl_b200.algos.ppo_recurrent.engine import RecurrentPPOEngine

    hp = dict(clip_coef=0.2, vf_coef=0.2, ent_coef=0.001, clip_vloss=False, normalize_advantages=False, max_grad_norm=0.5)
    opt = {"lr": 3e-4, "eps": 1e-4, "betas": (0.9, 0.999)}
    T, n_batches, epochs = 16, 8, 8
    g = torch.Generator().manual_seed(0)
    lengths = [16] * 512 + torch.randint(1, 16, (48,), generator=g).tolist()   # episode ends add short tail sequences
    S = len(lengths)
    workloads = {
        "vector_h64": dict(cnn_channels=0, screen=0, mlp_dim=8, dense=64, layers=1, layer_norm=True, cnn_features=512,
                           mlp_features=64, actions_dim=(4,), is_continuous=False, act="relu",
                           rnn=dict(hidden=64, pre=None, post=None)),
        "vector_h256": dict(cnn_channels=0, screen=0, mlp_dim=8, dense=64, layers=1, layer_norm=True, cnn_features=512,
                            mlp_features=64, actions_dim=(4,), is_continuous=False, act="relu",
                            rnn=dict(hidden=256, pre=None, post=None)),
        "pixel84x4_h64": dict(cnn_channels=4, screen=84, mlp_dim=0, dense=64, layers=1, layer_norm=True,
                              cnn_features=512, mlp_features=64, actions_dim=(6,), is_continuous=False, act="relu",
                              rnn=dict(hidden=64, pre=None, post=None)),
    }
    ref_ok = ref_harness.reference_available()
    if ref_ok:
        ref_harness.install()
        torch.distributions.Distribution.set_default_validate_args(False)   # padded rows (see DESIGN.md)
    for name, spec in workloads.items():
        eng = RecurrentPPOEngine(spec, hp, opt, "cuda", cu)
        init = default_init(eng.reference_shapes(), torch.Generator().manual_seed(1))
        eng.load_reference_state(init)
        data = RO.make_rollout(spec, T, lengths, seed=2)
        dev = {k: v.cuda() for k, v in data.items()}
        if "rgb" in dev:
            dev["rgb"] = dev["rgb"].to(torch.uint8)
        B = S // n_batches
        batches = [torch.randperm(S, generator=g)[i * B:(i + 1) * B].tolist() for i in range(n_batches)] * epochs
        prepared = eng.prepare(dev)
        seqs = torch.as_tensor(batches[0]).cuda()
        eng.minibatch_step(prepared, seqs)
        l0 = cu.launches
        eng.minibatch_step(prepared, seqs)
        launches = cu.launches - l0
        us_mb = timed_eager(lambda: eng.minibatch_step(prepared, seqs), args.steps) * 1e3
        eng.train(dev, batches)
        ms_train = timed_eager(lambda: eng.train(dev, batches), max(3, args.steps // 40))
        assert torch.isfinite(eng.losses).all()
        ref = None
        if ref_ok:
            import sheeprl.algos.ppo_recurrent.agent as RA
            import sheeprl.algos.ppo_recurrent.ppo_recurrent as RP

            RA.get_single_device_fabric = lambda f: f
            cfg = rec_cfg(spec, hp, n_batches, epochs)
            fab = ref_harness.FakeFabric("cuda")
            agent, _ = RA.build_agent(fab, spec["actions_dim"], False, cfg, obs_space(spec), None)
            ropt = torch.optim.Adam(agent.parameters(), lr=3e-4, eps=1e-4)
            rdata = {k: v.cuda() for k, v in data.items()}
            f = lambda: RP.train(fab, agent, ropt, rdata, None, cfg)  # noqa: E731
            f()
            ms_ref = timed_eager(f, max(3, args.steps // 40))
            ref = {"ms_per_train_call": ms_ref, "kind": "reference train(), torch eager, cuDNN LSTM, same GPU"}
        print(json.dumps({"metric": f"recurrent PPO train() [{name}] (T=16, {S} sequences, {n_batches} batches x "
                                    f"{epochs} epochs)", "value": ms_train, "unit": "ms/train call",
                          "us_per_minibatch": us_mb, "gpu_launches_per_minibatch": launches,
                          "minibatches_per_train_call": len(batches), "reference": ref}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    args = ap.parse_args()
    from sheeprl_b200.lib import CudaOps

    bench_ppo_recurrent(args, CudaOps())


if __name__ == "__main__":
    main()
