"""Per-phase cycle counters of the persistent RSSM scan kernels (csrc/rssm_scan.cu) at the BASELINE config:
Dreamer-V3 updates on synthetic data, counters of CTA 0 and CTA 1 read after each scan launch, averaged over the
profiled updates.

    python tools/scan_profile.py [--iters 5] [--json out.json]

Cycles convert to time through the kernels' own CUDA-event times, taken in the same launches: the clock a phase ran
at is (CTA 0's cycles of the launch) / (its event time), so the table needs no assumed SM clock.  The card's name,
power limit and SM clock are printed with it.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FWD = {0: "prologue", 12: "B1 step start + mask-mix + sync", 13: "B1 sync + slice sums", 14: "E LayerNorm", 15: "E logits product",
       1: "B1 h-part product (thread 0's warp)", 2: "A wait z (all rows)", 3: "A gather + send x_pre", 4: "B2 wait x rows, stats, normalise",
       5: "B2 product+stats send", 6: "C wait stats+merge", 7: "C gates+send h", 8: "D wait h rows", 9: "D product+send rp",
       10: "E wait rp rows", 11: "E sample + saves"}
BWD = {16: "prologue", 17: "P wait dxh_x rows+sums", 18: "P product+softmax bwd+send", 19: "Q wait d_post_raw rows",
       20: "Q product+send", 21: "R wait dxh_r rows+sums", 22: "R product+gate bwd+send", 23: "S 3x(wait+product)+sums",
       24: "S epilogue+send"}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5, help="profiled updates (after 2 warm-up updates)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scan_profile.py reads counters of kernels running on a GPU; none is visible")
    from bench import synthetic_batch
    from sheeprl_b200.configs import make_dv3_cfg
    from sheeprl_b200.engine import DV3Engine

    cfg = make_dv3_cfg("S")
    eng = DV3Engine(cfg, (2,), in_channels=3, device="cuda:0")
    from oracle import dv3_oracle as O   # initial parameters only (tool, not product)

    wm, actor, critic, target = O.init_params(cfg, (2,), seed=0)
    eng.wm.load(wm), eng.actor.load(actor), eng.critic.load(critic), eng.target.load(target)
    data = synthetic_batch(cfg, (2,), seed=1, device="cuda:0")
    acc = {"fwd": [[0] * 32, [0] * 32], "bwd": [[0] * 32, [0] * 32]}
    ms = {"fwd": [], "bwd": []}

    def timed(name, inner):
        def run(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            inner(*a, **k)
            e1.record()
            torch.cuda.synchronize()
            ms[name].append(e0.elapsed_time(e1))
            prof = eng.ops.rssm_scan_profile(eng._scan_ws)
            for cta in (0, 1):
                acc[name][cta] = [x + y for x, y in zip(acc[name][cta], prof[cta])]
        return run

    for _ in range(2):
        eng.train_step({k: v.clone() for k, v in data.items()})
    eng.ops.rssm_scan_fwd = timed("fwd", eng.ops.rssm_scan_fwd)
    eng.ops.rssm_scan_bwd = timed("bwd", eng.ops.rssm_scan_bwd)
    for _ in range(args.iters):
        eng.train_step({k: v.clone() for k, v in data.items()})
    torch.cuda.synchronize()
    assert eng.fused_scan and eng.ops.rssm_scan_error(eng._scan_ws) == 0
    T = cfg.algo.per_rank_sequence_length
    gpu = card()
    print("gpu (name, power limit, SM clock, max SM clock):", gpu)
    rep = {"gpu": gpu, "T": T, "iters": args.iters}
    for name, labels in (("fwd", FWD), ("bwd", BWD)):
        n = len(ms[name])
        kernel_ms = sum(ms[name]) / n
        mhz = sum(acc[name][0]) / n / (kernel_ms * 1e3)     # CTA 0's counters cover its whole launch
        print(f"{name}: {kernel_ms:.3f} ms per launch (CUDA events, incl. the workspace reset) = {kernel_ms * 1e3 / T:.2f} us/step; "
              f"CTA 0 counted {mhz:.0f} cycles per us")
        rep[name] = {"kernel_ms": kernel_ms, "us_per_step": kernel_ms * 1e3 / T, "cycles_per_us": mhz}
        for cta in (0, 1):
            tot = sum(acc[name][cta]) / n
            rows = {labels.get(i, str(i)): acc[name][cta][i] / n for i in range(32) if acc[name][cta][i]}
            rep[f"{name}_cta{cta}"] = {"total_cycles": tot, "us_per_step": tot / T / mhz,
                                       "cycles_per_step": {k: round(v / T, 1) for k, v in rows.items()}}
            print(f"  cta {cta}: {tot / T:.0f} cycles/step = {tot / T / mhz:.2f} us/step")
            for k, v in rows.items():
                print(f"    {k:36s} {v / T:10.1f} cycles/step")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(rep, f, indent=1)


if __name__ == "__main__":
    main()
