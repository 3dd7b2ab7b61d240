#!/usr/bin/env python
"""mog_bench.py -- learner step time of the mixture-of-Gaussians critic (K=5) against the categorical one (51 / 101
atoms), at config 2 (|s|=17, |a|=6, batch 256, tf32x3, wgmma chains) and config 5 shapes (batch 4096, n-step 5, bf16).

    python tools/mog_bench.py [--steps 300] [--regions 5] [--warmup 400]

All four learners live in one process and, per configuration, the timed regions of the two heads alternate, so clock
and co-tenant drift hit both alike.  A region is `--steps` device-sampled DDPG.train_n steps (CUDA-graph replays)
between CUDA events on the learner stream, after --warmup untimed steps (the first few hundred steps of a fresh process run
a few percent slow).  Prints the median us/step of each and the regions' spread ((max - min) / median), then the per-launch device times of one
DDPG.profile_step() (CUDA events around each launch), and one JSON line with the GPU name and power limit.
Needs a GPU: there is no CPU fallback.
"""
import argparse
import json
import os
import random
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info(index):
    out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit",
                          "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
    f = [x.strip() for x in out.stdout.strip().split(",")]
    if out.returncode != 0 or len(f) < 2:
        return {"name": None, "power_limit_w": None}
    return {"name": f[0], "power_limit_w": float(f[1])}


def make(d4pg, info, B, precision, n_steps):
    import torch
    torch.manual_seed(0); np.random.seed(0); random.seed(0)
    n = max(16384, 4 * B)
    dd = d4pg.DDPG(17, 6, memory_size=n, batch_size=B, critic_dist_info=info, precision=precision, sampling="device",
                   n_steps=n_steps, projection="nstep" if n_steps > 1 else "reference")
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters()), d4pg.SharedAdam(dd.critic.parameters()))
    rng = np.random.RandomState(1)
    dd.replayBuffer.add_batch(rng.randn(n, 17).astype(np.float32), rng.uniform(-1, 1, (n, 6)).astype(np.float32),
                              -3 * rng.rand(n), rng.randn(n, 17).astype(np.float32), rng.rand(n) < 0.05)
    return dd


def region_us(dd, steps):
    import torch
    L = dd._learner
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(L.stream)
    dd.train_n(steps)
    e1.record(L.stream)
    e1.synchronize()
    return 1000.0 * e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=400, help="untimed steps per learner before the first region")
    args = ap.parse_args()
    import torch
    import d4pg_b200 as d4pg
    mog = {"type": "mixture_of_gaussian", "n_components": 5}
    cases = {"c2_tf32x3": (256, "tf32x3", 1, {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": 51}),
             "c5_bf16": (4096, "bf16", 5, {"type": "categorical", "v_min": -150.0, "v_max": 150.0, "n_atoms": 101})}
    result = {"gpu": gpu_info(torch.cuda.current_device()), "steps": args.steps, "regions": args.regions}
    for name, (B, prec, nst, cat) in cases.items():
        dds = {"categorical": make(d4pg, cat, B, prec, nst), "mog_k5": make(d4pg, mog, B, prec, nst)}
        times = {k: [] for k in dds}
        for dd in dds.values():
            dd.train_n(max(args.warmup, 16))          # captures every graph variant; clocks and caches settle
        torch.cuda.synchronize()
        for _ in range(args.regions):
            for k, dd in dds.items():
                times[k].append(region_us(dd, args.steps))
        med = {k: float(np.median(v)) for k, v in times.items()}
        spread = {k: (max(v) - min(v)) / float(np.median(v)) for k, v in times.items()}
        result[name] = {"us_per_step": med, "regions_us": times, "spread": spread,
                        "mog_over_categorical": med["mog_k5"] / med["categorical"]}
        for k, dd in dds.items():
            prof = dd.profile_step()
            result[name]["profile_" + k] = [(n_, round(ms * 1000.0, 2)) for n_, ms in prof]
            print("%s %s: %.2f us/step (regions spread %.1f %%)" % (name, k, med[k], 100 * spread[k]))
            for n_, ms in prof:
                print("    %-28s %8.2f us" % (n_, ms * 1000.0))
        for dd in dds.values():
            dd._drop_learner()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
