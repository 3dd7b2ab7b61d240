#!/usr/bin/env python
"""clip_bench.py -- what global-norm gradient clipping and Adam weight decay cost the learner step: config 2 (|s|=17,
|a|=6, batch 256, 51 atoms, tf32x3, wgmma chains) and config 5 shapes (batch 4096, n-step 5, 101 atoms, bf16, level
plan), each with the options off, with clipping on both networks, and with weight decay alone.

    python tools/clip_bench.py [--steps 300] [--regions 5] [--warmup 400] [--max-norm 1e-3]

The three learners of a configuration live in one process and their timed regions alternate, so clock and co-tenant
drift hit all alike.  A region is `--steps` device-sampled DDPG.train_n steps (CUDA-graph replays) between CUDA events
on the learner stream, after --warmup untimed steps.  --max-norm is far below the critic's gradient norm on these
workloads, so every timed step clips it (the cost does not depend on the coefficient); the last step's norms are printed
beside it.  Prints the median us/step of each variant and the
regions' spread ((max - min) / median), the per-launch device time of grad_sqnorm and Adam from one
DDPG.profile_step() (CUDA events around each launch), and one JSON line with the GPU name and power limit.  Needs a
GPU: there is no CPU fallback.
"""
import argparse
import json
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from mog_bench import gpu_info, region_us    # noqa: E402


def make(d4pg, info, B, precision, n_steps, max_grad_norm, weight_decay):
    import torch
    torch.manual_seed(0); np.random.seed(0); random.seed(0)
    n = max(16384, 4 * B)
    dd = d4pg.DDPG(17, 6, memory_size=n, batch_size=B, critic_dist_info=info, precision=precision, sampling="device",
                   n_steps=n_steps, projection="nstep" if n_steps > 1 else "reference", max_grad_norm=max_grad_norm)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), weight_decay=weight_decay),
                               d4pg.SharedAdam(dd.critic.parameters(), weight_decay=weight_decay))
    rng = np.random.RandomState(1)
    dd.replayBuffer.add_batch(rng.randn(n, 17).astype(np.float32), rng.uniform(-1, 1, (n, 6)).astype(np.float32),
                              -3 * rng.rand(n), rng.randn(n, 17).astype(np.float32), rng.rand(n) < 0.05)
    return dd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=400, help="untimed steps per learner before the first region")
    ap.add_argument("--max-norm", type=float, default=1e-3)
    ap.add_argument("--weight-decay", type=float, default=1e-4)
    args = ap.parse_args()
    import torch
    import d4pg_b200 as d4pg
    d4pg._lib.require_cuda()
    cases = {"c2_tf32x3": (256, "tf32x3", 1, {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": 51}),
             "c5_bf16": (4096, "bf16", 5, {"type": "categorical", "v_min": -150.0, "v_max": 150.0, "n_atoms": 101})}
    variants = {"off": (None, 0.0), "clip": (args.max_norm, 0.0), "decay": (None, args.weight_decay)}
    result = {"gpu": gpu_info(torch.cuda.current_device()), "steps": args.steps, "regions": args.regions,
              "max_norm": args.max_norm, "weight_decay": args.weight_decay}
    for name, (B, prec, nst, info) in cases.items():
        dds = {k: make(d4pg, info, B, prec, nst, mx, wd) for k, (mx, wd) in variants.items()}
        times = {k: [] for k in dds}
        for dd in dds.values():
            dd.train_n(max(args.warmup, 16))          # captures every graph variant; clocks and caches settle
        torch.cuda.synchronize()
        for _ in range(args.regions):
            for k, dd in dds.items():
                times[k].append(region_us(dd, args.steps))
        med = {k: float(np.median(v)) for k, v in times.items()}
        spread = {k: (max(v) - min(v)) / float(np.median(v)) for k, v in times.items()}
        norms = dds["clip"].last_grad_norms()
        result[name] = {"us_per_step": med, "regions_us": times, "spread": spread, "last_norms_clip": norms,
                        "kernels_per_step": {k: dd.kernels_per_step() for k, dd in dds.items()},
                        "clip_over_off": med["clip"] / med["off"], "decay_over_off": med["decay"] / med["off"]}
        for k, dd in dds.items():
            prof = [(n_, ms * 1000.0) for n_, ms in dd.profile_step() if n_ in ("launch_grad_sqnorm", "launch_adam")]
            result[name]["profile_" + k] = [(n_, round(us, 2)) for n_, us in prof]
            print("%s %-5s: %7.2f us/step (regions spread %.1f %%, %d launches)  %s"
                  % (name, k, med[k], 100 * spread[k], dd.kernels_per_step(),
                     "  ".join("%s %.2f us" % (n_[7:], us) for n_, us in prof)))
        print("%s: clip / off = %.4f, decay / off = %.4f; last norms under clipping (actor, critic) = %.4g, %.4g against "
              "max_norm %g" % (name, result[name]["clip_over_off"], result[name]["decay_over_off"], norms[0], norms[1],
                               args.max_norm))
        for dd in dds.values():
            dd._drop_learner()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
