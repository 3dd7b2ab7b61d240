#!/usr/bin/env python
"""obs_norm_bench.py -- what observation normalization (DDPG(obs_norm=True)) costs: the device-sampled learner step at
config 2 (|s|=17, |a|=6, batch 256, 51 atoms, tf32x3, wgmma chains) and config 5 shapes (batch 4096, n-step 5, 101
atoms, bf16, level plan), each off and on, and an end-to-end pair through DDPG.train() (host pipeline) with a 256-row
add_batch before every step, whose statistics launch runs on the learner's ingest stream.

    python tools/obs_norm_bench.py [--steps 300] [--regions 5] [--warmup 400] [--e2e-steps 1000]

The two learners of a configuration live in one process and their timed regions alternate.  A learner region is
`--steps` DDPG.train_n steps between CUDA events on the learner stream; an e2e region is `--e2e-steps` iterations of
add_batch + train() timed by the host clock up to a device synchronize.  Prints the median us/step of each variant and
the regions' spread ((max - min) / median), the kernel time of one statistics launch for 256 rows and for 10^6 rows
(CUDA events over repeated launches), and one JSON line with the GPU name and power limit.  Needs a GPU.
"""
import argparse
import json
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from mog_bench import gpu_info, region_us    # noqa: E402


def rows(rng, n):
    scales = np.logspace(-2, 2, 17)
    return ((rng.randn(n, 17) * scales).astype(np.float32), rng.uniform(-1, 1, (n, 6)).astype(np.float32),
            -3 * rng.rand(n), (rng.randn(n, 17) * scales).astype(np.float32), rng.rand(n) < 0.05)


def make(d4pg, info, B, precision, n_steps, obs_norm, sampling="device"):
    import torch
    torch.manual_seed(0); np.random.seed(0); random.seed(0)
    n = max(16384, 4 * B)
    dd = d4pg.DDPG(17, 6, memory_size=n, batch_size=B, critic_dist_info=info, precision=precision, sampling=sampling,
                   n_steps=n_steps, projection="nstep" if n_steps > 1 else "reference", obs_norm=obs_norm)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters()), d4pg.SharedAdam(dd.critic.parameters()))
    dd.replayBuffer.add_batch(*rows(np.random.RandomState(1), n))
    return dd


def e2e_region_us(dd, steps, batches):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        dd.replayBuffer.add_batch(*batches[i % len(batches)])
        dd.train()
    torch.cuda.synchronize()
    return 1e6 * (time.perf_counter() - t0) / steps


def stats_kernel_us(d4pg, n, reps):
    """Device time of one d4pg_obs_norm_update launch (the statistics kernel an insert runs) on n rows of 17 features."""
    import torch
    from d4pg_b200 import _lib
    norm = d4pg.ObsNormalizer(obs_dim=17)
    x = torch.from_numpy(rows(np.random.RandomState(2), n)[0]).cuda()
    fn = _lib.lib().d4pg_obs_norm_update
    args = (_lib.ptr(norm.stats), _lib.ptr(norm.affine), 17, _lib.ptr(x), n, 17, norm.eps, _lib.stream_ptr())
    _lib.check(fn(*args))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn(*args)
    e1.record()
    e1.synchronize()
    return 1000.0 * e0.elapsed_time(e1) / reps


def summary(times):
    med = {k: float(np.median(v)) for k, v in times.items()}
    spread = {k: (max(v) - min(v)) / float(np.median(v)) for k, v in times.items()}
    return med, spread


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=400, help="untimed steps per learner before the first region")
    ap.add_argument("--e2e-steps", type=int, default=1000)
    args = ap.parse_args()
    import torch
    import d4pg_b200 as d4pg
    d4pg._lib.require_cuda()
    c2 = {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": 51}
    cases = {"c2_tf32x3": (256, "tf32x3", 1, c2),
             "c5_bf16": (4096, "bf16", 5, {"type": "categorical", "v_min": -150.0, "v_max": 150.0, "n_atoms": 101})}
    result = {"gpu": gpu_info(torch.cuda.current_device()), "steps": args.steps, "regions": args.regions}
    for name, (B, prec, nst, info) in cases.items():
        dds = {k: make(d4pg, info, B, prec, nst, on) for k, on in (("off", None), ("on", True))}
        times = {k: [] for k in dds}
        for dd in dds.values():
            dd.train_n(max(args.warmup, 16))
        torch.cuda.synchronize()
        for _ in range(args.regions):
            for k, dd in dds.items():
                times[k].append(region_us(dd, args.steps))
        med, spread = summary(times)
        result[name] = {"us_per_step": med, "regions_us": times, "spread": spread, "on_over_off": med["on"] / med["off"],
                        "kernels_per_step": {k: dd.kernels_per_step() for k, dd in dds.items()}}
        for k in dds:
            print("%s %-3s: %8.2f us/step (regions spread %.1f %%, %d launches)"
                  % (name, k, med[k], 100 * spread[k], dds[k].kernels_per_step()))
        print("%s: on / off = %.4f" % (name, med["on"] / med["off"]))
        for dd in dds.values():
            dd._drop_learner()
    # end to end: host pipeline, one 256-row add per step (its statistics launch on the ingest stream when on)
    rng = np.random.RandomState(3)
    batches = [rows(rng, 256) for _ in range(16)]
    dds = {k: make(d4pg, c2, 256, "tf32x3", 1, on, sampling="reference") for k, on in (("off", None), ("on", True))}
    for dd in dds.values():
        e2e_region_us(dd, max(args.warmup, 16), batches)
    times = {k: [] for k in dds}
    for _ in range(args.regions):
        for k, dd in dds.items():
            times[k].append(e2e_region_us(dd, args.e2e_steps, batches))
    med, spread = summary(times)
    result["e2e_c2_add256"] = {"us_per_step": med, "regions_us": times, "spread": spread,
                               "on_over_off": med["on"] / med["off"]}
    for k in dds:
        print("e2e c2 add256+train %-3s: %8.2f us/step (regions spread %.1f %%)" % (k, med[k], 100 * spread[k]))
    result["stats_kernel_us"] = {"rows_256": stats_kernel_us(d4pg, 256, 200), "rows_1e6": stats_kernel_us(d4pg, 10 ** 6, 3)}
    print("statistics launch: %.2f us for 256 rows, %.1f ms for 10^6 rows (17 features)"
          % (result["stats_kernel_us"]["rows_256"], result["stats_kernel_us"]["rows_1e6"] / 1000.0))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
