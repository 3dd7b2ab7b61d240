#!/usr/bin/env python
"""act_bench.py -- what one rollout step's action selection costs, DDPG.act against the reference's idiom
(main.py:145-146, 216-217, 279), with observation normalization on, at E environments per call.

    python tools/act_bench.py [--es 1,64,1024,4096] [--iters 200] [--regions 5] [--launches 1000]

For each shape (c2: |s|=17, |a|=6; c3: |s|=376, |a|=17) and E, in one process with alternating timed regions:
  reference  np.clip(actor(s).cpu().numpy() + eps * np.random.normal(mu, var, (E, |a|)), -1, 1)   host s
  act        ddpg.act(s).cpu().numpy()                                                          host s
  wall time per call (host clock; both end in a device-to-host copy, so the device work is inside).  Then the device
  time of one act launch (explore=True) against actor(s) (the normalizer launch + d4pg_actor_forward's four launches):
  CUDA events around `--launches` calls on device input with a 16-B row pitch, so act copies nothing.
Prints the median us of each and one JSON line with the GPU name and power limit.  Needs a GPU.
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
from mog_bench import gpu_info    # noqa: E402

SHAPES = {"c2": (17, 6), "c3": (376, 17)}
INFO = {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": 51}


def make(d4pg, S, A):
    torch.manual_seed(0); np.random.seed(0); random.seed(0)
    dd = d4pg.DDPG(S, A, memory_size=4096, batch_size=64, critic_dist_info=INFO, obs_norm=True)
    rng = np.random.RandomState(1)
    dd.replayBuffer.add_batch(rng.randn(4096, S).astype(np.float32), rng.uniform(-1, 1, (4096, A)).astype(np.float32),
                              -3 * rng.rand(4096), rng.randn(4096, S).astype(np.float32), rng.rand(4096) < 0.05)
    return dd


def reference_step(dd, s):
    nz = dd.noise
    a = dd.actor(s).cpu().numpy()
    return np.clip(a + nz.epsilon * np.random.normal(nz.mu, nz.var, size=a.shape), -1, 1)


def act_step(dd, s):
    return dd.act(s).cpu().numpy()


def wall_us(fn, dd, s, iters):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn(dd, s)
    return 1e6 * (time.perf_counter() - t0) / iters


def device_us(fn, launches):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        fn()
    e1.record()
    e1.synchronize()
    return 1000.0 * e0.elapsed_time(e1) / launches


def main():
    global torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--es", default="1,64,1024,4096")
    ap.add_argument("--iters", type=int, default=200, help="calls per wall-time region")
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--launches", type=int, default=1000, help="calls per device-time measurement")
    args = ap.parse_args()
    import torch
    import d4pg_b200 as d4pg
    d4pg._lib.require_cuda()
    result = {"gpu": gpu_info(torch.cuda.current_device()), "iters": args.iters, "regions": args.regions,
              "launches": args.launches}
    rng = np.random.RandomState(2)
    for name, (S, A) in SHAPES.items():
        dd = make(d4pg, S, A)
        for E in [int(e) for e in args.es.split(",")]:
            s = rng.randn(E, S).astype(np.float32)
            variants = {"reference": reference_step, "act": act_step}
            for fn in variants.values():
                wall_us(fn, dd, s, max(10, args.iters // 10))          # warm-up: buffers, module loads
            times = {k: [] for k in variants}
            for _ in range(args.regions):
                for k, fn in variants.items():
                    times[k].append(wall_us(fn, dd, s, args.iters))
            med = {k: float(np.median(v)) for k, v in times.items()}
            spread = {k: (max(v) - min(v)) / med[k] for k, v in times.items()}
            P = (S + 3) & ~3
            sd = torch.zeros(E, P, device="cuda")[:, :S]
            sd.copy_(torch.from_numpy(s))
            dev = {"act_launch": device_us(lambda: dd.act(sd), args.launches),
                   "actor_forward": device_us(lambda: dd.actor(sd), args.launches)}
            key = "%s_E%d" % (name, E)
            result[key] = {"wall_us": med, "wall_regions_us": times, "wall_spread": spread, "device_us": dev}
            print("%s E=%-5d wall: reference %8.1f us  act %8.1f us (spread %.1f / %.1f %%)   device: act %7.2f us  "
                  "actor() %7.2f us" % (name, E, med["reference"], med["act"], 100 * spread["reference"],
                                        100 * spread["act"], dev["act_launch"], dev["actor_forward"]))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
