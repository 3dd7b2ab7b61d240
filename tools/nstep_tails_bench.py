#!/usr/bin/env python
"""nstep_tails_bench.py -- what episode tails (DDPG(nstep_tails=True), DESIGN.md §3 "Episode tails") cost.

    python tools/nstep_tails_bench.py [--steps 200] [--regions 6] [--calls 200]

1. Learner step time with tails off and on at the c2 shapes (|s|=17, |a|=6, 51 atoms, B=256) and the c5 shapes
   (101 atoms, B=4096), both bf16, n_steps = 5, projection "nstep", device sampling.  The tails-on replay holds 10 % tail
   rows of horizons 1-4.  After a warm-up of every variant, timed regions of --steps train() calls alternate between
   off and on; each region runs to a synchronise.  Prints the median step time per variant and the spread of the
   regions ((max - min) / median).
2. add_steps per call at E = 1024 / 4096 (c2 shapes, n = 5, CUDA inputs) with tails off and on, on calls where a third
   of the environments ended at the previous call: wall time to a synchronise, and device time between CUDA events.
Ends with one JSON line with everything and the GPU name and power limit read in the same run.  Needs a GPU.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from mog_bench import gpu_info    # noqa: E402

CFG = {"c2": dict(S=17, A=6, atoms=51, v=(-50.0, 0.0), B=256, cap=1 << 20),
       "c5": dict(S=17, A=6, atoms=101, v=(-150.0, 150.0), B=4096, cap=1 << 20)}
N = 5


def learner(name, tails):
    import torch
    import d4pg_b200 as d4pg
    c = CFG[name]
    info = {"type": "categorical", "v_min": c["v"][0], "v_max": c["v"][1], "n_atoms": c["atoms"]}
    torch.manual_seed(0)
    dd = d4pg.DDPG(c["S"], c["A"], memory_size=c["cap"], batch_size=c["B"], critic_dist_info=info, n_steps=N,
                   projection="nstep", sampling="device", precision="bf16", nstep_tails=tails)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-4),
                               d4pg.SharedAdam(dd.critic.parameters(), lr=1e-4))
    rng = np.random.RandomState(0)
    n = c["cap"]
    dd.replayBuffer.add_batch(torch.as_tensor(rng.randn(n, c["S"]).astype(np.float32)).cuda(),
                              torch.as_tensor(rng.uniform(-1, 1, (n, c["A"])).astype(np.float32)).cuda(),
                              torch.as_tensor(-rng.rand(n)).cuda(),
                              torch.as_tensor(rng.randn(n, c["S"]).astype(np.float32)).cuda(),
                              torch.as_tensor(rng.rand(n) < 0.02).cuda())
    if tails:                                  # 10 % tail rows, horizons 1..n-1
        h = dd.replayBuffer._store.horizon
        sel = torch.as_tensor(rng.rand(n) < 0.1).cuda()
        h[sel] = torch.as_tensor(rng.randint(1, N, n).astype(np.uint8)).cuda()[sel]
    return dd


def bench_learner(steps, regions):
    import torch
    out = {}
    for name in CFG:
        dds = {t: learner(name, t) for t in (False, True)}
        for dd in dds.values():
            for _ in range(30):
                dd.train()
        torch.cuda.synchronize()
        times = {False: [], True: []}
        for r in range(regions):
            for t in ((False, True) if r % 2 == 0 else (True, False)):
                dd = dds[t]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(steps):
                    dd.train()
                torch.cuda.synchronize()
                times[t].append((time.perf_counter() - t0) / steps * 1e6)
        for t, v in times.items():
            med = float(np.median(v))
            out["%s_%s" % (name, "on" if t else "off")] = dict(us_per_step=med, spread=(max(v) - min(v)) / med)
        del dds
    return out


def bench_add_steps(calls):
    import torch
    import d4pg_b200 as d4pg
    S, A = CFG["c2"]["S"], CFG["c2"]["A"]
    out = {}
    for E in (1024, 4096):
        rng = np.random.RandomState(E)
        pool = []
        for k in range(8):
            ended = torch.zeros(E, dtype=torch.bool)
            ended[k % 3::3] = True                 # a third of the environments end at every call
            pool.append((torch.as_tensor(rng.randn(E, S).astype(np.float32)).cuda(), torch.rand(E, A, device="cuda"),
                         torch.rand(E, dtype=torch.float64, device="cuda"),
                         torch.as_tensor(rng.randn(E, S).astype(np.float32)).cuda(),
                         torch.zeros(E, dtype=torch.bool, device="cuda"), ended.cuda()))
        for tails in (False, True):
            buf = d4pg.PrioritizedReplayBuffer(1 << 20, 0.6, obs_dim=S, act_dim=A, nstep_tails=tails)
            for k in range(20):
                buf.add_steps(*pool[k % 8], n_steps=N, gamma=0.99)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            rows = 0
            t0 = time.perf_counter()
            e0.record()
            for k in range(calls):
                rows += buf.add_steps(*pool[k % 8], n_steps=N, gamma=0.99)
            e1.record()
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) / calls * 1e6
            out["E%d_%s" % (E, "on" if tails else "off")] = dict(us_wall_per_call=wall,
                                                                   us_device_per_call=e0.elapsed_time(e1) / calls * 1e3,
                                                                   rows_per_call=rows / calls)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--regions", type=int, default=6)
    ap.add_argument("--calls", type=int, default=200)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "nstep_tails_bench.py needs a GPU"
    res = dict(gpu=gpu_info(0), learner=bench_learner(args.steps, args.regions), add_steps=bench_add_steps(args.calls))
    for k, v in res["learner"].items():
        print("learner %-8s %8.1f us/step  spread %.1f %%" % (k, v["us_per_step"], 100 * v["spread"]))
    for k, v in res["add_steps"].items():
        print("add_steps %-9s wall %7.1f us  device %7.1f us  rows %.0f" % (k, v["us_wall_per_call"],
                                                                          v["us_device_per_call"], v["rows_per_call"]))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
