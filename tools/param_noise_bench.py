#!/usr/bin/env python
"""param_noise_bench.py -- the device cost of adaptive parameter-space noise.

    python tools/param_noise_bench.py [--launches 500] [--regions 7]

In one process, CUDA events around `--launches` back-to-back calls per region, the variants of each row alternating
region by region, median over `--regions` (and the spread, (max - min) / median):
  perturb  ddpg.perturb_actor()  at c2 (|s|=17, |a|=6) and c3 (|s|=376, |a|=17): one actor_perturb_kernel launch
  adapt    ddpg.adapt_param_noise(states) at B = 256 and 1024, both shapes: perturb + 2 x d4pg_act + adapt kernel
  act      ddpg.act(s) at E = 1, 64, 1024 (c2 and c3, obs_norm on, device input with a 16-B row pitch):
           "gaussian" = the default GaussianNoise, no parameter noise; "param" = param_noise with noise = None;
           "param+gaussian" = both.  All three run the same act_chain_kernel; the parameter-noise variants read the
           perturbed actor's buffer.
At small sizes these regions measure how fast the host issues the calls, not the kernels.  So the kernels' own device
durations are read afterwards with torch.profiler over `--profiled` calls of each op (median per kernel name).
Prints one line per row and one JSON line with the GPU name and power limit.  Needs a GPU.
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
from mog_bench import gpu_info    # noqa: E402

SHAPES = {"c2": (17, 6), "c3": (376, 17)}
INFO = {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": 51}


def make(d4pg, S, A):
    torch.manual_seed(0); np.random.seed(0); random.seed(0)
    dd = d4pg.DDPG(S, A, memory_size=4096, batch_size=64, critic_dist_info=INFO, obs_norm=True,
                   param_noise=d4pg.AdaptiveParamNoiseSpec())
    rng = np.random.RandomState(1)
    dd.replayBuffer.add_batch(rng.randn(4096, S).astype(np.float32), rng.uniform(-1, 1, (4096, A)).astype(np.float32),
                              -3 * rng.rand(4096), rng.randn(4096, S).astype(np.float32), rng.rand(4096) < 0.05)
    return dd


def pitched(rng, E, S):
    x = torch.zeros(E, (S + 3) & ~3, device="cuda")[:, :S]
    x.copy_(torch.from_numpy(rng.randn(E, S).astype(np.float32)))
    return x


def region_us(fn, launches):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        fn()
    e1.record()
    e1.synchronize()
    return 1000.0 * e0.elapsed_time(e1) / launches


def compare(variants, launches, regions):
    """{name: (median us, spread, [region us])} with the variants alternating region by region."""
    for fn in variants.values():
        for _ in range(10):
            fn()                                              # warm-up: buffers, module loads
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    for _ in range(regions):
        for k, fn in variants.items():
            times[k].append(region_us(fn, launches))
    out = {}
    for k, v in times.items():
        med = float(np.median(v))
        out[k] = {"median_us": med, "spread": (max(v) - min(v)) / med, "regions_us": v}
    return out


def kernel_us(fn, calls):
    """{kernel name: median device duration in us} of the kernels `calls` calls of fn launch (torch.profiler)."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    dur = {}
    for e in prof.events():
        if e.device_type == DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset")):
            name = e.name.split("(")[0].split("<")[0].replace("d4pg::", "")
            dur.setdefault(name, []).append(e.time_range.elapsed_us())
    return {k: float(np.median(v)) for k, v in dur.items()}


def main():
    global torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=500, help="calls per timed region")
    ap.add_argument("--regions", type=int, default=7)
    ap.add_argument("--profiled", type=int, default=50, help="calls per kernel-duration measurement")
    args = ap.parse_args()
    import torch
    import d4pg_b200 as d4pg
    d4pg._lib.require_cuda()
    result = {"gpu": gpu_info(torch.cuda.current_device()), "launches": args.launches, "regions": args.regions}
    rng = np.random.RandomState(2)

    def show(key, r):
        result[key] = r
        print("%-22s " % key + "  ".join("%s %8.2f us (spread %4.1f %%)" % (k, v["median_us"], 100 * v["spread"])
                                         for k, v in r.items()))
    for name, (S, A) in SHAPES.items():
        dd = make(d4pg, S, A)
        show("%s_perturb" % name, compare({"perturb_actor": dd.perturb_actor}, args.launches, args.regions))
        for B in (256, 1024):
            s = pitched(rng, B, S)
            show("%s_adapt_B%d" % (name, B), compare({"adapt_param_noise": lambda: dd.adapt_param_noise(s)},
                                                     args.launches, args.regions))
        s = pitched(rng, 256, S)
        for what, fn in (("perturb", dd.perturb_actor), ("adapt_B256", lambda: dd.adapt_param_noise(s))):
            k = result["%s_kernels_%s" % (name, what)] = kernel_us(fn, args.profiled)
            print("%-22s kernels: " % ("%s_%s" % (name, what)) + "  ".join("%s %.2f us" % kv for kv in k.items()))
        spec, gauss = dd.param_noise, dd.noise

        def variant(pn, nz, s):
            def run():
                dd.param_noise, dd.noise = pn, nz
                dd.act(s)
            return run
        for E in (1, 64, 1024):
            s = pitched(rng, E, S)
            show("%s_act_E%d" % (name, E), compare({"gaussian": variant(None, gauss, s), "param": variant(spec, None, s),
                                                    "param+gaussian": variant(spec, gauss, s)},
                                                   args.launches, args.regions))
        dd.param_noise, dd.noise = spec, gauss
    print(json.dumps(result))


if __name__ == "__main__":
    main()
