#!/usr/bin/env python
"""qr_bench.py -- learner step time of the quantile-regression critic against the categorical one at the same width:
config 2 (|s|=17, |a|=6, batch 256, tf32x3, wgmma chains), 51 atoms against N=51, and config 5 shapes (batch 4096,
n-step 5, bf16), 101 atoms against N=101.

    python tools/qr_bench.py [--steps 300] [--regions 5] [--warmup 400]

Both learners of a configuration live in one process and their timed regions alternate, so clock and co-tenant drift
hit both alike.  A region is `--steps` device-sampled DDPG.train_n steps (CUDA-graph replays) between CUDA events on the
learner stream, after --warmup untimed steps.  Prints the median us/step of each and the regions' spread
((max - min) / median), then the per-launch device times of one DDPG.profile_step() (CUDA events around each launch),
and one JSON line with the GPU name and power limit.  Needs a GPU: there is no CPU fallback.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from mog_bench import gpu_info, make, region_us    # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=400, help="untimed steps per learner before the first region")
    args = ap.parse_args()
    import torch
    import d4pg_b200 as d4pg
    cases = {"c2_tf32x3": (256, "tf32x3", 1, {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": 51}),
             "c5_bf16": (4096, "bf16", 5, {"type": "categorical", "v_min": -150.0, "v_max": 150.0, "n_atoms": 101})}
    result = {"gpu": gpu_info(torch.cuda.current_device()), "steps": args.steps, "regions": args.regions}
    for name, (B, prec, nst, cat) in cases.items():
        qr = {"type": "quantile", "n_quantiles": cat["n_atoms"], "kappa": 1.0}
        dds = {"categorical": make(d4pg, cat, B, prec, nst), "quantile": make(d4pg, qr, B, prec, nst)}
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
                        "quantile_over_categorical": med["quantile"] / med["categorical"]}
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
